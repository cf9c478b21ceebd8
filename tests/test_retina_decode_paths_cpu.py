"""Decode_TRT (tensorrtx_b200/csrc/retina_decode.cu) in float64, and a mirror of how trtx_retina_decode_enqueue dispatches a call.

The float64 reference follows the reference's CalDetection (retinaface/decode.cu:110-165, retinafaceAntiCov/decode.cu:110-155)
with INPUT_H / INPUT_W made runtime and every image of the batch decoded.  Per image its rows come in ascending prior order
(level, cell, k), the order the pack writes.

  * Priors decide where a row goes, so they are built with the fp32 / fp64 expressions of the reference, which numpy
    reproduces bit for bit: RetinaFace `(float)(((double)x + 0.5) / w)` and `(float)anchor * (k + 1) / in_w` (one fp32
    division), AntiCov `7.5 + x * step` with the level's fixed stride 8, 16, 32 and the integer `anchor * 2 / (k + 1)`.
  * Everything after the priors is float64: exp, the box algebra, the landmarks and the conf softmax.  Where the kernel
    rounds to fp32, a float64 value of magnitude >= 2^128 - 2^103 becomes +-inf, and expf is +0 below ln 2^-150 and +inf
    above ln(2^128 - 2^103), as fp32 would have it.  So inf and NaN come out where the kernel's fp32 arithmetic makes them.

Error bound of each column, from the fp32 arithmetic of the kernel (u = 2^-24 and ud = 2^-53 the fp32 and fp64 unit
roundoffs; every fp32 operation rounds once, by at most u times its result):
  * CUDA expf is within 2 ulp, and an ulp of a normal result r is at most 2u |r|: expf(t) = exp(t) (1 + 4u).
  * RetinaFace centre `bx = p0 + v * 0.1 * p2`: three double roundings (the last two may be one FMA) and the reference's own
    float64 ones, then one rounding to fp32: e_bx = u |bx| + 8 ud (|p0| + |v 0.1 p2|).
  * RetinaFace size `bw = p2 * expf((float)(v * 0.2))`: the argument t rounds to fp32, which moves exp(t) by |t| u relative
    (taken as 1.01 |t| u for the second order), expf adds 4u and the product u: e_bw = (1.01 |t| + 6) u |bw|.  AntiCov
    reads v as the argument, so e_bw = 5.1 u |bw| there.  A subnormal expf result has an absolute error of 2^-148 instead;
    both bounds add p2 2^-147.
  * AntiCov centre `bx = prior + v * prior2` in fp32, contracted into one FMA or not: e_bx = u (|v p2| + |bx|).
  * `x1 -= w / 2` (w / 2 is exact): e_x1 = e_bx + e_bw / 2 + u |x1|.  AntiCov's `x1 -= (w - 1) / 2` rounds w - 1 as well:
    e_x1 = e_bx + (e_bw + u |w - 1|) / 2 + u |x1|.
  * `x2 += x1`: e_x2 = e_bw + e_x1 + u |x2|.
  * RetinaFace `*= in_w`: e_out = in_w e + u |out|; the same for y with in_h.
  * Landmarks `prior + v * 0.1 * prior2` (AntiCov 0.2) are the double expression of the centre: u |l| + 8 ud (...), then
    RetinaFace's `*= in_w`.
  * RetinaFace conf `p = expf(c2) / (expf(c1) + expf(c2))`: 4u from each expf, u from the sum and u from the division:
    10.5 u |p|.  AntiCov's conf and mask conf are copies: bound 0, compared bit for bit.
The reference and the bound hold for logits outside [-104.5, -87] (where expf is subnormal and loses its relative precision)
and away from ln(2^128 - 2^103) = 88.72; the generators below keep to that.  A random RetinaFace prior whose |p - gate| is
within 4x its conf bound would be kept or dropped by rounding alone, so the generators resample its logits.

The CPU tests check that the C oracle (oracle/trtx_oracle.c) lies within the bound on every shape class, that each injected
defect of the decode moves some value by more than 1000x its bound (or changes the kept set) wherever it changes anything,
and that every injected defect fails the comparison.  tests/test_retina_decode_paths_gpu.py holds the device to the same
comparison."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import pytest

from tensorrtx_b200 import synth

F32 = np.float32
U = 2.0 ** -24
UD = 2.0 ** -53
OVF = 2.0 ** 128 - 2.0 ** 103             # the smallest float64 magnitude that rounds to fp32 inf
EXP_OVER = math.log(OVF)                  # expf(t) = +inf above
EXP_UNDER = math.log(2.0 ** -150)         # expf(t) = +0 below
SUB = 2.0 ** -147                         # absolute error bound of a subnormal expf result, with margin

FACE, ANTICOV = 0, 1                      # trtx_retina_params.variant
VARIANTS = {FACE: "face", ANTICOV: "anticov"}
CHANNELS = {FACE: 32, ANTICOV: 38}
DET = {FACE: 15, ANTICOV: 16}
STRIDES = (8, 16, 32)
LEVEL_ANCHOR = (16, 64, 256)
KERNEL = {FACE: "retina_scan_kernel", ANTICOV: "anticov_scan_kernel"}
DTYPE_SIZE = {"f32": 4, "f16": 2}
DTYPE_T = {"f32": "float", "f16": "__half"}
PACK_CHUNK = 1024                         # retina_pack_kernel's kPackChunk


def float_le(x: float) -> float:
    """the largest fp32 t <= x: `(double)p <= x` is `p <= t` for an fp32 p"""
    t = F32(x)
    return float(t if float(t) <= x else np.nextafter(t, F32(-np.inf)))


GATE = float_le(0.02)                     # DecodePlugin's gate (decode.cu:131)

# (in_h, in_w) shape classes, and what each is for
SHAPES = [(640, 640),     # VEC=4, retina_b16's size
          (480, 640),     # VEC=4, the size the reference compiles in
          (488, 648),     # g odd at level 0: VEC=1
          (32, 32),       # the minimum: one partial tile per level
          (64, 64),       # VEC=4, every tile partial
          (640, 660),     # 660 / 20 = 33 at level 2
          (640, 40),      # 40 / 2 = 20 at level 1, 40 / 1 = 40 at level 2
          (1080, 1920),   # large, uneven level sizes
          (4480, 4480)]   # 12 863 tiles at VEC=1: past what one shared-memory prefix of 48 KB held


def shape_id(s):
    return f"{s[0]}x{s[1]}"


def batches(shape):
    h, w = shape
    if h * w > 1080 * 1920:
        return [1]
    return [1, 3, 16] + ([64] if h * w <= 64 * 64 else [])


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror: trtx_retina_decode_enqueue and retina_layout
# ---------------------------------------------------------------------------------------------------------------------
def grids(in_h, in_w):
    """per level (gh, gw, g) with floor grids per axis"""
    return [(in_h // s, in_w // s, (in_h // s) * (in_w // s)) for s in STRIDES]


def total_priors(in_h, in_w):
    return sum(2 * g for _, _, g in grids(in_h, in_w))


def _align(v, a=256):
    return (v + a - 1) // a * a


def dispatch(variant, dtype, in_h, in_w, batch, addr_mod=(0, 0, 0)):
    """what trtx_retina_decode_enqueue launches for heads whose byte addresses are addr_mod modulo 16: the scan
    instantiation, its tiles per image and level offsets, the pack's passes, the workspace the call needs and the size
    trtx_retina_workspace_size reports"""
    es = DTYPE_SIZE[dtype]
    vec = 4
    for (_, _, g), m in zip(grids(in_h, in_w), addr_mod):
        if g % 4 != 0 or m % (4 * es) != 0:
            vec = 1

    def layout(v):
        tiles, slots, tile_begin = 0, 0, []
        for _, _, g in grids(in_h, in_w):
            tile_begin.append(tiles)
            tiles += -(-g // (32 * v))
            slots += 2 * g
        return tiles, slots, tile_begin, _align(4 * batch * tiles) + _align(4 * 16 * batch * slots)

    tiles, slots, tile_begin, need = layout(vec)
    return dict(kernel=f"{KERNEL[variant]}<{DTYPE_T[dtype]}, {vec}>", vec=vec, tiles=tiles, tile_begin=tile_begin,
                slots=slots, pack_passes=-(-tiles // PACK_CHUNK), workspace=need, workspace_size=layout(1)[3])


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
DEFECTS = {FACE: ("no_half", "swap_wh", "anchor_k", "lmk_scale", "gate_strictness"),
           ANTICOV: ("step_from_width", "lmk_scale", "half_width", "gate_strictness")}


def priors(variant, in_h, in_w, defect=None):
    """per prior in (level, cell, k) order: (p0, p1, p2, p3) as float64 arrays holding the fp32 priors the reference
    computes.  defect: 'no_half' (a RetinaFace centre without + 0.5), 'swap_wh' (in_w and in_h exchanged in p2 and p3),
    'anchor_k' (anchor * (2 - k) for anchor * (k + 1)), 'step_from_width' (the AntiCov step in_w / w)."""
    out = [[], [], [], []]
    for (gh, gw, g), s, anchor in zip(grids(in_h, in_w), STRIDES, LEVEL_ANCHOR):
        cell = np.repeat(np.arange(g), 2)
        k = np.tile(np.arange(2), g)
        y, x = np.divmod(cell, gw)
        if variant == FACE:
            half = 0.0 if defect == "no_half" else 0.5
            p0 = ((x + half) / gw).astype(F32)
            p1 = ((y + half) / gh).astype(F32)
            a = F32(anchor) * ((2 - k) if defect == "anchor_k" else (k + 1)).astype(F32)
            dw, dh = (in_h, in_w) if defect == "swap_wh" else (in_w, in_h)
            p2, p3 = a / F32(dw), a / F32(dh)
        else:
            step = in_w // gw if defect == "step_from_width" else s
            p0 = (7.5 + x * step).astype(F32)
            p1 = (7.5 + y * step).astype(F32)
            p2 = p3 = (anchor * 2 // (k + 1)).astype(F32)
        for o, v in zip(out, (p0, p1, p2, p3)):
            o.append(v.astype(np.float64))
    return [np.concatenate(o) for o in out]


def _ovf(x):
    """a float64 result the kernel rounds to fp32: +-inf where fp32 overflows"""
    return np.where(np.abs(x) >= OVF, np.copysign(np.inf, x), x)


def _expf(t):
    """expf's value range in float64: +0 below ln 2^-150, +inf above ln(2^128 - 2^103)"""
    return np.where(t < EXP_UNDER, 0.0, np.where(t > EXP_OVER, np.inf, np.exp(np.minimum(t, 700.0))))


def face_conf(c1, c2):
    e1, e2 = _expf(c1), _expf(c2)
    return e2 / (e1 + e2)


@dataclass
class Ref:
    counts: np.ndarray       # [B]
    rows: list               # per image [n, F] float64
    bound: list              # per image [n, F]
    prior: list              # per image [n] prior index in (level, cell, k) order


def _gather(heads, variant, B, keep_fn):
    """(image, prior, per-prior channel values [n, C]) of the kept priors, image-major and in prior order"""
    bs, ps, vals = [], [], []
    base = 0
    for h in heads:
        h = np.asarray(h).reshape(B, CHANNELS[variant], -1)
        g = h.shape[2]
        keep = keep_fn(h)                                       # [B, g, 2]
        b, cell, k = np.nonzero(keep)
        ch = np.arange(CHANNELS[variant])
        v = h[b[:, None], ch[None, :], cell[:, None]].astype(np.float64)   # [n, C]
        bs.append(b)
        ps.append(base + cell * 2 + k)
        vals.append(np.concatenate([v, k[:, None].astype(np.float64)], 1))
        base += 2 * g
    b, p, v = np.concatenate(bs), np.concatenate(ps), np.concatenate(vals)
    order = np.lexsort((p, b))
    return b[order], p[order], v[order]


def reference(heads, variant, in_h, in_w, gate=GATE, defect=None):
    """float64 rows, bounds and prior indices of every image.  heads: the three levels' [B, C, g] (float32, or float16
    widened exactly); gate: the fp32 trtx_retina_params.gate (RetinaFace only).  defect: one of DEFECTS[variant]."""
    B = np.asarray(heads[0]).shape[0]
    P = priors(variant, in_h, in_w, defect)
    with np.errstate(all="ignore"):
        if variant == FACE:
            def keep_fn(h):
                c = h[:, 8:12].astype(np.float64)
                p = np.stack([face_conf(c[:, 0], c[:, 1]), face_conf(c[:, 2], c[:, 3])], -1)
                return ~(p < gate) if defect == "gate_strictness" else ~(p <= gate)
        else:
            def keep_fn(h):
                c = np.stack([h[:, 2], h[:, 3]], -1).astype(np.float64)
                return ~(c <= 0.5) if defect == "gate_strictness" else ~(c < 0.5)
        b, p, v = _gather(heads, variant, B, keep_fn)
        k = v[:, -1].astype(np.int64)
        kk = np.arange(len(k))
        p0, p1, p2, p3 = (q[p] for q in P)
        F = DET[variant]
        rows, bound = np.empty((len(p), F)), np.empty((len(p), F))
        if variant == FACE:
            bbox = v[kk[:, None], 4 * k[:, None] + np.arange(4)]
            lmk = v[kk[:, None], 12 + 10 * k[:, None] + np.arange(10)]
            cls = v[kk[:, None], 8 + 2 * k[:, None] + np.arange(2)]
            ls = 0.2 if defect == "lmk_scale" else 0.1
            for col, (pc, pw, scale) in enumerate(((p0, p2, in_w), (p1, p3, in_h))):
                t = bbox[:, col] * 0.1 * pw
                bx = _ovf(pc + t)
                e_bx = U * np.abs(bx) + 8 * UD * (np.abs(pc) + np.abs(t))
                a = _ovf(bbox[:, 2 + col] * 0.2)
                bw = _ovf(pw * _expf(a))
                e_bw = np.where(bw == 0, 0.0, (1.01 * np.abs(a) + 6) * U * np.abs(bw)) + pw * SUB   # a = -inf: bw = 0
                x1 = _ovf(bx - bw / 2)
                e_x1 = e_bx + e_bw / 2 + U * np.abs(x1)
                x2 = _ovf(bw + x1)
                e_x2 = e_bw + e_x1 + U * np.abs(x2)
                for c, (x, e) in ((col, (x1, e_x1)), (col + 2, (x2, e_x2))):
                    rows[:, c] = _ovf(x * scale)
                    bound[:, c] = e * scale + U * np.abs(rows[:, c])
            rows[:, 4] = face_conf(cls[:, 0], cls[:, 1])
            bound[:, 4] = 10.5 * U * np.abs(rows[:, 4])
            for i in range(10):
                pc, pw, scale = (p0, p2, in_w) if i % 2 == 0 else (p1, p3, in_h)
                t = lmk[:, i] * ls * pw
                lv = _ovf(pc + t)
                e = U * np.abs(lv) + 8 * UD * (np.abs(pc) + np.abs(t))
                rows[:, 5 + i] = _ovf(lv * scale)
                bound[:, 5 + i] = e * scale + U * np.abs(rows[:, 5 + i])
        else:
            bbox = v[kk[:, None], 4 + 4 * k[:, None] + np.arange(4)]
            lmk = v[kk[:, None], 12 + 10 * k[:, None] + np.arange(10)]
            conf = v[kk, 2 + k]
            mask = v[kk, 36 + k]
            ls = 0.1 if defect == "lmk_scale" else 0.2
            for col, (pc, pw) in enumerate(((p0, p2), (p1, p3))):
                t = bbox[:, col] * pw
                bx = _ovf(pc + t)
                e_bx = U * (np.abs(t) + np.abs(bx))
                bw = _ovf(pw * _expf(bbox[:, 2 + col]))
                e_bw = 5.1 * U * np.abs(bw) + pw * SUB
                if defect == "half_width":
                    x1 = _ovf(bx - bw / 2)
                    e_x1 = e_bx + e_bw / 2 + U * np.abs(x1)
                else:
                    x1 = _ovf(bx - (bw - 1) / 2)
                    e_x1 = e_bx + (e_bw + U * np.abs(bw - 1)) / 2 + U * np.abs(x1)
                x2 = _ovf(bw + x1)
                rows[:, col], bound[:, col] = x1, e_x1
                rows[:, col + 2], bound[:, col + 2] = x2, e_bw + e_x1 + U * np.abs(x2)
            rows[:, 4], bound[:, 4] = conf, 0.0
            for i in range(10):
                pc, pw = (p0, p2) if i % 2 == 0 else (p1, p3)
                t = lmk[:, i] * ls * pw
                rows[:, 5 + i] = _ovf(pc + t)
                bound[:, 5 + i] = U * np.abs(rows[:, 5 + i]) + 8 * UD * (np.abs(pc) + np.abs(t))
            rows[:, 15], bound[:, 15] = mask, 0.0
    counts = np.bincount(b, minlength=B)
    cut = np.concatenate([[0], np.cumsum(counts)])
    sl = lambda a: [a[cut[i]:cut[i + 1]] for i in range(B)]
    return Ref(counts, sl(rows), sl(bound), sl(p))


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
COLUMN_GROUPS = {FACE: {"box": slice(0, 4), "conf": slice(4, 5), "lmk": slice(5, 15)},
                 ANTICOV: {"box": slice(0, 4), "conf": slice(4, 5), "lmk": slice(5, 15), "mask": slice(15, 16)}}


def canonical_bits(x):
    """fp32 bits with every NaN made one NaN"""
    x = np.ascontiguousarray(x, F32)
    return np.where(np.isnan(x), F32(np.nan), x).view(np.uint32)


def split_output(out, variant, B):
    """the plugin buffer [B, 1 + total_priors * F] -> (counts [B], per image rows [count, F] fp32)"""
    F = DET[variant]
    out = np.asarray(out, F32).reshape(B, -1)
    counts = out[:, 0]
    assert np.all(counts == np.floor(counts)) and np.all(counts >= 0), counts
    n = counts.astype(np.int64)
    return n, [out[b, 1:1 + n[b] * F].reshape(n[b], F) for b in range(B)]


def assert_matches(out, ref: Ref, variant, msg=""):
    """The decoded buffer `out` [B, 1 + total_priors * F] (fp32) against the float64 reference: the count of every image
    exactly; non-finite values where the reference has them, of the same kind; every finite value within its column's
    bound, and bound-0 (copied) columns bit for bit.  Returns {column group: (largest |out - ref| / bound, and the error and
    bound where it is)}."""
    B = len(ref.counts)
    counts, rows = split_output(out, variant, B)
    assert np.array_equal(counts, ref.counts), (msg, "counts", counts.tolist()[:8], ref.counts.tolist()[:8])
    stats = {g: (0.0, 0.0, 0.0) for g in COLUMN_GROUPS[variant]}
    for b in range(B):
        got, r, tol = rows[b].astype(np.float64), ref.rows[b], ref.bound[b]
        fin = np.isfinite(r)
        same_kind = np.where(fin, np.isfinite(got), (np.isnan(got) == np.isnan(r)) & ((got == r) | np.isnan(r)))
        if not same_kind.all():
            i = tuple(np.argwhere(~same_kind)[0])
            raise AssertionError(f"{msg}: image {b} row {i[0]} (prior {ref.prior[b][i[0]]}) column {i[1]}: got {got[i]!r}, "
                                 f"reference {r[i]!r}")
        exact = tol == 0
        if exact.any():
            ok = canonical_bits(rows[b])[exact] == canonical_bits(r.astype(F32))[exact]
            assert ok.all(), (msg, f"image {b}: copied column differs", np.argwhere(exact)[np.argmin(ok)])
        with np.errstate(invalid="ignore"):
            err = np.where(fin, np.abs(got - r), 0.0)
        bad = fin & ~(err <= tol)
        if bad.any():
            i = tuple(np.argwhere(bad)[0])
            raise AssertionError(f"{msg}: image {b}: {int(bad.sum())} of {int(fin.sum())} values off the float64 reference, "
                                 f"first at row {i[0]} (prior {ref.prior[b][i[0]]}) column {i[1]}: got {got[i]!r}, reference "
                                 f"{r[i]!r}, bound {tol[i]:.3g}")
        for g, s in COLUMN_GROUPS[variant].items():
            e, t = err[:, s][fin[:, s]], tol[:, s][fin[:, s]]
            if len(e):
                ratio = np.where(e > 0, e / np.where(t > 0, t, 1.0), 0.0)
                i = int(np.argmax(ratio))
                if ratio[i] > stats[g][0]:
                    stats[g] = (float(ratio[i]), float(e[i]), float(t[i]))
    return stats


def defect_ratio(bad: Ref, ref: Ref):
    """the largest |defective - reference| / bound over the values of rows kept by both (inf where a copied column
    changes); None when the kept sets differ"""
    if not np.array_equal(bad.counts, ref.counts) or any(not np.array_equal(a, c) for a, c in zip(bad.prior, ref.prior)):
        return None
    worst = 0.0
    for a, r, t in zip(bad.rows, ref.rows, ref.bound):
        with np.errstate(all="ignore"):
            d = np.abs(a - r)
            ratio = np.where(np.isfinite(d) & (d > 0), d / t, 0.0)
        worst = max(worst, float(np.nanmax(ratio, initial=0.0)))
    return worst


def same(bad: Ref, ref: Ref):
    return (np.array_equal(bad.counts, ref.counts) and
            all(np.array_equal(a, c) for a, c in zip(bad.prior, ref.prior)) and
            all(np.array_equal(a, c, equal_nan=True) for a, c in zip(bad.rows, ref.rows)))


def as_output(ref: Ref, variant, in_h, in_w):
    """the plugin buffer a decode with exactly these rows (rounded to fp32) would write, zero past each image's rows"""
    F = DET[variant]
    B = len(ref.counts)
    out = np.zeros((B, 1 + total_priors(in_h, in_w) * F), F32)
    for b in range(B):
        out[b, 0] = ref.counts[b]
        with np.errstate(over="ignore"):
            out[b, 1:1 + len(ref.rows[b]) * F] = ref.rows[b].astype(F32).reshape(-1)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# heads: value classes
# ---------------------------------------------------------------------------------------------------------------------
VALUES = ("sparse", "dense", "empty", "nonfinite")

# special priors of the 'nonfinite' class: (name, {(channel offset group, index): value}); groups are 'cls' (RetinaFace
# (bg, face) logits, AntiCov face probability), 'box', 'lmk', 'mask'.  PASS marks a prior that passes the gate.
PASS = {FACE: {("cls", 0): -1.0, ("cls", 1): 3.0}, ANTICOV: {("cls", 0): 0.9}}
SPECIALS = {
    FACE: [{("cls", 1): np.nan}, {("cls", 0): np.nan}, {("cls", 0): -200.0, ("cls", 1): -200.0},
           {("cls", 0): 0.5, ("cls", 1): 95.0}, {("cls", 0): 95.0, ("cls", 1): 0.0}, {("cls", 0): 150.0, ("cls", 1): 120.0},
           {**PASS[FACE], ("box", 2): np.inf}, {**PASS[FACE], ("box", 3): -np.inf},
           {**PASS[FACE], ("box", 0): 1e30, ("box", 2): 600.0}, {**PASS[FACE], ("box", 1): -3e38, ("box", 3): -1e30},
           {**PASS[FACE], ("box", 0): np.nan}, {**PASS[FACE], ("box", 0): 3e38}, {**PASS[FACE], ("lmk", 0): np.inf, ("lmk", 3): -np.inf, ("lmk", 7): np.nan},
           {**PASS[FACE], ("box", 2): 65504.0, ("box", 0): -65504.0, ("lmk", 4): 65504.0},
           {**PASS[FACE], ("box", 0): 2.0 ** -24, ("box", 3): 6.0e-8, ("lmk", 1): -2.0 ** -20},
           {("cls", 0): -65504.0, ("cls", 1): 65504.0}],
    ANTICOV: [{("cls", 0): np.nan}, {("cls", 0): np.inf}, {("cls", 0): -np.inf}, {("cls", 0): 65504.0},
              {("cls", 0): 2.0 ** -24}, {**PASS[ANTICOV], ("box", 2): np.inf}, {**PASS[ANTICOV], ("box", 3): -np.inf},
              {**PASS[ANTICOV], ("box", 0): 1e30, ("box", 2): 100.0}, {**PASS[ANTICOV], ("box", 1): -1e30, ("box", 3): -1e30},
              {**PASS[ANTICOV], ("box", 0): 3e38}, {**PASS[ANTICOV], ("lmk", 0): np.inf, ("lmk", 5): np.nan}, {**PASS[ANTICOV], ("mask", 0): np.nan},
              {**PASS[ANTICOV], ("mask", 0): -np.inf}, {**PASS[ANTICOV], ("box", 2): 65504.0, ("lmk", 9): -65504.0},
              {**PASS[ANTICOV], ("box", 0): 2.0 ** -24, ("lmk", 2): 6.0e-8}],
}


def _channel(variant, group, i, k):
    if variant == FACE:
        return {"box": 4 * k, "cls": 8 + 2 * k, "lmk": 12 + 10 * k}[group] + i
    return {"cls": 2 + k, "box": 4 + 4 * k, "lmk": 12 + 10 * k, "mask": 36 + k}[group] + i


def _resample_gate_band(heads, rng, gate, half):
    """RetinaFace: redraw both logits of every finite prior whose |p - gate| is within 4x its conf bound"""
    for h in heads:
        for _ in range(20):
            with np.errstate(all="ignore"):
                c = h[:, 8:12].astype(np.float64)
                p = np.stack([face_conf(c[:, 0], c[:, 1]), face_conf(c[:, 2], c[:, 3])], 1)   # [B, 2, g]
                band = np.abs(p - gate) <= 4 * 10.5 * U * np.abs(p)
            if not band.any():
                break
            b, k, cell = np.nonzero(band)
            for j in (0, 1):
                v = rng.normal(0.0, 3.0, len(b)).astype(F32)
                h[b, 8 + 2 * k + j, cell] = v.astype(np.float16).astype(F32) if half else v
        else:
            raise AssertionError("could not clear the gate band")


def make_heads(variant, in_h, in_w, B, values, seed, half=False):
    """the three levels' heads [B, C, g] float32 (fp16-representable when half) of one value class:
    sparse: the synth generators; dense: every prior passes the gate; empty: none does; nonfinite: sparse heads with the
    SPECIALS written over some priors of every level (different ones per image)"""
    rng = np.random.default_rng(seed)
    if values in ("sparse", "nonfinite"):
        gen = synth.retina_heads if variant == FACE else synth.anticov_heads
        heads = gen(B, seed=seed, in_h=in_h, in_w=in_w)
    else:
        heads = []
        for _, _, g in grids(in_h, in_w):
            h = rng.standard_normal((B, CHANNELS[variant], g), dtype=np.float32)
            h[:, 4 if variant == ANTICOV else 0:][:, :8] *= F32(0.5)
            if variant == FACE:
                lo = rng.uniform(-3.0, 1.0, (B, 2, g))
                gap = rng.uniform(5.0, 10.0, (B, 2, g))                     # p > 0.993 or p < 0.0068
                dense = values == "dense"
                h[:, 8:12:2] = (lo if dense else lo + gap).astype(F32)      # background
                h[:, 9:12:2] = (lo + gap if dense else lo).astype(F32)      # face
            else:
                h[:, 0:4] = rng.uniform(0.5, 1.0, (B, 4, g)) if values == "dense" else rng.uniform(0.0, 0.49, (B, 4, g))
                h[:, 32:38] = rng.uniform(0.0, 1.0, (B, 6, g))
            heads.append(h)
    if values == "nonfinite":
        sp = SPECIALS[variant]
        for h in heads:
            g = h.shape[2]
            for b in range(B):
                cells = rng.permutation(g)[:len(sp)]
                for j, cell in enumerate(cells):
                    k = int(rng.integers(0, 2))
                    for (grp, i), val in sp[(j + b) % len(sp)].items():
                        h[b, _channel(variant, grp, i, k), cell] = val
    if half:
        with np.errstate(over="ignore"):
            heads = [h.astype(np.float16).astype(F32) for h in heads]
    if variant == FACE:
        _resample_gate_band(heads, rng, GATE, half)
    return [np.ascontiguousarray(h) for h in heads]


def gate_heads(variant, in_h, in_w, B, seed, half=False):
    """RetinaFace: a third of the priors with equal logits (p = 0.5 exactly), a third clearly kept, a third clearly dropped
    at any gate near 0.5.  AntiCov: face probabilities 0.5, nextafter(0.5, 0) and clear ones."""
    rng = np.random.default_rng(seed)
    heads = []
    for _, _, g in grids(in_h, in_w):
        h = rng.standard_normal((B, CHANNELS[variant], g), dtype=np.float32)
        pick = rng.integers(0, 3, (B, 2, g))
        if variant == FACE:
            c1 = rng.uniform(-5, 5, (B, 2, g)).astype(F32)
            if half:
                c1 = c1.astype(np.float16).astype(F32)
            c2 = np.where(pick == 0, c1, np.where(pick == 1, c1 + F32(3), c1 - F32(3)))
            h[:, 8:12:2], h[:, 9:12:2] = c1, c2
        else:
            t = np.float16 if half else F32
            below = F32(np.nextafter(t(0.5), t(0)))
            v = np.where(pick == 0, F32(0.5), np.where(pick == 1, below, F32(0.75)))
            h[:, 2:4] = v
            h[:, 0:2] = rng.uniform(0, 1, (B, 2, g))
        heads.append(h.astype(np.float16).astype(F32) if half else h)
    return heads


# ---------------------------------------------------------------------------------------------------------------------
# GPU case list (tests/test_retina_decode_paths_gpu.py): (variant, dtype, shape, batch, values)
# ---------------------------------------------------------------------------------------------------------------------
def gpu_cases():
    cases = []
    for variant in (FACE, ANTICOV):
        for dtype in ("f32", "f16"):
            for shape in SHAPES:
                bs = batches(shape)
                for B in bs:
                    cases.append((variant, dtype, shape, B, "sparse"))
                for values in ("dense", "empty", "nonfinite"):
                    cases.append((variant, dtype, shape, min(3, bs[-1]), values))
    return cases


def case_id(c):
    variant, dtype, shape, B, values = c
    return f"{VARIANTS[variant]}-{dtype}-{shape_id(shape)}-b{B}-{values}"


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_decode(oracle, heads, variant, in_h, in_w):
    if variant == FACE:
        return oracle.retina_decode(heads, in_h=in_h, in_w=in_w, gate=0.02)[0]
    return oracle.anticov_decode(heads, in_h=in_h, in_w=in_w)[0]


@pytest.mark.parametrize("values", ["sparse", "dense", "nonfinite"])
@pytest.mark.parametrize("shape", SHAPES, ids=shape_id)
@pytest.mark.parametrize("variant", [FACE, ANTICOV], ids=VARIANTS.get)
def test_oracle_within_the_bound(oracle, variant, shape, values):
    """oracle_retina_decode / oracle_anticov_decode (plain C, no FMA, glibc expf) lie within the float64 bound"""
    in_h, in_w = shape
    B = 1 if in_h * in_w > 1080 * 1920 else 2
    for half in (False, True):
        heads = make_heads(variant, in_h, in_w, B, values, seed=in_h + in_w + 7 * len(values), half=half)
        ref = reference(heads, variant, in_h, in_w)
        assert ref.counts.sum() > 0
        if values == "dense":
            assert (ref.counts == total_priors(in_h, in_w)).all()
        assert_matches(_oracle_decode(oracle, heads, variant, in_h, in_w), ref, variant, f"{shape} half={half}")


@pytest.mark.parametrize("variant", [FACE, ANTICOV], ids=VARIANTS.get)
def test_empty_heads_keep_nothing(oracle, variant):
    for shape in SHAPES[:7]:
        heads = make_heads(variant, *shape, 2, "empty", seed=3)
        ref = reference(heads, variant, *shape)
        assert (ref.counts == 0).all()
        assert_matches(_oracle_decode(oracle, heads, variant, *shape), ref, variant)


def test_nonfinite_heads_reach_every_special_kind():
    """the 'nonfinite' class really keeps NaN conf, NaN / +-inf boxes and landmarks, and drops -inf / 0-probability priors"""
    for variant in (FACE, ANTICOV):
        heads = make_heads(variant, 64, 64, 3, "nonfinite", seed=1)
        ref = reference(heads, variant, 64, 64)
        rows = np.concatenate(ref.rows)
        assert np.isnan(rows[:, 4]).any()
        assert np.isposinf(rows[:, :4]).any() and np.isneginf(rows[:, :4]).any() and np.isnan(rows[:, :4]).any()
        assert np.isinf(rows[:, 5:15]).any() and np.isnan(rows[:, 5:15]).any()
        if variant == ANTICOV:
            assert np.isnan(rows[:, 15]).any() and np.isinf(rows[:, 4]).any()


@pytest.mark.parametrize("variant", [FACE, ANTICOV], ids=VARIANTS.get)
def test_gate_boundary(oracle, variant):
    """RetinaFace: equal logits give p = 0.5 exactly, dropped at gate 0.5 and kept at nextafter(0.5, 0); AntiCov keeps a
    probability of exactly 0.5 and drops nextafter(0.5, 0)"""
    heads = gate_heads(variant, 64, 64, 2, seed=5)
    g1 = float(np.nextafter(F32(0.5), F32(0)))
    if variant == FACE:
        at, below = reference(heads, FACE, 64, 64, gate=0.5), reference(heads, FACE, 64, 64, gate=g1)
        equal = sum(int(((h[:, 8:12:2] == h[:, 9:12:2])).sum()) for h in heads)
        assert equal > 100 and below.counts.sum() - at.counts.sum() == equal
    else:
        ref = reference(heads, ANTICOV, 64, 64)
        n05 = sum(int((h[:, 2:4] == F32(0.5)).sum()) for h in heads)
        n75 = sum(int((h[:, 2:4] == F32(0.75)).sum()) for h in heads)
        assert n05 > 100 and ref.counts.sum() == n05 + n75
        assert_matches(_oracle_decode(oracle, heads, ANTICOV, 64, 64), ref, ANTICOV)


# the shape classes where each defect changes the decode of sparse heads (the gate defect only changes priors at the gate)
CHANGES = {"no_half": set(SHAPES), "anchor_k": set(SHAPES), "lmk_scale": set(SHAPES), "half_width": set(SHAPES),
           "swap_wh": {s for s in SHAPES if s[0] != s[1]}, "step_from_width": {(640, 660), (640, 40)},
           "gate_strictness": set()}


@pytest.mark.parametrize("variant,defect", [(v, d) for v in (FACE, ANTICOV) for d in DEFECTS[v]],
                         ids=[f"{VARIANTS[v]}-{d}" for v in (FACE, ANTICOV) for d in DEFECTS[v]])
def test_injected_defects_fail(variant, defect):
    """each defect changes the decode exactly on the classes of CHANGES; where it does, it moves some value by more than
    1000x its bound (or changes the kept set), and assert_matches rejects it"""
    changed = set()
    for shape in SHAPES:
        heads = make_heads(variant, *shape, 1, "sparse", seed=11)
        ref = reference(heads, variant, *shape)
        bad = reference(heads, variant, *shape, defect=defect)
        if same(bad, ref):
            continue
        changed.add(shape)
        ratio = defect_ratio(bad, ref)
        assert ratio is None or ratio >= 1000, (shape, ratio)
        with pytest.raises(AssertionError):
            assert_matches(as_output(bad, variant, *shape), ref, variant)
    assert changed == CHANGES[defect], sorted(changed ^ CHANGES[defect])
    if defect == "gate_strictness":
        heads = gate_heads(variant, 64, 64, 1, seed=2)
        gate = 0.5 if variant == FACE else GATE
        ref, bad = reference(heads, variant, 64, 64, gate=gate), reference(heads, variant, 64, 64, gate=gate, defect=defect)
        assert defect_ratio(bad, ref) is None
        with pytest.raises(AssertionError):
            assert_matches(as_output(bad, variant, 64, 64), ref, variant)


def test_reference_rows_pass_their_own_comparison():
    """rounding the float64 rows to fp32 stays within the bound: the comparison does not reject a correct decode"""
    for variant in (FACE, ANTICOV):
        for shape in ((640, 660), (32, 32)):
            heads = make_heads(variant, *shape, 2, "nonfinite", seed=4)
            ref = reference(heads, variant, *shape)
            assert_matches(as_output(ref, variant, *shape), ref, variant)


def test_priors_follow_the_reference_expressions():
    """spot values: RetinaFace centres (x + 0.5) / w and sizes anchor * (k + 1) / in_w in fp32; AntiCov centres on the
    fixed stride and integer sizes 32 / 16, 128 / 64, 512 / 256"""
    p0, p1, p2, p3 = priors(FACE, 480, 640)
    assert p0[0] == F32(0.5 / 80) and p1[0] == F32(0.5 / 60) and p2[1] == F32(32) / F32(640) and p3[1] == F32(32) / F32(480)
    p0, p1, p2, _ = priors(ANTICOV, 640, 660)
    g0, g1 = 80 * 82, 40 * 41
    last = 2 * (g0 + g1) + 2 * (20 * 20 - 1)       # level 2, cell (19, 19), k = 0
    assert p0[last] == 7.5 + 19 * 32 and p1[last] == 7.5 + 19 * 32
    assert priors(ANTICOV, 640, 660, "step_from_width")[0][last] == 7.5 + 19 * 33
    assert p2[[0, 1, 2 * g0, 2 * g0 + 1, last, last + 1]].tolist() == [32, 16, 128, 64, 512, 256]


def test_dispatch_mirror_matches_the_library():
    """the mirror's workspace size and prior count are the library's; 4480x4480 takes 3 217 tiles per image at VEC=4 and
    12 863 at VEC=1, whose prefix (51 456 B) is past 48 KB and takes 13 pack passes"""
    from tensorrtx_b200 import _lib as L
    lib = L.load()
    for shape in SHAPES:
        for B in batches(shape):
            p = L.RetinaParams(in_h=shape[0], in_w=shape[1])
            d = dispatch(FACE, "f32", *shape, B)
            assert lib.trtx_retina_workspace_size(C.byref(p), B) == d["workspace_size"] >= d["workspace"]
            assert lib.trtx_retina_total_priors(C.byref(p)) == total_priors(*shape)
    a, o = dispatch(FACE, "f32", 4480, 4480, 1), dispatch(FACE, "f32", 4480, 4480, 1, addr_mod=(4, 4, 4))
    assert (a["vec"], a["tiles"], a["pack_passes"]) == (4, 3217, 4)
    assert (o["vec"], o["tiles"], o["pack_passes"]) == (1, 12863, 13) and 4 * (o["tiles"] + 1) == 51456 > 48 * 1024
    assert dispatch(FACE, "f16", 640, 640, 1, addr_mod=(8, 0, 0))["vec"] == 4
    assert dispatch(FACE, "f16", 640, 640, 1, addr_mod=(0, 2, 0))["vec"] == 1
    assert dispatch(ANTICOV, "f32", 640, 640, 16)["tiles"] == 67


def test_gpu_cases_reach_every_scan_instantiation():
    """the GPU case list runs every one of the eight scans: aligned heads take VEC=4 where every grid is a multiple of 4
    cells, and every case runs again on heads one element off alignment (VEC=1)"""
    reached = set()
    for variant, dtype, shape, B, _ in gpu_cases():
        es = DTYPE_SIZE[dtype]
        reached.add(dispatch(variant, dtype, *shape, B)["kernel"])
        reached.add(dispatch(variant, dtype, *shape, B, addr_mod=(es, es, es))["kernel"])
    want = {f"{KERNEL[v]}<{t}, {vec}>" for v in (FACE, ANTICOV) for t in DTYPE_T.values() for vec in (1, 4)}
    assert reached == want
    # and the aligned runs alone reach VEC=1 (488x648, 640x40 ... ) as well as VEC=4
    aligned = {dispatch(v, d, *s, B)["vec"] for v, d, s, B, _ in gpu_cases()}
    assert aligned == {1, 4}
