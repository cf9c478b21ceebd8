"""Inputs of the RefineDet post-process path tests, shared by tests/test_refinedet_paths_gpu.py (the kernel against the
reference's arithmetic) and tests/test_refinedet_paths_cpu.py (the oracle against the transcription, and the geometry each
case claims in NumPy float64), so that both pin the same cases.

TEST INFRASTRUCTURE ONLY.  Every builder returns a Case: heads [B, P, 4], [B, P, 2], [B, P, 4], [B, P, C] float32, the
post-process keywords, the frame sizes (or None) and whether scores tie (then only the oracle's tie rule decides the
order).  Crafted geometry uses zero arm_loc and odm_loc: a decoded box is then its prior's corners exactly (exp(0) = 1 and
every product with a zero offset is +0), so `boxes` below is the box the reference and the library compute."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import refinedet as RO

F32 = np.float32
V0, V1 = float(F32(0.1)), float(F32(0.2))
SIDES = tuple(range(64, 1025, 64))                      # every side the library accepts: P = 255 .. 65280
TOP_KS = (1, 2, 63, 64, 65, 128, 129, 1000, 1023, 1024)  # mask of 1 word .. 16 words
SIDE_CLASSES = (2, 21, 25, 81)
HUGE = 1e20                                             # centre offset of the identical boxes (see `edges`)


@dataclass
class Case:
    h: list
    kw: dict
    sizes: list | None = None
    ties: bool = False
    claims: dict = field(default_factory=dict)  # class -> kept count the geometry promises (nms_thresh 0.45)


# ------------------------------------------------------------------ geometry ------------------------------------------
def levels(net: int):
    """[(first prior, cells a side)] of the four levels."""
    out, off = [], 0
    for k in range(4):
        f = net >> (3 + k)
        out.append((off, f))
        off += 3 * f * f
    return out


def prior_index(net: int, k: int, i: int, j: int, a: int = 0) -> int:
    off, f = levels(net)[k]
    return off + (i * f + j) * 3 + a


def decode(prior, arm_loc, odm_loc):
    """The two decode steps in float64, op by op as the reference: prior [n, 4], offsets [n, 4] float32 -> corners [n, 4].
    NumPy's exp; with zero offsets (exp(0) = 1) the result is the reference's on any device."""
    al, ol = np.asarray(arm_loc, np.float64), np.asarray(odm_loc, np.float64)
    with np.errstate(all="ignore"):
        d01 = prior[:, :2] + (al[:, :2] * V0) * prior[:, 2:]
        d23 = prior[:, 2:] * np.exp(al[:, 2:] * V1)
        c = d01 + (ol[:, :2] * V0) * d23
        s = d23 * np.exp(ol[:, 2:] * V1)
        x1 = c - s / 2
        return np.concatenate([x1, x1 + s], 1)


def boxes(net: int) -> np.ndarray:
    """Every prior's decoded box under zero offsets [P, 4]."""
    pr = RO.priors(net)
    z = np.zeros((len(pr), 4), F32)
    return decode(pr, z, z)


def iou(bi, bj, round_i: bool = True):
    """nms()'s IoU of box i [4] against boxes j [n, 4]: j's corners clamped by i's (rounded to float, as
    `x1[i].item().toFloat()`, when round_i) as Tensor::clamp does (a NaN on either side gives NaN), inter * 1.0 /
    ((area_j - inter) + area_i) with unrounded areas."""
    bi, bj = np.asarray(bi, np.float64), np.atleast_2d(np.asarray(bj, np.float64))
    lo = bi.astype(F32).astype(np.float64) if round_i else bi
    with np.errstate(all="ignore"):
        xx1 = np.minimum(np.maximum(bj[:, 0], lo[0]), RO.INT_MAX * 1.0)
        yy1 = np.minimum(np.maximum(bj[:, 1], lo[1]), RO.INT_MAX * 1.0)
        xx2 = np.minimum(np.maximum(bj[:, 2], RO.INT_MIN * 1.0), lo[2])
        yy2 = np.minimum(np.maximum(bj[:, 3], RO.INT_MIN * 1.0), lo[3])
        w = np.minimum(np.maximum(xx2 - xx1, 0.0), RO.INT_MAX * 1.0)
        h = np.minimum(np.maximum(yy2 - yy1, 0.0), RO.INT_MAX * 1.0)
        inter = w * h
        area_i = (bi[2] - bi[0]) * (bi[3] - bi[1])
        area_j = (bj[:, 2] - bj[:, 0]) * (bj[:, 3] - bj[:, 1])
        return inter * 1.0 / ((area_j - inter) + area_i)


def nms_keep(b, thresh: float, round_i: bool = True) -> list:
    """Greedy NMS over boxes [m, 4] already in score order -> kept positions (j dropped where !(IoU < thresh))."""
    removed = np.zeros(len(b), bool)
    keep = []
    for i in range(len(b)):
        if removed[i]:
            continue
        keep.append(i)
        removed[i + 1:] |= ~(iou(b[i], b[i + 1:], round_i) < np.float64(F32(thresh)))
    return keep


def disjoint_squares(net: int) -> list:
    """Level-0 square anchors four cells apart (a square anchor spans four cells): pairwise disjoint, (f / 4)^2 of them."""
    f = net >> 3
    return [prior_index(net, 0, i, j) for i in range(0, f, 4) for j in range(0, f, 4)]


def chain(net: int, rows) -> list:
    """Level-0 square anchors along whole rows of cells: neighbours overlap 3/5, next-but-one neighbours 1/3."""
    f = net >> 3
    return [prior_index(net, 0, i, j) for i in rows for j in range(f)]


def ramp(n: int, lo: float = 0.02, hi: float = 0.99) -> np.ndarray:
    """n distinct descending float32 scores in [lo, hi]."""
    v = np.linspace(hi, lo, n, dtype=F32)
    assert len(np.unique(v)) == n
    return v


def blank(B: int, net: int, C: int):
    """Zero offsets, objectness 0.5 everywhere (kept by obj_thresh 0.01), all scores 0."""
    P = RO.num_priors(net)
    return [np.zeros((B, P, 4), F32), np.full((B, P, 2), 0.5, F32), np.zeros((B, P, 4), F32), np.zeros((B, P, C), F32)]


def frame_sizes(B: int) -> list:
    return [(64 + 29 * b, 48 + 17 * b) for b in range(B)]


# ------------------------------------------------------------------ cases --------------------------------------------
def side(net: int) -> Case:
    """Seeded tie-free heads at one side with random offsets: every level's first and last three priors (the level
    search's edges) are candidates of every class, and at S = 1024 every seventh prior from 65024 on (the top of the
    uint16 range); classes 1 and 2 hold more than top_k candidates.  C and top_k cycle over SIDE_CLASSES and TOP_KS."""
    n = SIDES.index(net)
    C, K, P = SIDE_CLASSES[n % len(SIDE_CLASSES)], TOP_KS[n % len(TOP_KS)], RO.num_priors(net)
    always = {q for off, f in levels(net) for q in (off, off + 1, off + 2, off + 3 * f * f - 3, off + 3 * f * f - 2,
                                                     off + 3 * f * f - 1)}
    if net == 1024:
        always |= set(range(65024, P, 7))
    h = list(RO.heads(2, net, C, seed=net, objects=40 if C == 2 else 8, dense=min(P // 2, K + 40), always=sorted(always)))
    return Case(h, {"net": net, "top_k": K}, frame_sizes(2))


def cut(K: int) -> Case:
    """S = 1024, C = 7: class c holds 0, 1, K - 1, K, K + 1 and K + 8000 candidates.  The K best of each are pairwise
    disjoint squares (all kept), the rest score lower, anywhere; so the kept count is min(n, K) and the select's cut (from
    K + 1 on) decides which box is last."""
    net, C = 1024, 7
    h = blank(1, net, C)
    P = RO.num_priors(net)
    rng = np.random.default_rng(K)
    sq = np.array(disjoint_squares(net))
    others = np.setdiff1d(np.arange(P), sq)
    claims = {}
    for c, n in zip(range(1, C), (0, 1, K - 1, K, K + 1, K + 8000)):
        top = min(n, len(sq))
        ids = np.concatenate([rng.permutation(sq)[:top], rng.choice(others, n - top, replace=False)]).astype(int)
        h[3][0, ids, c] = ramp(n) if n else []
        claims[c] = min(n, K)
    return Case(h, {"net": net, "top_k": K}, frame_sizes(1), claims=claims)


def edges(nms_thresh: float) -> Case:
    """S = 1024, top_k 1024, C = 5, zero offsets except where noted; the classes use disjoint sets of priors:
      1  a chain along level-0 rows 0, 64 and 127 (128 cells each), scores descending along the rows: the kept set
         alternates, and the 384 sorted boxes cross mask words 64 .. 320;
      2  1500 identical boxes: level-0 wide anchors whose ARM centre offset (1e20) swamps the prior's centre (below half
         an ulp of the sum) and whose ODM offset (-1e20) takes the same amount back, so every box is (-w/2, -h/2, w/2,
         h/2) of the same anchor size; exactly one is kept, at nms_thresh 1 too (IoU 1);
      3  256 level-1 squares with random offsets, one in four with a NaN in one of them (NaN corners, NaN IoUs);
      4  192 level-2 anchors, four in five of zero width, height or both (exp(-inf) = 0): 0 / 0 IoUs between them."""
    net, C = 1024, 5
    h = blank(1, net, C)
    rng = np.random.default_rng(17)
    ids = chain(net, (0, 64, 127))
    h[3][0, ids, 1] = ramp(len(ids))
    f0 = net >> 3
    wide = np.array([prior_index(net, 0, i, j, 1) for i in range(f0) for j in range(f0)])
    ids = rng.choice(wide, 1500, replace=False)
    h[0][0, ids, :2] = HUGE
    h[2][0, ids, :2] = -HUGE
    h[3][0, ids, 2] = rng.permutation(ramp(len(ids)))
    ids = np.array([prior_index(net, 1, i, j) for i in range(10, 26) for j in range(10, 26)])
    h[0][0, ids] = rng.normal(0, 0.3, (len(ids), 4))
    h[2][0, ids] = rng.normal(0, 0.3, (len(ids), 4))
    nan = ids[rng.permutation(len(ids))[:len(ids) // 4]]
    h[0][0, nan[::2], rng.integers(0, 4, len(nan[::2]))] = np.nan
    h[2][0, nan[1::2], rng.integers(0, 4, len(nan[1::2]))] = np.nan
    h[3][0, ids, 3] = rng.permutation(ramp(len(ids)))
    ids = np.array([prior_index(net, 2, i, j, a) for i in range(4, 12) for j in range(4, 12) for a in range(3)])
    for r, (t, e) in enumerate(((0, 2), (0, 3), (0, None), (2, 2), (None, None))):
        sel = ids[r::5]
        if t is not None and e is not None:
            h[t][0, sel, e] = -np.inf
        elif t is not None:
            h[t][0, sel, 2:] = -np.inf
    h[3][0, ids, 4] = rng.permutation(ramp(len(ids)))
    return Case(h, {"net": net, "top_k": 1024, "nms_thresh": nms_thresh}, frame_sizes(1), claims={1: 192, 2: 1})


def pair_search(net: int = 320, n: int = 600):
    """Among the zero-offset boxes of the first n priors at `net`, the first pair (i, j), in index order, whose IoU (i
    rounded) lies in (0.3, 0.7) and is not a float; and the first pair where some float t lies between the IoU with i
    rounded and the IoU without, so that rounding i decides `IoU < t` -> ((i, j, iou), (i, j, t))."""
    b = boxes(net)[:n]
    straddle = flip = None
    for i in range(n):
        r, u = iou(b[i], b), iou(b[i], b, round_i=False)
        for j in np.flatnonzero((r > 0.3) & (r < 0.7)):
            if j == i:
                continue
            if straddle is None and float(F32(r[j])) != r[j]:
                straddle = (i, int(j), float(r[j]))
            lo, hi = min(r[j], u[j]), max(r[j], u[j])
            t = F32(lo) if float(F32(lo)) > lo else np.nextafter(F32(lo), F32(1))
            if flip is None and float(t) <= hi and (r[j] < t) != (u[j] < t):
                flip = (i, int(j), float(t))
        if straddle and flip:
            return straddle, flip
    raise AssertionError("no pair found")


def pair(i: int, j: int, nms_thresh: float, net: int = 320) -> Case:
    """Priors i (score 0.9) and j (0.8) the only candidates, zero offsets."""
    h = blank(1, net, 2)
    h[3][0, i, 1], h[3][0, j, 1] = 0.9, 0.8
    return Case(h, {"net": net, "top_k": 2, "nms_thresh": nms_thresh}, frame_sizes(1))


def frames(B: int) -> Case:
    """S = 64, C = 2 (one class), top_k 63, obj_thresh 0.5, B frames of distinct sizes.  Per frame: random offsets, 60
    candidates with distinct scores, one at exactly score_thresh 0.2f and one a float either side of it, one +inf score
    (ranked first), NaN scores (never candidates) and NaN offsets; with B >= 3 frame 1 has every objectness <= obj_thresh
    (0.5 itself included): an empty frame between two others."""
    net, K = 64, 63
    P = RO.num_priors(net)
    rng = np.random.default_rng(1000 + B)
    arm_loc = rng.normal(0, 0.4, (B, P, 4)).astype(F32)
    odm_loc = rng.normal(0, 0.4, (B, P, 4)).astype(F32)
    arm_conf = np.zeros((B, P, 2), F32)
    arm_conf[..., 1] = rng.uniform(0, 1, (B, P))
    odm_conf = np.zeros((B, P, 2), F32)
    th = F32(0.2)
    special = np.array([th, np.nextafter(th, F32(0)), np.nextafter(th, F32(1)), np.inf], F32)
    for b in range(B):
        ids = rng.choice(P, 70, replace=False)
        vals = ramp(60, 0.05, 0.95)
        vals = vals[~np.isin(vals, special)][:56]
        odm_conf[b, ids[:56], 1] = rng.permutation(vals)
        odm_conf[b, ids[56:60], 1] = special
        arm_conf[b, ids[56:60], 1] = 0.9
        odm_conf[b, ids[60:64], 1] = np.nan
        arm_conf[b, ids[62:64], 1] = 0.9
        arm_loc[b, ids[64], 0] = np.nan
        odm_loc[b, ids[65], 3] = np.nan
    if B >= 3:
        arm_conf[1, :, 1] = rng.uniform(0, 0.5, P)
        arm_conf[1, ::7, 1] = 0.5
    arm_conf[..., 0] = 1 - arm_conf[..., 1]
    return Case([arm_loc, arm_conf, odm_loc, odm_conf], {"net": net, "top_k": K, "obj_thresh": 0.5}, frame_sizes(B))


def many_classes(net: int) -> Case:
    """C = 1024 at S = 64 or 128, top_k 2 (so most classes are cut by the select), two frames: class c holds c % 5
    candidates with random offsets and distinct scores across the whole range, so rows fail `score < TH` in every pass of
    512 rows and the frames total well above 1025 rows."""
    C, B = 1024, 2
    P = RO.num_priors(net)
    rng = np.random.default_rng(net)
    arm_loc = rng.normal(0, 0.5, (B, P, 4)).astype(F32)
    odm_loc = rng.normal(0, 0.5, (B, P, 4)).astype(F32)
    arm_conf = np.zeros((B, P, 2), F32)
    arm_conf[..., 1] = rng.uniform(0.02, 1, (B, P))
    arm_conf[..., 0] = 1 - arm_conf[..., 1]
    odm_conf = rng.uniform(0, 0.009, (B, P, C)).astype(F32)
    for b in range(B):
        for c in range(1, C):
            n = c % 5
            vals = rng.uniform(0.0101, 0.99, n).astype(F32)
            assert len(np.unique(vals)) == n
            odm_conf[b, rng.choice(P, n, replace=False), c] = vals
    return Case([arm_loc, arm_conf, odm_loc, odm_conf], {"net": net, "top_k": 2}, [(1920, 1080), (333, 777)])


def negative_conf() -> Case:
    """S = 1024, C = 3, top_k 1024, conf_thresh -0.5: every prior is a candidate of every class.  Half the priors fail
    the ARM filter (their scores become +-0); class 1 has 200 distinct positive scores over raw scores of +0, -0 and
    -0.001, class 2 only +0 and -0: the cut falls inside a tie of +-0 across all P.  Scores tie, so the order is the
    library's tie rule."""
    net, C = 1024, 3
    h = blank(1, net, C)
    P = RO.num_priors(net)
    rng = np.random.default_rng(5)
    h[1][0, :, 1] = np.where(rng.random(P) < 0.5, F32(0.005), F32(0.5))
    h[3][0, :, 1] = rng.choice(np.array([0.0, -0.0, -0.001], F32), P)
    h[3][0, rng.choice(P, 200, replace=False), 1] = ramp(200, 0.05, 0.95)
    h[3][0, :, 2] = rng.choice(np.array([0.0, -0.0], F32), P)
    return Case(h, {"net": net, "top_k": 1024, "conf_thresh": -0.5}, frame_sizes(1), ties=True)
