"""The YOLO instance-mask kernels (tensorrtx_b200/csrc/mask.cu) in float64, on every shape class the GPU tests run.

process_mask of the segmentation drivers is
    m[y, x] = sigmoid(sum_j c_j * p_j[y, x])   for (x, y) in get_downscale_rect(bbox, 4), 0 elsewhere    (mh x mw cells)
    M       = cv::resize(m, net_w x net_h, INTER_LINEAR)
scale_mask crops M to the letterboxed frame and resizes it to the frame the same way, and the segmentation post-process keeps
the pixels of get_rect(img, bbox) where !(S <= 0.5).  The float64 reference has three parts:
  * the rectangle: get_downscale_rect in fp32, as each variant spells it (V8 reads l, t, r, b as x, y, w, h and truncates,
    V5 takes cx, cy, w, h and rounds).  It is discrete, so it is computed exactly as defined.  Where one of its four
    float -> int conversions is undefined (NaN, +-inf, past the int range) the mask is all zeros -- the library's rule;
  * the cells: sigmoid(sum c_j p_j) in float64;
  * OpenCV's bilinear taps (`fx = (float)((d + 0.5) * scale - 0.5)`, floor, clamp to the border with a zero fraction),
    discrete again and kept exactly, and the two blends in float64 with those fp32 weights (`1.0f - fx`, `fx`).

Error bound of one pixel, from the fp32 arithmetic of the kernels (u = 2^-24):
  * a cell: the dot product `e += c_j * p_j` in order, one rounding per product and per sum, is off by at most
    gamma_nm * S with S = sum_j |c_j p_j| and gamma_n = n u / (1 - n u); sigmoid' <= 1/4, so that moves the cell by
    1/4 gamma_nm S.  expf (<= 2 ulp in CUDA, 1 in glibc: a relative 4u on exp(-e)) moves sigmoid by at most
    sigma (1 - sigma) 4u <= u; the sum 1 + E and the division by one rounding each, u each.  Cell bound: 1/4 gamma_nm S + 3u;
    cells outside the rectangle are exact zeros on both sides;
  * a blend reads four cells with weights of sum <= 1 + 2u and rounds six times (four products, two sums) values <= 1 + 2u:
    pixel bound = (1 + 4u) * max over the four cells it reads of their bound + 6u.
scale_mask applies the same blend to M, so its bound is the same expression over the bounds of the four M pixels it reads.
The tests below check the reference against the CPU oracle (the fp32 expressions of the reference drivers) within that
bound, that the bound is far below the error of one wrong tap, and that each of four injected defects fails the comparison
on every shape class.  tests/test_mask_paths_gpu.py holds the kernels to the same reference."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import pytest

F32 = np.float32
U = 2.0 ** -24
V8, V5 = 0, 1
DEFECTS = ("tap", "v5_trunc", "halo", "threshold")


def gamma(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------------------------
# shape classes: the nets, coefficient counts and row layouts both entries accept
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Shape:
    net_w: int
    net_h: int
    nm: int = 32
    layout: str = "r39o7"   # r39o7: the NMS output's (39, 7); r38o6: (38, 6); end: the block ends a longer row

    @property
    def mw(self):
        return self.net_w // 4

    @property
    def mh(self):
        return self.net_h // 4

    @property
    def row(self):
        """(row_floats, coeff_offset), the row widened where nm coefficients need it"""
        if self.layout == "r39o7":
            return max(39, 7 + self.nm), 7
        if self.layout == "r38o6":
            return max(38, 6 + self.nm), 6
        return 18 + self.nm, 18

    @property
    def id(self):
        R, off = self.row
        return f"net{self.net_w}x{self.net_h}-nm{self.nm}-r{R}o{off}"


NETS = [(640, 640), (640, 480), (544, 544), (1280, 1280), (64, 64), (1024, 256)]
NET_SHAPES = [Shape(w, h) for w, h in NETS]
# 640 x 480: tiles partial on one axis.  Every coefficient count with every row layout; (32, r39o7) is a net class already
ROW_SHAPES = [Shape(640, 480, nm, layout) for nm in (1, 32, 64) for layout in ("r39o7", "r38o6", "end")
              if (nm, layout) != (32, "r39o7")]
SHAPES = NET_SHAPES + ROW_SHAPES
# non-finite and out-of-range coordinates: 3e9 is past 2^31 but 7.5e8 cells; 1e10 is past it in cells as well
BAD_VALUES = [np.nan, np.inf, -np.inf, 3e9, -3e9, 1e10, -1e10]


# ---------------------------------------------------------------------------------------------------------------------
# the boxes
# ---------------------------------------------------------------------------------------------------------------------
def _as_variant(variant, x, y, w, h):
    """A box covering net pixels [x, x + w) x [y, y + h), in the variant's process_mask format."""
    if variant == V8:
        return [x, y, w, h]
    return [x + w / 2, y + h / 2, w, h]


def edge_boxes(variant, net_w, net_h):
    """Boxes on 16-cell tile edges and one cell either side, 0 and 1 cell wide, the whole mask, half outside, and (V5)
    centres and sizes at exact .5 cells."""
    mw, mh = net_w // 4, net_h // 4
    out = []
    ex = sorted({c for k in range(0, mw // 16 + 1) for c in (16 * k - 1, 16 * k, 16 * k + 1) if 0 <= c <= mw})
    ey = sorted({c for k in range(0, mh // 16 + 1) for c in (16 * k - 1, 16 * k, 16 * k + 1) if 0 <= c <= mh})
    # pairs of tile-edge cells as the rectangle's first and last cell: start on an edge, end on one (the first 12 and the
    # last 4 starts)
    for i, a in enumerate(ex[:-1]):
        if 12 <= i < len(ex) - 5:
            continue
        b = ex[min(len(ex) - 1, i + 3)]
        ya, yb = ey[i % max(1, len(ey) - 1)], ey[min(len(ey) - 1, i % max(1, len(ey) - 1) + 2)]
        out.append(_as_variant(variant, 4 * a, 4 * ya, 4 * (b - a), 4 * max(yb - ya, 1)))
    cx, cy = 4 * (mw // 2), 4 * (mh // 2)
    out += [_as_variant(variant, cx, cy, 0, 40), _as_variant(variant, cx, cy, 4, 40),        # 0 and 1 cell wide
            _as_variant(variant, cx, cy, 40, 0), _as_variant(variant, cx, cy, 40, 4),        # 0 and 1 cell high
            _as_variant(variant, cx, cy, 2, 2),                                             # under one cell
            _as_variant(variant, 0, 0, net_w, net_h),                                       # the whole mask
            _as_variant(variant, -20, -12, net_w + 40, net_h + 24),                         # more than the mask
            _as_variant(variant, -net_w / 4, cy / 2, net_w / 2, net_h / 3),                 # half outside, each side
            _as_variant(variant, 3 * net_w / 4, cy / 2, net_w / 2, net_h / 3),
            _as_variant(variant, cx / 2, -net_h / 4, net_w / 3, net_h / 2),
            _as_variant(variant, cx / 2, 3 * net_h / 4, net_w / 3, net_h / 2),
            _as_variant(variant, net_w + 8, 8, 40, 40), _as_variant(variant, 8, -80, 40, 40)]  # wholly outside
    if variant == V5:
        # left / 4, top / 4 at k + .5 (round() away from zero), and a width of j + .5 cells
        for k in (0, 1, mw // 2 - 1, mw - 2):
            out.append([4 * k + 2 + 4, 4 * (k % mh) + 2 + 4, 8, 8])   # left = 4k + 2: k + .5 cells
            out.append([4 * k + 2 + 5, 4 * (k % mh) + 6, 10, 10])      # width 2.5 cells
        out.append([2.0, 2.0, 12.0, 12.0])                            # left = -4: -1 cell; top / 4 = -.5 -> -1
    return out


def undefined_boxes(variant, net_w, net_h):
    """A finite box with one coordinate replaced by NaN, +-inf or a value past 2^31, for every coordinate; and (V5) a box
    whose left is defined but whose width in cells is past INT_MAX; and boxes whose four conversions are defined but whose
    right (bottom) end in cells lies far below 0 (V5: below INT_MIN)."""
    base = _as_variant(variant, net_w / 4, net_h / 4, net_w / 3, net_h / 3)
    out = []
    for c in range(4):
        for v in BAD_VALUES:
            b = list(base)
            b[c] = v
            out.append(b)
    if variant == V5:
        out.append([1e9, net_h / 2, 1e10, 100.0])
        # every conversion defined, but rx + rw (ry + rh) about -4e9: below INT_MIN, so the 64-bit end must not wrap
        out += [[-1.2e10, net_h / 2, -8e9, 100.0], [net_w / 2, -1.2e10, 100.0, -8e9]]
    else:
        out += [[0.0, 5.0, -8e9, 50.0], [5.0, 0.0, 50.0, -8e9]]   # rw (rh) about -2e9, defined
    return out


def random_boxes(rng, variant, net_w, net_h, n):
    out = []
    for _ in range(n):
        x, y = rng.uniform(-0.1 * net_w, 0.9 * net_w), rng.uniform(-0.1 * net_h, 0.9 * net_h)
        w, h = rng.uniform(2, 0.6 * net_w), rng.uniform(2, 0.6 * net_h)
        out.append(_as_variant(variant, x, y, w, h))
    return out


def make_dets(rng, shape, boxes, pad_rows=0):
    """One image's dets [1 + K * R]: count = len(boxes), each row box, conf, class, nm coefficients at the offset."""
    R, off = shape.row
    K = len(boxes) + pad_rows
    d = np.zeros(1 + K * R, F32)
    d[0] = len(boxes)
    rows = d[1:].reshape(K, R)
    scale = 2.0 if shape.nm == 1 else 0.6
    for i, b in enumerate(boxes):
        rows[i, :4] = np.asarray(b, np.float64).astype(F32)
        rows[i, 4:6] = [rng.uniform(0.3, 1.0), rng.integers(0, 80)]
        rows[i, off:off + shape.nm] = rng.standard_normal(shape.nm) * scale
    return d


def make_proto(rng, shape, batch=1):
    return rng.standard_normal((batch, shape.nm, shape.mh, shape.mw)).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _trunc(v):
    """(int)v, or None where it is undefined"""
    v = float(v)
    return int(v) if -2147483648.0 <= v < 2147483648.0 else None


def _round(v):
    """(int)round((double)v) (C round: half away from zero), or None where it is undefined"""
    v = float(v)
    if not math.isfinite(v):
        return None
    r = math.copysign(math.floor(abs(v) + 0.5), v)
    return int(r) if -2147483648.0 <= r <= 2147483647.0 else None


def downscale_cells(variant, bbox, net_w, net_h, defect=None):
    """get_downscale_rect in fp32, clipped to the mask: (x_lo, x_hi, y_lo, y_hi) cells; an empty range where a conversion
    is undefined.  defect "v5_trunc": V5 truncates instead of rounding."""
    b = np.asarray(bbox, F32)
    four = F32(4)
    with np.errstate(all="ignore"):
        if variant == V8:
            left, top = b[0], b[1]
            right, bottom = F32(b[0] + b[2]), F32(b[1] + b[3])
            left = F32(0) if left < 0 else left
            top = F32(0) if top < 0 else top
            right = F32(net_w) if right > net_w else right
            bottom = F32(net_h) if bottom > net_h else bottom
            left, top, right, bottom = left / four, top / four, right / four, bottom / four
            conv = _trunc
        else:
            two = F32(2)
            left, top = F32(b[0] - b[2] / two), F32(b[1] - b[3] / two)
            right, bottom = F32(b[0] + b[2] / two), F32(b[1] + b[3] / two)
            left, top, right, bottom = left / four, top / four, right / four, bottom / four
            conv = _trunc if defect == "v5_trunc" else _round
        r = [conv(left), conv(top), conv(F32(right - left)), conv(F32(bottom - top))]
    if any(v is None for v in r):
        return 0, 0, 0, 0
    rx, ry, rw, rh = r
    mw, mh = net_w // 4, net_h // 4
    return max(rx, 0), min(rx + rw, mw), max(ry, 0), min(ry + rh, mh)


def cells64(variant, proto, bbox, coeffs, net_w, net_h, defect=None):
    """(m [mh, mw] float64 sigmoid cells, bound [mh, mw] of the fp32 kernel's cells) for one detection"""
    nm, mh, mw = proto.shape
    m = np.zeros((mh, mw))
    bound = np.zeros((mh, mw))
    x0, x1, y0, y1 = downscale_cells(variant, bbox, net_w, net_h, defect)
    if x0 < x1 and y0 < y1:
        c = np.asarray(coeffs, np.float64)
        p = proto[:, y0:y1, x0:x1].astype(np.float64)
        e = np.tensordot(c, p, axes=1)
        with np.errstate(over="ignore"):
            m[y0:y1, x0:x1] = 1.0 / (1.0 + np.exp(-e))
        bound[y0:y1, x0:x1] = 0.25 * gamma(nm) * np.tensordot(np.abs(c), np.abs(p), axes=1) + 3 * U
    return m, bound


def taps(dst, src, defect=None):
    """OpenCV's bilinear taps of `dst` outputs over `src` inputs: (s0, s1, w0, w1), weights fp32.  defect "tap": the first
    tap one cell to the right; "halo": the second tap is the first (min(s + 1, src - 1) replaced by s)."""
    scale = src / dst
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    lo, hi = s < 0, s >= src - 1
    f[lo | hi] = 0
    s[lo] = 0
    s[hi] = src - 1
    s1 = np.minimum(s + 1, src - 1)
    if defect == "tap":
        s = np.minimum(s + 1, src - 1)
    if defect == "halo":
        s1 = s
    return s, s1, (F32(1) - f).astype(F32), f


def blend64(src, ty, tx, bound=None):
    """Bilinear resize of float64 src [sh, sw] with taps ty (rows) and tx (columns): (values, bound) in float64; bound is
    the pixel bound from the bounds of the four inputs each pixel reads, or None."""
    sy, sy1, b0, b1 = ty
    sx, sx1, a0, a1 = tx
    a0, a1 = a0.astype(np.float64)[None, :], a1.astype(np.float64)[None, :]
    b0, b1 = b0.astype(np.float64)[:, None], b1.astype(np.float64)[:, None]
    r0, r1 = src[sy], src[sy1]
    out = (r0[:, sx] * a0 + r0[:, sx1] * a1) * b0 + (r1[:, sx] * a0 + r1[:, sx1] * a1) * b1
    if bound is None:
        return out, None
    q0, q1 = bound[sy], bound[sy1]
    worst = np.maximum(np.maximum(q0[:, sx], q0[:, sx1]), np.maximum(q1[:, sx], q1[:, sx1]))
    return out, worst * (1 + 4 * U) + 6 * U


def process_mask64(variant, proto, bbox, coeffs, net_w, net_h, defect=None, rows=None):
    """The float64 process_mask of one detection: (M [net_h, net_w], bound); rows: only these output rows."""
    nm, mh, mw = proto.shape
    m, cb = cells64(variant, proto, bbox, coeffs, net_w, net_h, defect)
    if not cb.any():   # an empty rectangle: every pixel blends four exact zeros
        n = net_h if rows is None else len(rows)
        return np.zeros((n, net_w)), np.full((n, net_w), 6 * U)
    ty = taps(net_h, mh, defect if defect == "halo" else None)
    tx = taps(net_w, mw, defect if defect == "tap" else None)
    if rows is not None:
        ty = tuple(t[rows] for t in ty)
    return blend64(m, ty, tx, cb)


def scale_mask64(M, bound, crop, img_w, img_h, rows=None):
    """scale_mask of a float64 net-size mask: the crop (x, y, w, h) resized to img_w x img_h -> (S, bound)"""
    x, y, w, h = crop
    ty, tx = taps(img_h, h), taps(img_w, w)
    if rows is not None:
        ty = tuple(t[rows] for t in ty)
    src = M[y:y + h, x:x + w]
    return blend64(src, ty, tx, None if bound is None else bound[y:y + h, x:x + w])


def select64(S, rect, img_w, img_h, rows=None, defect=None):
    """draw_mask_bbox's selection: 255 where (x, y) lies in get_rect clipped to the frame and S > 0.5 (S <= 0.5 is skipped;
    defect "threshold": S < 0.5 kept instead)."""
    x, y, w, h = (int(v) for v in rect)
    ys = np.arange(img_h) if rows is None else np.asarray(rows)
    xs = np.arange(img_w)
    inside = ((ys >= max(y, 0)) & (ys < min(y + h, img_h)))[:, None] & ((xs >= max(x, 0)) & (xs < min(x + w, img_w)))[None, :]
    keep = S < 0.5 if defect == "threshold" else S > 0.5
    return np.where(inside & keep, 255, 0).astype(np.uint8)


def canvas64(variant, proto, row, shape, img_w, img_h, crop, rect, rows=None, defect=None):
    """(canvas, S, bound of S) of one detection row, float64; rows: only these canvas rows"""
    R, off = shape.row
    if rect == (0, 0, 0, 0) or rect[2] <= 0 or rect[3] <= 0:
        n = img_h if rows is None else len(rows)
        z = np.zeros((n, img_w))
        return z.astype(np.uint8), z, z
    x, y, w, h = crop
    ty = taps(img_h, h)
    need = np.unique(np.concatenate([ty[0], ty[1]] if rows is None else [ty[0][rows], ty[1][rows]])) + y
    M = np.zeros((shape.net_h, shape.net_w))
    Mb = np.zeros((shape.net_h, shape.net_w))
    M[need], Mb[need] = process_mask64(variant, proto, row[:4], row[off:off + shape.nm], shape.net_w, shape.net_h,
                                       defect if defect != "threshold" else None, rows=need)
    S, sb = scale_mask64(M, Mb, crop, img_w, img_h, rows)
    return select64(S, rect, img_w, img_h, rows, defect), S, sb


def excess(got, ref, bound):
    """max of |got - ref| / bound (> 1 fails)"""
    return float(np.max(np.abs(got.astype(np.float64) - ref) / bound))


# ---------------------------------------------------------------------------------------------------------------------
# seg_canvas_kernel's shared-memory caps, as the library sizes them (trtx_yolo_seg_launch_caps runs the enqueue's own
# seg_fill_frames on the host), and what a band really needs
# ---------------------------------------------------------------------------------------------------------------------
SEG_BAND, SEG_MAX_Y, SEG_MAX_LY = 8, 16, 32
UNSUPPORTED = 4   # TRTX_ERR_UNSUPPORTED


def launch_caps(net_w, net_h, frames):
    """(rc, caps) of trtx_yolo_seg_launch_caps: caps = (M rows, cell rows, M columns, cell columns, dynamic smem bytes)"""
    import ctypes as C

    from tensorrtx_b200 import _lib as L
    from tensorrtx_b200 import plugins as P
    descs, _ = P._frames(frames, None, 0, None, False)
    q = L.MaskParams(V8, net_w, net_h, net_w // 4, net_h // 4, 32, 39, 7, 1)
    caps = (C.c_int32 * 5)()
    rc = L.load().trtx_yolo_seg_launch_caps(C.byref(q), descs, len(frames), caps)
    return rc, tuple(caps)


def band_needs(net_w, net_h, img_w, img_h, crop):
    """The most y slots, cell slots, M columns and cell columns any band of the frame lists (seg_canvas_kernel's thread 0
    lists, for get_rect covering the whole frame, which needs the most)."""
    cx, cy, cw, ch = crop
    mh, mw = net_h // 4, net_w // 4
    sy, sy1, _, _ = taps(img_h, ch)
    ly, ly1, _, _ = taps(net_h, mh)
    most_y = most_ly = 0
    for y0 in range(0, img_h, SEG_BAND):
        Y = set((sy[y0:y0 + SEG_BAND] + cy).tolist()) | set((sy1[y0:y0 + SEG_BAND] + cy).tolist())
        LY = set(ly[list(Y)].tolist()) | set(ly1[list(Y)].tolist())
        most_y, most_ly = max(most_y, len(Y)), max(most_ly, len(LY))
    sx, sx1, _, _ = taps(img_w, cw)
    Xa, Xb = cx + sx[0], cx + sx1[-1]
    lx, lx1, _, _ = taps(net_w, mw)
    return most_y, most_ly, Xb - Xa + 1, lx1[Xb] - lx[Xa] + 1


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
def _boxes(rng, variant, shape, n_rand=6):
    return edge_boxes(variant, shape.net_w, shape.net_h) + undefined_boxes(variant, shape.net_w, shape.net_h) + \
        random_boxes(rng, variant, shape.net_w, shape.net_h, n_rand)


def test_reference_rectangle_matches_the_drivers():
    """downscale_cells spells get_downscale_rect as the drivers do: V8 truncates, V5 rounds half away from zero, and the
    undefined conversions give an empty range."""
    assert downscale_cells(V8, [5, 6, 21, 22], 640, 640) == (1, 6, 1, 6)      # x: 1 + (int)(6.5 - 1.25); y: 1 + (int)5.5
    assert downscale_cells(V5, [10, 10, 12, 12], 640, 640) == (1, 4, 1, 4)    # left 4 -> 1; 12/4 = 3
    assert downscale_cells(V5, [6, 6, 8, 8], 640, 640) == (1, 3, 1, 3)        # left 2 -> .5 -> 1; width 2
    assert downscale_cells(V5, [6, 6, 8, 8], 640, 640, "v5_trunc") == (0, 2, 0, 2)
    assert downscale_cells(V5, [-2, 6, 8, 8], 640, 640)[0:2] == (0, 0)        # left -6/4 = -1.5 -> -2, width 2 -> 0
    assert downscale_cells(V8, [5, 5, np.inf, 50], 640, 640) == (1, 159, 1, 13)  # right clamps to the net: defined
    for v in (np.nan, np.inf, 1e10):
        assert downscale_cells(V8, [v, 5, 50, 50], 640, 640) == (0, 0, 0, 0)
    assert downscale_cells(V5, [1e9, 320, 1e10, 100], 640, 640) == (0, 0, 0, 0)  # left defined, width past INT_MAX
    assert downscale_cells(V8, [3e9, 5, 50, 50], 640, 640)[0] == 750000000     # past 2^31 in pixels, not in cells
    x0, x1, y0, y1 = downscale_cells(V5, [-1.2e10, 320, -8e9, 100], 640, 640)   # rx, rw about -2e9: defined, empty
    assert x0 == 0 and x1 < -2 ** 31 and (y0, y1) == (68, 93)   # top 67.5 -> 68, height 25


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s.id)
def test_process_mask_reference_matches_oracle(oracle, shape):
    """On every shape class, both variants: the oracle's process_mask (the drivers' fp32 expressions, glibc expf) lies
    within the bound of the float64 reference on every pixel; the bound is at least 1000x under the error of one wrong tap;
    and every injected defect of the reference breaks the comparison."""
    rng = np.random.default_rng(1000 + shape.net_w + shape.net_h + shape.nm + 100 * shape.row[0] + shape.row[1])
    proto = make_proto(rng, shape)[0]
    R, off = shape.row
    for variant in (V8, V5):
        boxes = _boxes(rng, variant, shape)
        d = make_dets(rng, shape, boxes)
        rows = d[1:].reshape(len(boxes), R)
        worst, worst_bound, tap_err = 0.0, 0.0, []
        caught = {k: False for k in DEFECTS if k != "threshold" and (k != "v5_trunc" or variant == V5)}
        for row in rows:
            got = oracle.process_mask(variant, proto, row[:4], row[off:off + shape.nm], shape.net_w, shape.net_h)
            ref, bound = process_mask64(variant, proto, row[:4], row[off:off + shape.nm], shape.net_w, shape.net_h)
            assert excess(got, ref, bound) <= 1.0, (shape.id, variant, row[:4])
            worst = max(worst, float(np.abs(got - ref).max()))
            worst_bound = max(worst_bound, float(bound.max()))
            for k in caught:
                if not caught[k]:
                    bad, _ = process_mask64(variant, proto, row[:4], row[off:off + shape.nm], shape.net_w, shape.net_h, k)
                    caught[k] = excess(got, bad, bound) > 1.0
                    if k == "tap" and np.any(bad != ref):
                        tap_err.append(float(np.abs(bad - ref).max()))
        assert all(caught.values()), (shape.id, variant, caught)
        assert tap_err and worst_bound * 1000 < max(tap_err), (worst_bound, tap_err)
        print(f"{shape.id} v{variant}: oracle |err| {worst:.2e}, bound {worst_bound:.2e}, one tap {max(tap_err):.2e}")


def _seg_frames(shape):
    """Frames whose scale_mask crop is not empty at this net"""
    from oracle import seg_post as SP
    frames = [(1, 1), (2, 2), (4, 4), (8, 8), (333, 1001), (1282, 719)]
    return [(w, h) for w, h in frames if min(SP.scale_mask_rect(w, h, shape.net_w, shape.net_h)[2:]) > 0]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s.id)
def test_seg_reference_matches_oracle(shape):
    """The float64 canvas equals the oracle's segmentation post-process except where |S64 - 0.5| is within S's bound, its
    S is within the bound of the oracle's S, and every defect (the threshold written as < 0.5 included) breaks it."""
    from oracle import seg_post as SP
    rng = np.random.default_rng(2000 + shape.net_w + shape.net_h + shape.nm + 100 * shape.row[0] + shape.row[1])
    proto = make_proto(rng, shape)[0]
    R, off = shape.row
    for variant in (V8, V5):
        boxes = random_boxes(rng, variant, shape.net_w, shape.net_h, 5) + edge_boxes(variant, shape.net_w, shape.net_h)[-8:]
        d = make_dets(rng, shape, boxes)
        K = len(boxes)
        caught = {k: False for k in DEFECTS if k != "v5_trunc" or variant == V5}
        for w, h in _seg_frames(shape):
            crop = SP.scale_mask_rect(w, h, shape.net_w, shape.net_h)
            orows, ocanv, oS = SP.seg_postprocess(variant, proto, d, w, h, max_rows=K, row_floats=R, coeff_offset=off,
                                                  max_masks=K, net_w=shape.net_w, net_h=shape.net_h, scaled=True)
            rows = None if w * h <= 200_000 else np.unique(np.linspace(0, h - 1, 40).astype(int))
            for k in range(K):
                row = d[1 + k * R:1 + (k + 1) * R]
                rect = tuple(int(v) for v in orows[1 + 6 * k:5 + 6 * k])
                c, S, sb = canvas64(variant, proto, row, shape, w, h, crop, rect, rows)
                oc, os_ = (ocanv[k], oS[k]) if rows is None else (ocanv[k][rows], oS[k][rows])
                near = np.abs(S - 0.5) <= sb
                assert not np.any((c != oc) & ~near), (shape.id, variant, (w, h), k)
                if rect[2] > 0 and rect[3] > 0:
                    assert excess(os_, S, sb) <= 1.0
                for dk in caught:
                    if not caught[dk]:
                        bc, _, _ = canvas64(variant, proto, row, shape, w, h, crop, rect, rows, dk)
                        caught[dk] = bool(np.any((bc != oc) & ~near))
        assert all(caught.values()), (shape.id, variant, caught)


@pytest.mark.parametrize("shape", NET_SHAPES, ids=lambda s: s.id)
def test_seg_caps_cover_every_band(shape):
    """The library's shared-memory caps for the canvas kernel hold what every band of a frame lists, at every net, on tiny,
    mixed and 8K frames: a cap one row short would let the M rows overwrite the cells.  The dynamic shared memory is the two
    regions, M [rows x columns] and cells [rows x columns]."""
    from oracle import seg_post as SP
    frames = [(1, 1), (2, 2), (4, 4), (8, 8), (16, 9), (3, 17), (333, 1001), (1282, 719), (1920, 1080), (7680, 4320)]
    for w, h in frames:
        crop = SP.scale_mask_rect(w, h, shape.net_w, shape.net_h)
        rc, caps = launch_caps(shape.net_w, shape.net_h, [(w, h)])
        if min(crop[2:]) <= 0:
            assert rc == UNSUPPORTED, (shape.id, (w, h))    # the empty crop
            continue
        assert rc == 0, (shape.id, (w, h))
        y_cap, ly_cap, x_cap, lx_cap, smem = caps
        ny, nly, nX, nLX = band_needs(shape.net_w, shape.net_h, w, h, crop)
        assert ny <= y_cap <= SEG_MAX_Y and nly <= ly_cap <= SEG_MAX_LY, (shape.id, (w, h), ny, nly, caps)
        assert nX <= x_cap and nLX <= lx_cap <= shape.mw, (shape.id, (w, h), nX, nLX, caps)
        assert smem == (y_cap * x_cap + ly_cap * lx_cap) * 4
    # a 1 x 1 frame reaches the hard limits: 16 rows of M, 32 low-resolution rows
    assert launch_caps(shape.net_w, shape.net_h, [(1, 1)])[1][:2] == (16, 32)


def largest_seg_net():
    """The largest square net whose canvas launch the library accepts for a 1 x 1 frame (the smallest frame needs the most:
    every band hits the hard caps and the crop is the whole net)."""
    n = 2560
    while launch_caps(n, n, [(1, 1)])[0] != 0:
        n -= 4
    return n


def test_largest_seg_net():
    """2408^2 is the largest: 96 bytes per net column (16 M rows + 32 cell rows of a quarter column) within 227 KB less the
    library's 1 KB margin for the kernel's static arrays.  A 4 x 4 frame at 2560^2 would need 240 KB and is refused."""
    assert largest_seg_net() == 2408
    assert launch_caps(2408, 2408, [(1, 1)]) == (0, (16, 32, 2408, 602, 231168))
    assert launch_caps(2412, 2412, [(1, 1)])[0] == UNSUPPORTED
    assert launch_caps(2560, 2560, [(4, 4)]) == (UNSUPPORTED, (16, 32, 2560, 640, 245760))
    assert launch_caps(640, 640, [(1, 1)]) == (0, (16, 32, 640, 160, 61440))     # the 640 net's most: 60 KB
    assert launch_caps(640, 640, [(1920, 1080), (1, 5000)])[0] == UNSUPPORTED   # an empty crop refuses the call
