"""RoIAlign (tensorrtx_b200/csrc/roi_align.cu) in float64, and a mirror of how trtx_roi_align_typed dispatches a call.

The float64 reference is separable.  Every sample of a bin has one y coordinate and one x coordinate, its bilinear weights
are products of a y weight and an x weight, and it counts only when both coordinates are valid.  So a bin is

    out[c, ph, pw] = (1 / count) * Ay[ph] . F[c] . Ax[pw]^T

where Ay[ph, h] sums the y weights that the samples of row ph put on map row h (0 for a sample outside the map), and Ax
likewise.  The geometry (start, bin size, sampling grid, count) is built with the fp32 arithmetic of the kernel, because it
decides which samples exist; everything after it (sample coordinates, weights, sums) is float64.

Tolerance of one bin, from the fp32 arithmetic of the kernel (u = 2^-24, unit roundoff):
  * one sample: the four weights `hy * hx` (one rounding each), `hy = 1 - ly` (one rounding), one multiply and three fused
    multiply-adds: at most 6 u * S_s, with S_s = sum over the four taps of |w * v|;
  * `output_val += val`, count times: each addition rounds by at most u * |partial sum| <= u * S, S = sum of S_s;
  * `/ count`: u * |bin|;
  * the sample coordinate itself is rounded: `start + p * bin + (i + .5f) * bin / grid` takes 5 roundings, and the kernel may
    contract `roi * scale - 0.5` into an FMA, which moves start and end by an ulp and the bin size with them.  The coordinate
    is off by at most d = u * (|y| + |start + p * bin| + 3 |p * bin| + 3 |bin| + 16 M), M the largest of |start|, |end|,
    |roi * scale| on that axis.  A bilinear value is Lipschitz in y with constant sum_x w_x |F[h + 1, x] - F[h, x]| (taken
    over the cell of the sample and its two neighbours, as d may cross a cell edge), so the sample moves by at most
    d_y * Gy + d_x * Gx.
  Together: tol = ((count + 8) u S + sum_s (d_y Gy + d_x Gx)) / |count| + u |bin|, every term separable like the bin.
Two things are not continuous in the coordinates, and the bins they touch are "unpinned" and left out of the float64
comparison (tests/test_roi_align_paths_gpu.py still compares them bit for bit between the two kernels):
  * the sampling grid `ceil(roi_height / P)`: when the FMA and non-FMA forms of the geometry give different grids;
  * the validity cutoffs `y < -1 || y > size` of bilinear_interpolate: a sample within max(1e-3, 2 d) of one, where one ulp
    adds or drops a whole tap."""
from __future__ import annotations

import numpy as np
import pytest

F32 = np.float32
U = 2.0 ** -24

# roi_align.cu: kRoiMaxTable, kRoiChannelsPerCta, kRoiWindowBytes, and RoiWin<T> {kCU, kGroup, kPad, kMin} by element size
MAX_TABLE, CPC, WINDOW_BYTES = 256, 64, 65536
WIN = {4: (8, 8, 4, 4), 2: (16, 16, 8, 8)}


# ---------------------------------------------------------------------------------------------------------------------
# fp32 geometry (RoiAlign.cu:104-127, roi_geom in roi_align.cu)
# ---------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 a * b + c with one rounding: a * b is exact in float64, the sum's float64 rounding error is recovered with
    TwoSum and decides the one case where rounding the float64 sum to fp32 is not the rounding of the exact value (a tie)."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, F32).astype(np.float64) for x in (a, b, c)))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    r = s.astype(F32)
    r2 = np.nextafter(r, np.where(s > r, F32(np.inf), F32(-np.inf)).astype(F32))
    tie = (r.astype(np.float64) != s) & (np.abs(s - r) == np.abs(s - r2.astype(np.float64))) & (err != 0)
    toward_r2 = np.sign(err) == np.sign(r2.astype(np.float64) - s)
    return np.where(tie & toward_r2, r2, r)


def geometry(rois, P, scale, sampling, fma=False):
    """Per proposal, fp32: (start_h, start_w, bin_h, bin_w, grid_h, grid_w, count) as the kernel computes them; fma: the
    form with `roi * scale - 0.5` contracted into one fused multiply-add."""
    r = np.asarray(rois, F32).reshape(-1, 4)
    s, half = F32(scale), F32(0.5)
    with np.errstate(all="ignore"):
        st = fma32(r, s, -half) if fma else (r * s) - half
        start_w, start_h, end_w, end_h = st[:, 0], st[:, 1], st[:, 2], st[:, 3]
        roi_w, roi_h = end_w - start_w, end_h - start_h
        bin_h, bin_w = roi_h / F32(P), roi_w / F32(P)
        if sampling > 0:
            gh = gw = np.full(len(r), sampling, np.int64)
        else:
            gh, gw = np.ceil(roi_h / F32(P)).astype(np.int64), np.ceil(roi_w / F32(P)).astype(np.int64)
    count = (gh * gw).astype(F32)
    return dict(start_h=start_h, start_w=start_w, end_h=end_h, end_w=end_w, bin_h=bin_h, bin_w=bin_w, gh=gh, gw=gw,
                count=count, rs=np.abs(r.astype(np.float64) * np.float64(s)))


def samples32(start, binsz, p, i, grid, fma=False):
    """roi_sample in fp32: `start + p * bin + static_cast<float>(i + .5f) * bin / static_cast<float>(grid)`"""
    p32, bin32 = np.asarray(p, F32), F32(binsz)
    head = fma32(p32, bin32, F32(start)) if fma else F32(start) + p32 * bin32
    return head + (np.asarray(i, F32) + F32(0.5)) * bin32 / F32(grid)


def axis_taps32(y, size):
    """axis_tap of roi_align.cu on fp32 coordinates: (low, high, valid)"""
    y = np.asarray(y, F32)
    valid = ~((y.astype(np.float64) < -1.0) | (y.astype(np.float64) > size))
    yc = np.where(y <= 0, F32(0), y)
    low = yc.astype(np.int64)
    clamp = low >= size - 1
    low = np.where(clamp, size - 1, low)
    high = np.where(clamp, size - 1, low + 1)
    return low, high, valid


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror: window_ok and the channels per pass of roi_align_launch / roi_align_window_kernel
# ---------------------------------------------------------------------------------------------------------------------
def kernel_for(P, C, H, W, es):
    """which kernel trtx_roi_align_typed launches for element size es (4: fp32, 2: fp16): 'window', 'direct' or
    'unsupported' (TRTX_ERR_UNSUPPORTED, nothing launched)"""
    if P > 32 or P * P > 256:
        return "unsupported"
    return "window" if P == 14 and C % (16 // es) == 0 and H * W <= WINDOW_BYTES // 16 else "direct"


def cpass_for(cells, es):
    """(channels per pass, regime) of a window of `cells` cells: 'cpass64', 'cpass_mid' (kGroup..56) or 'kmin'"""
    _, group, pad, kmin = WIN[es]
    cpass = min(CPC, (WINDOW_BYTES // es // cells - pad) & ~(group - 1))
    if cpass < group:
        return kmin, "kmin"
    return cpass, "cpass64" if cpass == CPC else "cpass_mid"


def cpass_boundaries(es):
    """the largest window (cells) of each of the regimes cpass64 and cpass_mid"""
    last = {}
    for cells in range(1, WINDOW_BYTES // 16 + 1):
        last[cpass_for(cells, es)[1]] = cells
    return last["cpass64"], last["cpass_mid"]


def window_hull(rois, P, scale, sampling, H, W, fma=False):
    """per proposal: None when the kernel does not tabulate its samples (a grid of more than 256 entries per axis, or none),
    () when no sample is inside the map, else (y0, y1, x0, x1, grid_h, grid_w) of the window kernel's hull"""
    g = geometry(rois, P, scale, sampling, fma)
    out = []
    for n in range(len(g["gh"])):
        gh, gw = int(g["gh"][n]), int(g["gw"][n])
        if not (gh > 0 and gw > 0 and P * gh <= MAX_TABLE and P * gw <= MAX_TABLE):
            out.append(None)
            continue
        ph, iy = np.divmod(np.arange(P * gh), gh)
        pw, ix = np.divmod(np.arange(P * gw), gw)
        ly, hy, vy = axis_taps32(samples32(g["start_h"][n], g["bin_h"][n], ph, iy, gh, fma), H)
        lx, hx, vx = axis_taps32(samples32(g["start_w"][n], g["bin_w"][n], pw, ix, gw, fma), W)
        if not vy.any() or not vx.any():
            out.append(())
            continue
        out.append((int(ly[vy].min()), int(hy[vy].max()), int(lx[vx].min()), int(hx[vx].max()), gh, gw))
    return out


def regimes(rois, P, C, H, W, scale, sampling, es):
    """The code paths of roi_align.cu one call takes, as names '<dtype>:<kernel>:<path>'.  Window kernel paths: untabled (the
    direct code on coordinates computed on the fly), outside (every sample outside the map), cpass64 / cpass_mid / kmin,
    round_full@<cpass regime> / round_partial@<cpass regime> (tap rounds of kCU channels), pow2 / div (the divide by count),
    fill_mul / fill_div (a window cell's row by multiplication or by division).  A proposal whose paths differ between the
    FMA and non-FMA forms of the geometry adds none."""
    dt = "f32" if es == 4 else "f16"
    k = kernel_for(P, C, H, W, es)
    if k != "window":
        if k == "direct":
            g = geometry(rois, P, scale, sampling)
            tab = (g["gh"] > 0) & (g["gw"] > 0) & (P * g["gh"] <= MAX_TABLE) & (P * g["gw"] <= MAX_TABLE)
            return {f"{dt}:direct:{'tabled' if t else 'untabled'}" for t in tab}
        return {f"{dt}:{k}"}
    cu = WIN[es][0]
    got = set()
    for a, b in zip(window_hull(rois, P, scale, sampling, H, W), window_hull(rois, P, scale, sampling, H, W, fma=True)):
        if a != b:
            continue
        if a is None:
            got.add("untabled")
            continue
        if a == ():
            got.add("outside")
            continue
        y0, y1, x0, x1, gh, gw = a
        ww, cells = x1 - x0 + 1, (y1 - y0 + 1) * (x1 - x0 + 1)
        cpass, name = cpass_for(cells, es)
        got |= {name, "fill_mul" if cells * ww <= 65536 else "fill_div", "pow2" if (gh * gw) & (gh * gw - 1) == 0 else "div"}
        for c_begin in range(0, C, CPC):
            c_end = min(C, c_begin + CPC)
            for cb in range(c_begin, c_end, cpass):
                nc = min(cpass, c_end - cb)
                for k0 in range(0, nc, cu):
                    got.add(f"round_{'full' if nc - k0 >= cu else 'partial'}@{name}")
    return {f"{dt}:window:{r}" for r in got}


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _axis(start, end, rs, binsz, grid, P, size):
    """(A, T, cut): the summed y (or x) weights A[p, h] of the samples of bin row p, their coordinate error bounds on the
    sample's cell T[p, h], and whether a sample of row p lies at a validity cutoff"""
    A = np.zeros((P, size))
    T = np.zeros((P, size))
    cut = np.zeros(P, bool)
    if grid <= 0:
        return A, T, cut
    start, binsz = np.float64(start), np.float64(binsz)
    p, i = np.divmod(np.arange(P * grid), grid)
    y = start + p * binsz + (i + .5) * binsz / grid
    M = max(abs(np.float64(start)), abs(np.float64(end)), *rs)
    d = U * (np.abs(y) + np.abs(start + p * binsz) + 3 * np.abs(p * binsz) + 3 * abs(binsz) + 16 * M)
    near = (np.abs(y + 1) <= np.maximum(1e-3, 2 * d)) | (np.abs(y - size) <= np.maximum(1e-3, 2 * d))
    np.logical_or.at(cut, p, near)
    valid = ~((y < -1.0) | (y > size))
    yc = np.maximum(y, 0.0)
    low = np.floor(yc).astype(np.int64)
    clamp = low >= size - 1
    low = np.where(clamp, size - 1, low)
    high = np.where(clamp, size - 1, low + 1)
    l = np.where(clamp, 0.0, yc - low)
    v = valid.astype(np.float64)
    np.add.at(A, (p, low), v * (1 - l))
    np.add.at(A, (p, high), v * l)
    np.add.at(T, (p, low), v * d)
    return A, T, cut


def _slope(F, axis):
    """Lipschitz constant of the bilinear value along `axis` around each cell: max |difference| over the cell's edge pairs
    h-1|h, h|h+1, h+1|h+2"""
    D = np.abs(np.diff(F, axis=axis))
    pad = [(0, 0)] * F.ndim
    pad[axis] = (2, 2)
    D = np.pad(D, pad)
    n = F.shape[axis]
    take = lambda k: np.take(D, np.arange(k, k + n), axis=axis)
    return np.maximum(np.maximum(take(1), take(2)), take(3))


def reference(rois, feat, P, scale, sampling):
    """One image: rois [N, 4] fp32, feat [C, H, W] finite -> (bins [N, C, P, P] float64, tol [N, C, P, P], pinned [N, P, P])."""
    rois = np.asarray(rois, F32).reshape(-1, 4)
    F = np.asarray(feat, np.float64)
    C, H, W = F.shape
    N = len(rois)
    g, gf = geometry(rois, P, scale, sampling), geometry(rois, P, scale, sampling, fma=True)
    aF, Gy, Gx = np.abs(F), _slope(F, 1), _slope(F, 2)
    out = np.empty((N, C, P, P))
    tol = np.empty((N, C, P, P))
    pinned = np.empty((N, P, P), bool)
    for n in range(N):
        gh, gw = int(g["gh"][n]), int(g["gw"][n])
        Ay, Ty, cy = _axis(g["start_h"][n], g["end_h"][n], g["rs"][n, 1::2], g["bin_h"][n], gh, P, H)
        Ax, Tx, cx = _axis(g["start_w"][n], g["end_w"][n], g["rs"][n, 0::2], g["bin_w"][n], gw, P, W)
        count = np.float64(g["count"][n])
        with np.errstate(all="ignore"):
            val = Ay @ F @ Ax.T
            out[n] = val / count
            S = Ay @ aF @ Ax.T
            coord = Ty @ Gy @ Ax.T + Ay @ Gx @ Tx.T
            tol[n] = ((abs(count) + 8) * U * S + coord) / abs(count) + U * np.abs(out[n])
        same_grid = gh == int(gf["gh"][n]) and gw == int(gf["gw"][n])
        pinned[n] = same_grid & ~cy[:, None] & ~cx[None, :]
    return out, tol, pinned


def assert_close_to_reference(got, rois, feat, P, scale, sampling, msg=""):
    """got [N, C, P, P] (one image) against the float64 reference: NaN bins where the reference has them (0 / 0), pinned
    bins within their tolerance.  Returns the number of bins compared."""
    ref, tol, pinned = reference(rois, feat, P, scale, sampling)
    got = np.asarray(got, np.float64)
    nan = np.isnan(ref)
    pin = np.broadcast_to(pinned[:, None], ref.shape)
    assert np.array_equal(np.isnan(got) & pin, nan & pin), (msg, "NaN bins differ")
    m = pin & ~nan
    err = np.abs(got - ref)
    bad = m & ~(err <= tol)
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError(f"{msg}: {int(bad.sum())} of {int(m.sum())} bins off the float64 reference, first at "
                             f"(n, c, ph, pw) = {tuple(i)}: got {got[tuple(i)]!r}, reference {ref[tuple(i)]!r}, tol {tol[tuple(i)]:.3g}")
    return int(m.sum())


# ---------------------------------------------------------------------------------------------------------------------
# proposals, in feature-map units u = roi * spatial_scale (sample coordinates are u - 0.5)
# ---------------------------------------------------------------------------------------------------------------------
FAMILIES = ("inside", "straddle_top", "straddle_bottom", "straddle_left", "straddle_right", "outside_top", "outside_bottom",
            "outside_left", "outside_right", "one_axis", "subcell", "larger", "zero", "negative")


def proposals(rng, H, W, P, scale, n_each, max_cells=None):
    """n_each proposals of every family of FAMILIES, [len(FAMILIES) * n_each, 4] fp32 image coordinates.  max_cells bounds
    a side (adaptive sampling: grid = ceil(side / P), so 60 * P keeps it at 60 per axis)."""
    mc = max_cells or 1e9
    out = []

    def side(size, lo=0.3):
        return np.exp(rng.uniform(np.log(lo), np.log(max(lo * 1.01, min(size, mc))), n_each))

    for fam in FAMILIES:
        h, w = side(H), side(W)
        y1, x1 = rng.uniform(0, 1, n_each) * np.maximum(H - h, 0), rng.uniform(0, 1, n_each) * np.maximum(W - w, 0)
        if fam == "straddle_top":
            y1 = -h * rng.uniform(0.2, 0.8, n_each)
        elif fam == "straddle_bottom":
            y1 = H - h * rng.uniform(0.2, 0.8, n_each)
        elif fam == "straddle_left":
            x1 = -w * rng.uniform(0.2, 0.8, n_each)
        elif fam == "straddle_right":
            x1 = W - w * rng.uniform(0.2, 0.8, n_each)
        elif fam == "outside_top":
            y1 = -h - rng.uniform(0.6, 5, n_each)
        elif fam == "outside_bottom":
            y1 = H + 1.6 + rng.uniform(0, 5, n_each)
        elif fam == "outside_left":
            x1 = -w - rng.uniform(0.6, 5, n_each)
        elif fam == "outside_right":
            x1 = W + 1.6 + rng.uniform(0, 5, n_each)
        elif fam == "one_axis":           # x inside, y wholly above or below the map
            y1 = np.where(rng.random(n_each) < 0.5, -h - rng.uniform(0.6, 5, n_each), H + 1.6 + rng.uniform(0, 5, n_each))
        elif fam == "subcell":
            h, w = rng.uniform(0.02, 0.9, n_each), rng.uniform(0.02, 0.9, n_each)
            y1, x1 = rng.uniform(-0.5, H, n_each), rng.uniform(-0.5, W, n_each)
        elif fam == "larger":
            gy, gx = min(H * 0.5 + 1, (mc - H) / 2), min(W * 0.5 + 1, (mc - W) / 2)
            y1, x1 = -rng.uniform(0.5, max(0.6, gy), n_each), -rng.uniform(0.5, max(0.6, gx), n_each)
            h, w = H - 2 * y1, W - 2 * x1
        elif fam == "zero":
            h = w = np.zeros(n_each)
        elif fam == "negative":
            h, w = -rng.uniform(0.1, 3, n_each), np.where(rng.random(n_each) < 0.5, -rng.uniform(0.1, 3, n_each), w)
        out.append(np.stack([x1, y1, x1 + w, y1 + h], -1))
    return (np.concatenate(out) / scale).astype(F32)


def fit_axis(target, size, P, scale, sampling):
    """(u1, u2) in feature units whose samples span exactly `target` map rows (hull high - low + 1) in both forms of the
    geometry, with neither outermost sample within 0.05 of a cell edge"""
    pg = P * (sampling if sampling > 0 else max(1, -(-target // P)))
    guess = (target - 1) * pg / max(1, pg - 1)     # the outermost samples sit half a sample spacing inside the proposal
    for u0, length in ((u0, l) for u0 in (0.3, 0.75, 1.2) for l in np.arange(max(0.05, guess - 3), guess + 3, 1 / 64)):
        r = np.array([[u0 / scale, u0 / scale, (u0 + length) / scale, (u0 + length) / scale]], F32)
        got = []
        for fma in (False, True):
            g = geometry(r, P, scale, sampling, fma)
            grid = int(g["gh"][0])
            if grid <= 0 or P * grid > MAX_TABLE:
                break
            p, i = np.divmod(np.arange(P * grid), grid)
            y = samples32(g["start_h"][0], g["bin_h"][0], p, i, grid, fma)
            low, high, valid = axis_taps32(y, size)
            frac = np.array([y.min(), y.max()], np.float64) % 1     # the outermost samples decide the hull
            if not valid.all() or (np.minimum(frac, 1 - frac) < 0.05).any():
                break
            got.append(int(high.max() - low.min() + 1))
        if got == [target, target]:
            return u0, u0 + float(length)
    raise AssertionError(f"no proposal spans {target} cells of {size}")


def hull_proposal(wh, ww, H, W, P, scale, sampling):
    """one proposal [4] fp32 whose window kernel hull is wh x ww cells"""
    y1, y2 = fit_axis(wh, H, P, scale, sampling)
    x1, x2 = fit_axis(ww, W, P, scale, sampling)
    return (np.array([x1, y1, x2, y2]) / scale).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks of the reference itself
# ---------------------------------------------------------------------------------------------------------------------
def test_cpass_boundaries_follow_the_kernel_formula():
    """fp32: 64 channels per pass up to 240 cells, 8..56 up to 1365, 4 (16 bytes per cell) beyond; fp16: 455 and 1365"""
    assert cpass_boundaries(4) == (240, 1365)
    assert cpass_boundaries(2) == (455, 1365)
    assert cpass_for(4096, 4) == (4, "kmin") and cpass_for(4096, 2) == (8, "kmin")
    assert kernel_for(14, 84, 64, 64, 4) == "window" and kernel_for(14, 84, 64, 64, 2) == "direct"
    assert kernel_for(14, 64, 65, 64, 4) == "direct" and kernel_for(7, 64, 50, 67, 4) == "direct"
    assert kernel_for(17, 8, 7, 9, 4) == "unsupported" and kernel_for(16, 8, 7, 9, 4) == "direct"


def test_fma32_rounds_once():
    rng = np.random.default_rng(0)
    a, b, c = (rng.standard_normal(20000).astype(F32) * F32(100) for _ in range(3))
    from fractions import Fraction
    for k in range(0, 20000, 97):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        r = fma32(a[k], b[k], c[k])
        lo, hi = np.nextafter(r, F32(-np.inf)), np.nextafter(r, F32(np.inf))
        err = abs(Fraction(float(r)) - exact)
        assert err <= abs(Fraction(float(lo)) - exact) and err <= abs(Fraction(float(hi)) - exact)
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is an fp32 tie; the float64 sum with +-2^-80 is still the tie, the exact one is not
    x = F32(1 + 2.0 ** -12)
    assert fma32(x, x, F32(2.0 ** -80)) == F32(1 + 2.0 ** -11 + 2.0 ** -23)
    assert fma32(x, x, F32(-2.0 ** -80)) == F32(1 + 2.0 ** -11)


# the shapes of tests/test_roi_align_paths_gpu.py: (P, C, H, W, spatial_scale, sampling_ratio)
MATRIX = [(14, 4, 1, 1, 1 / 8, 0), (14, 8, 1, 67, 1 / 4, 2), (14, 20, 50, 1, 1 / 32, 3), (14, 64, 7, 9, 1.0, 0),
          (14, 68, 50, 67, 0.3, 0), (14, 84, 64, 64, 1 / 16, 4), (14, 8, 1, 4096, 1 / 8, 2), (14, 20, 4096, 1, 1 / 4, 1),
          (14, 8, 64, 64, 1 / 16, 19), (1, 1, 50, 67, 1 / 16, 0), (2, 3, 7, 9, 1 / 4, 2), (7, 5, 65, 64, 1 / 8, 0),
          (7, 6, 50, 67, 1 / 32, 37), (16, 5, 200, 272, 0.3, 0), (16, 4, 64, 64, 1.0, 17), (14, 3, 200, 272, 1 / 16, 2)]


def _ids(m):
    return [f"P{p}-c{c}-{h}x{w}-s{s:.4g}-sr{sr}" for p, c, h, w, s, sr in m]


@pytest.mark.parametrize("P,C,H,W,scale,sampling", MATRIX, ids=_ids(MATRIX))
def test_reference_equals_the_oracle_within_tolerance(oracle, P, C, H, W, scale, sampling):
    """the fp32 CPU restatement of the reference kernel (oracle/trtx_oracle.c) is within the float64 reference's tolerance"""
    rng = np.random.default_rng(P * 1000 + C + H + W)
    rois = proposals(rng, H, W, P, scale, 2, max_cells=60 * P if sampling == 0 else None)
    feat = rng.standard_normal((C, H, W)).astype(F32)
    n = assert_close_to_reference(oracle.roi_align(rois, feat, P, scale, sampling), rois, feat, P, scale, sampling)
    assert n > 0.5 * len(rois) * C * P * P


@pytest.mark.parametrize("P", [1, 2, 4, 7, 14, 16])
@pytest.mark.parametrize("sampling", [0, 1, 2, 3])
def test_reference_equals_torchvision_on_pinned_bins(P, sampling):
    """torchvision.ops.roi_align(aligned=True) is the same operation in float64 with float64 geometry; where the fp32
    geometry of the kernel is exact (dyadic corners, bins of a dyadic size) the two agree to rounding"""
    torch = pytest.importorskip("torch")
    tv = pytest.importorskip("torchvision")
    rng = np.random.default_rng(P * 10 + sampling)
    C, H, W, scale = 3, 23, 31, 1 / 8
    n = 60
    u1 = rng.integers(-16, 8 * W, (n, 2)) / 8                  # corners on multiples of 1/8 cell
    side = rng.integers(1, 8 * min(H, 30), (n, 2)) * P / 8     # sides of a multiple of P / 8 cells: bin sizes k / 8
    rois = np.concatenate([u1, u1 + side], 1) / scale
    rois = np.concatenate([rois, proposals(rng, H, W, P, scale, 2, max_cells=30 * P)]).astype(F32)
    rois = rois[(rois[:, 2] > rois[:, 0]) & (rois[:, 3] > rois[:, 1])]   # torchvision counts at least one sample
    feat = rng.standard_normal((C, H, W))
    ref, _, pinned = reference(rois, feat, P, scale, sampling)
    boxes = torch.cat([torch.zeros(len(rois), 1, dtype=torch.float64), torch.from_numpy(rois.astype(np.float64))], 1)
    tvo = tv.ops.roi_align(torch.from_numpy(feat)[None], boxes, (P, P), scale, sampling, aligned=True).numpy()
    g = geometry(rois, P, scale, sampling)
    r64 = rois.astype(np.float64) * scale - 0.5
    exact = ((g["start_w"] == r64[:, 0]) & (g["start_h"] == r64[:, 1]) & (g["bin_w"] == (r64[:, 2] - r64[:, 0]) / P) &
             (g["bin_h"] == (r64[:, 3] - r64[:, 1]) / P))
    m = np.broadcast_to((pinned & exact[:, None, None])[:, None], ref.shape)
    assert m.sum() > 0.4 * ref.size
    np.testing.assert_allclose(ref[m], tvo[m], rtol=0, atol=1e-12)


@pytest.mark.parametrize("P,C,H,W,scale,sampling", [(14, 2, 50, 67, 1 / 16, 0), (14, 2, 7, 9, 1.0, 2), (7, 2, 64, 64, 1 / 8, 3),
                                                     (2, 2, 1, 67, 1 / 4, 0), (16, 2, 50, 1, 1 / 32, 4), (1, 2, 65, 64, 0.3, 0)])
def test_tolerance_is_tighter_than_one_sample(P, C, H, W, scale, sampling):
    """On bins of at most 64 samples, leaving out any one valid sample moves a bin by more than 10x its tolerance -- so a
    lost sample, a wrong tap, a wrong channel or a wrong divisor cannot pass.  The map is positive (every sample's value is
    at least 0.5) so that no sample happens to be worth nothing; coordinates are below 100 cells (the coordinate term of
    the tolerance grows with their ulp)."""
    rng = np.random.default_rng(P + H + W)
    rois = proposals(rng, H, W, P, scale, 3, max_cells=60 * P if sampling == 0 else None)
    feat = rng.uniform(0.5, 1.5, (C, H, W))
    ref, tol, pinned = reference(rois, feat, P, scale, sampling)
    g = geometry(rois, P, scale, sampling)
    checked = 0
    for n in range(len(rois)):
        gh, gw, count = int(g["gh"][n]), int(g["gw"][n]), float(g["count"][n])
        if not (0 < count <= 64 and gh > 0):
            continue
        for ph in range(0, P, max(1, P // 4)):
            for pw in range(0, P, max(1, P // 4)):
                if not pinned[n, ph, pw]:
                    continue
                y = np.float64(g["start_h"][n]) + ph * np.float64(g["bin_h"][n]) + (np.arange(gh) + .5) * np.float64(g["bin_h"][n]) / gh
                x = np.float64(g["start_w"][n]) + pw * np.float64(g["bin_w"][n]) + (np.arange(gw) + .5) * np.float64(g["bin_w"][n]) / gw
                vy, vx = ~((y < -1) | (y > H)), ~((x < -1) | (x > W))
                if not (vy.any() and vx.any()):
                    continue
                # the smallest valid sample is at least 0.5: dropping it moves the bin by at least 0.5 / count
                assert (0.5 / count > 10 * tol[n, :, ph, pw]).all(), (n, ph, pw, count, tol[n, :, ph, pw].max())
                checked += 1
    assert checked > 10
