"""The CenterNet decode's map generators and its float64 reference, checked on the CPU; tests/test_centernet_paths_gpu.py
runs the device on the same maps.

centernet_peaks_kernel streams each class map through shared memory in strips of R = max(1, 4096 / W) rows with a halo row
above and below, appends positive or NaN peaks to a 5120-entry list in cell order, cuts that list to its K best whenever the
next strip could overflow it (after a cut a cell needs a key strictly above the cut key), and merges the first K zero-valued
cells in when fewer than K candidates exist.  The generators here plant what those paths can get wrong: peaks and larger
neighbours across every strip seam, plateaus at the final cut key on both sides of a cut, NaN counts around K, sigmoids
that differ only in the low key byte, and maps with fewer than K candidates.  Each is checked against the definition
(test_centernet_cpu.definition_decode) and the C oracle (CO.decode), and the strip schedule model confirms the cuts happen.

Float64 reference.  decode64 computes the sigmoid, the 3 x 3 peak test and the order in float64.  The kernel's sigmoid is
logist(x) = 1 / (1 + expf(-x)) in float32 (u = 2^-24):
    expf is within 2 ulp (CUDA) -- a relative error of at most 4u on E = exp(-x); it moves 1 / (1 + E) by a relative
    E / (1 + E) * 4u = (1 - s) 4u.  The sum 1 + E and the division round once each: u each.  A subnormal quotient rounds
    with an absolute error of at most 2^-150 instead.
    bound(s) = s ((1 - s) 4u + 2u) (1 + 8u) + 2^-150.
Cells and classes must equal float64's; each score must lie within bound of the float64 sigmoid.  Where two adjacent ranks of
the float64 order (rank K - 1 against the first rank left out included) differ by a nonzero gap within twice the bound, the
float32 order may swap them: those ranks are excused from the cell check and counted."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import centernet as CO

from test_centernet_cpu import assert_dets, definition_decode, tie_free_heads

U = 2.0 ** -24
LIST_CAP, STRIP_CELLS = 5120, 4096


def strip_rows(W):
    return max(1, STRIP_CELLS // W)


def sigmoid64(heat):
    with np.errstate(over="ignore", invalid="ignore"):
        return 1.0 / (1.0 + np.exp(-np.asarray(heat, np.float64)))


def sigmoid32(heat):
    """the definition's float32 sigmoid (glibc expf)"""
    with np.errstate(over="ignore", invalid="ignore"):
        return (np.float32(1) / (np.float32(1) + np.exp(-np.asarray(heat, np.float32)))).astype(np.float32)


def logist_bound(s):
    s = np.nan_to_num(np.asarray(s, np.float64), nan=0.0)
    return s * ((1 - s) * 4 * U + 2 * U) * (1 + 8 * U) + 2.0 ** -150


def _suppress(s):
    """the 3 x 3 peak test on sigmoids s [C, H, W] (any float type): s where s equals the NaN-propagating max of its clipped
    window, else s * 0 -> the suppressed values, flat"""
    Cn, H, W = s.shape
    p = np.full((Cn, H + 2, W + 2), -np.inf, s.dtype)
    p[:, 1:-1, 1:-1] = s
    m = np.full_like(s, -np.inf)
    for dy in range(3):
        for dx in range(3):
            win = p[:, dy:dy + H, dx:dx + W]
            m = np.where(np.isnan(m) | np.isnan(win), np.nan, np.maximum(m, win))
    with np.errstate(invalid="ignore"):
        return (s * (m == s).astype(s.dtype)).reshape(-1)


def order_of(v):
    """flat indices by NaN first, then descending value, ties to the smaller flat index"""
    flat = np.arange(v.size)
    return np.lexsort((flat, -np.nan_to_num(v, nan=0.0), ~np.isnan(v)))


def boxes_of(order, v, wh, reg, H, W):
    """dets [len(order), 6] for flat indices `order` with scores v[order], boxes in the kernel's float32 arithmetic"""
    HW = H * W
    cell = order % HW
    ys, xs = (cell // W).astype(np.float32), (cell % W).astype(np.float32)
    x = xs + reg[0].reshape(-1)[cell]
    y = ys + reg[1].reshape(-1)[cell]
    hw, hh = wh[0].reshape(-1)[cell] / np.float32(2), wh[1].reshape(-1)[cell] / np.float32(2)
    return np.stack([x - hw, y - hh, x + hw, y + hh, np.asarray(v, np.float32)[order], (order // HW).astype(np.float32)], 1)


def definition_from_sig(s, wh, reg, k):
    """definition_decode with the sigmoids given (float32 [C, H, W]) instead of computed from logits"""
    Cn, H, W = s.shape
    v = _suppress(s)
    return boxes_of(order_of(v)[:k], v, wh, reg, H, W)


def uncertain_peaks(s64):
    """cells whose 3 x 3 peak test could go the other way in float32: a neighbour within twice the bound, not equal"""
    Cn, H, W = s64.shape
    b = logist_bound(s64)
    out = np.zeros(s64.shape, bool)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy == dx == 0:
                continue
            a = s64[:, max(dy, 0):H + min(dy, 0), max(dx, 0):W + min(dx, 0)]
            n = s64[:, max(-dy, 0):H + min(-dy, 0), max(-dx, 0):W + min(-dx, 0)]
            ba = b[:, max(dy, 0):H + min(dy, 0), max(dx, 0):W + min(dx, 0)]
            with np.errstate(invalid="ignore"):
                near = (a != n) & (np.abs(a - n) <= 2 * ba)
            out[:, max(dy, 0):H + min(dy, 0), max(dx, 0):W + min(dx, 0)] |= near
    return out


def decode64(heat, k):
    """-> (order [k + 1 or fewer] flat indices, v64 flat suppressed float64 values, peak-test ambiguities in the top k + 1)"""
    s64 = sigmoid64(heat)
    v = _suppress(s64)
    order = order_of(v)[:k + 1]
    unc = uncertain_peaks(s64).reshape(-1)
    # an ambiguous cell matters only if its sigmoid could reach the top k + 1
    floor = np.nan_to_num(v[order[-1]], nan=np.inf)
    with np.errstate(invalid="ignore"):
        risky = int((unc & ~(sigmoid64(heat).reshape(-1) < floor - 2 * logist_bound(floor))).sum())
    return order, v, risky


def check_f64(dets, heat, wh, reg, k):
    """dets [k, 6] of one image against the float64 reference -> (max |score - f64|, max bound, excused ranks)"""
    Cn, H, W = heat.shape
    order, v, risky = decode64(heat, k)
    assert risky == 0, "the map has peak tests within the float32 error: not a tie-free map"
    want = boxes_of(order[:k], v, wh, reg, H, W)
    vals = v[order]
    b = logist_bound(vals)
    excused = np.zeros(k, bool)
    for r in range(len(order) - 1):
        g = vals[r] - vals[r + 1]
        if g > 0 and g <= 2 * max(b[r], b[r + 1]):
            excused[r] = True
            if r + 1 < k:
                excused[r + 1] = True
    got = np.asarray(dets)
    ok = ~excused
    assert np.array_equal(got[ok][:, [0, 1, 2, 3, 5]], want[ok][:, [0, 1, 2, 3, 5]]), "cells or classes differ from float64"
    sc, ref = got[:, 4].astype(np.float64), vals[:k]
    assert np.array_equal(np.isnan(sc), np.isnan(ref))
    fin = ~np.isnan(ref)
    err = np.abs(sc[fin] - ref[fin])
    lim = np.where(excused[fin], 3, 1) * b[:k][fin]
    assert np.all(err <= lim), float(np.max(err / lim))
    return (float(err.max()) if err.size else 0.0), (float(b[:k][fin].max()) if fin.any() else 0.0), int(excused.sum())


def cut_schedule(heat, k):
    """The peaks kernel's strip and cut schedule for one class map, on the float32 sigmoids of the definition -> (strips
    that start with a cut, the key of the K-th best at the end or None when fewer than k cells are candidates).  Keys as
    cn_key: NaN above all, then the float order of non-negative values."""
    H, W = heat.shape
    v = _suppress(sigmoid32(heat)[None])
    key = np.where(np.isnan(v), np.uint64(1 << 32), v.astype(np.float32).view(np.uint32).astype(np.uint64))
    cand = (v > 0) | np.isnan(v)
    R = strip_rows(W)
    lst, floor, cuts = np.zeros(0, np.uint64), -1, []

    def select(lst):
        o = np.lexsort((np.arange(lst.size), -lst.astype(np.float64)))[:k]
        return lst[np.sort(o)], int(lst[o[-1]])

    for s, y0 in enumerate(range(0, H, R)):
        cells = min(R, H - y0) * W
        if lst.size + cells > LIST_CAP:
            lst, floor = select(lst)
            cuts.append(s)
        i = np.arange(y0 * W, y0 * W + cells)
        add = i[cand[i] & (key[i].astype(np.int64) > floor)]
        lst = np.concatenate([lst, key[add]])
    final = select(lst)[1] if lst.size >= k else None
    return cuts, final


def check_both(dets, heat, wh, reg, k, msg=""):
    """one image's dets against the C oracle and the definition (assert_dets)"""
    assert_dets(dets, CO.decode(heat, wh, reg, k), msg)
    assert_dets(dets, definition_decode(heat, wh, reg, k), msg)


def _boxes(rng, Cn, H, W):
    return rng.uniform(0, 60, (2, H, W)).astype(np.float32), rng.uniform(0, 1, (2, H, W)).astype(np.float32)


# ------------------------------------------------------------------ strip seams ----------------------------------------
def seam_sizes():
    """(W, H): for each W, H with a one-row last strip (R + 1, 3R + 1) and a full last strip (3R); a map narrower than 4
    columns fits one strip at any H <= 1024"""
    out = []
    for W in (1, 3, 64, 100, 1000, 1023, 1024):
        R = strip_rows(W)
        hs = (1024, 2) if R >= 1024 else (R + 1, 3 * R, 3 * R + 1)
        out += [(W, H) for H in hs]
    return out + [(1024, 1), (1024, 2)]


SEAM_KINDS = ("above", "below", "diag_above", "diag_below", "equal")


def seam_heads(seed, Cn, H, W):
    """Tie-free low logits in [-15, -4] with patterns planted across each strip seam (the first row y of every strip but
    the first; a map of one strip gets them at row H // 2), at columns 0 and W - 1 and every 16th column between:
      above       (y - 1, x) larger than (y, x): the cell on the strip's first row is no peak
      below       the mirror: the cell on the previous strip's last row is no peak
      diag_above  (y - 1, x +- 1) larger than (y, x);  diag_below  (y, x +- 1) larger than (y - 1, x)
      equal       (y - 1, x) == (y, x): both peaks (the test is <=)
    Planted logits lie in [0.25, 4), distinct except the equal pairs.  -> heat, wh, reg, must-be-peak and must-not-be-peak
    flat indices."""
    rng = np.random.default_rng(seed)
    heat = rng.permutation(np.linspace(-15.0, -4.0, Cn * H * W)).astype(np.float32).reshape(Cn, H, W)
    R = strip_rows(W)
    seams = list(range(R, H, R)) or ([H // 2] if H >= 2 else [])
    peaks, dead = set(), set()
    cnt = 0
    for c in range(Cn):
        for si, y in enumerate(seams):
            cols = ([0] if si % 2 == 0 else [W - 1]) if W < 8 else sorted({0, W - 1, *range(16, W - 4, 16)})
            for j, x in enumerate(cols):
                kind = SEAM_KINDS[(si + j + c) % 5]
                if W == 1 and kind.startswith("diag"):
                    kind = kind[5:]
                a = np.float32(0.25 + 0.004 * cnt)
                big = np.float32(a + 0.002)
                cnt += 1
                xd = x + 1 if x + 1 < W else x - 1
                cell = {"above": ((y, x), (y - 1, x)), "below": ((y - 1, x), (y, x)),
                        "diag_above": ((y, x), (y - 1, xd)), "diag_below": ((y - 1, x), (y, xd))}
                if kind == "equal":
                    heat[c, y - 1, x] = heat[c, y, x] = a
                    peaks |= {(c * H + y - 1) * W + x, (c * H + y) * W + x}
                    continue
                (ly, lx), (by, bx) = cell[kind]
                heat[c, ly, lx], heat[c, by, bx] = a, big
                dead.add((c * H + ly) * W + lx)
                peaks.add((c * H + by) * W + bx)
    assert cnt * 0.004 < 3.7
    wh, reg = _boxes(rng, Cn, H, W)
    return heat, wh, reg, peaks, dead


def seam_k(H, W, npeaks):
    return min(H * W, npeaks + 20, 1024)


def flat_of(dets, H, W):
    """flat indices c * H * W + y * W + x of dets made with reg = wh = 0 (box corners at the cell)"""
    d = np.asarray(dets)
    return (d[:, 5].astype(np.int64) * H + d[:, 1].astype(np.int64)) * W + d[:, 0].astype(np.int64)


@pytest.mark.parametrize("W,H", seam_sizes(), ids=lambda v: str(v))
def test_seam_generator(W, H):
    """The planted peaks are peaks and the planted losers are not, under the definition, the oracle and float64; every
    planted peak makes the top K and no loser does; no peak test is within the float32 error."""
    heat, wh, reg, peaks, dead = seam_heads(W * 1031 + H, 2, H, W)
    v = _suppress(sigmoid32(heat))
    assert all(v[i] > 0 for i in peaks) and all(v[i] == 0 for i in dead)
    k = seam_k(H, W, len(peaks))
    got = CO.decode(heat, wh, reg, k)
    check_both(got, heat, wh, reg, k, (W, H))
    check_f64(got, heat, wh, reg, k)
    zero = np.zeros_like(wh)
    cells = set(flat_of(CO.decode(heat, zero, zero, k), H, W).tolist())
    assert peaks <= cells and not (dead & cells)


# ------------------------------------------------------------------ cuts -----------------------------------------------
def rising_heads(seed, H=256, W=256):
    """One class, tie-free, each strip's logits above every earlier strip's: every strip brings ~W * R / 9 peaks above any
    cut key, so the list is cut again and again at every K; the K best lie in the last strips."""
    rng = np.random.default_rng(seed)
    R = strip_rows(W)
    g = np.linspace(-15.0, 3.0, H * W).astype(np.float32)
    heat = np.empty((H, W), np.float32)
    for y0 in range(0, H, R):
        n = min(R, H - y0) * W
        heat[y0:y0 + min(R, H - y0)] = rng.permutation(g[y0 * W:y0 * W + n]).reshape(-1, W)
    wh, reg = _boxes(rng, 1, H, W)
    return heat[None], wh, reg


PLATEAU_P = np.float32(0.5)
PLATEAU_ROWS = (17, 145, 225)  # first rows of the plateau blocks: strips 1, 9 and 14 of a 256-wide map


def plateau_heads(seed, k, H=256, W=256):
    """One class: tie-free background logits in [-15, -2] (~455 peaks per strip, so the list is cut), A = k // 3 isolated
    larger logits in [1, 3], and three blocks of the plateau logit 0.5 (every cell a peak) in flat order from rows 17, 145,
    225.  The K best are the A larger cells and the first m = k - A plateau cells: all of block 1 and the first m - b1 of
    block 2, so the final cut key is the plateau's and its kept cells lie on both sides of a cut (for k > 1).
    -> heat [1, H, W], wh, reg, the flat indices of the kept plateau cells."""
    rng = np.random.default_rng(seed)
    heat = rng.permutation(np.linspace(-15.0, -2.0, H * W)).astype(np.float32).reshape(H, W)
    A = k // 3
    m = k - A
    b1 = (m + 1) // 2
    sizes = (b1, m - b1 + max(5, m // 2), 50)
    cells = np.concatenate([np.arange(r * W, r * W + n) for r, n in zip(PLATEAU_ROWS, sizes)])
    heat.reshape(-1)[cells] = PLATEAU_P
    pb = np.pad(heat == PLATEAU_P, 1)
    near = np.zeros((H, W), bool)
    for dy in range(3):
        for dx in range(3):
            near |= pb[dy:dy + H, dx:dx + W]
    lattice = [(y, x) for y in range(2, H - 1, 4) for x in range(2, W - 1, 4) if not near[y, x]]
    pick = rng.choice(len(lattice), A, replace=False)
    for v, p in zip(rng.permutation(np.linspace(1.0, 3.0, A)), pick):
        heat[lattice[p]] = np.float32(v)
    wh, reg = _boxes(rng, 1, H, W)
    return heat[None], wh, reg, cells[:m]


CUT_K = (1, 100, 1024)


@pytest.mark.parametrize("k", CUT_K)
def test_cut_generators(k):
    """rising_heads cuts the list at least 3 times; plateau_heads cuts it between its first two blocks, ends on the plateau
    key, and the K best take the earliest plateau cells; both follow the oracle, the definition and float64."""
    heat, wh, reg = rising_heads(k)
    cuts, _ = cut_schedule(heat[0], k)
    assert len(cuts) >= 3, cuts
    got = CO.decode(heat, wh, reg, k)
    check_both(got, heat, wh, reg, k, k)
    check_f64(got, heat, wh, reg, k)
    heat, wh, reg, kept = plateau_heads(k, k)
    cuts, final = cut_schedule(heat[0], k)
    strip = [r // strip_rows(256) for r in PLATEAU_ROWS]
    assert any(strip[0] < s <= strip[1] for s in cuts), cuts
    assert final == int(sigmoid32(PLATEAU_P).view(np.uint32)), final
    got = CO.decode(heat, wh, reg, k)
    check_both(got, heat, wh, reg, k, k)
    zero = np.zeros_like(wh)
    cells = flat_of(CO.decode(heat, zero, zero, k), 256, 256)
    at_p = cells[CO.decode(heat, zero, zero, k)[:, 4] == sigmoid32(PLATEAU_P)]
    assert np.array_equal(np.sort(at_p), kept)
    if k > 1:
        assert kept[-1] >= PLATEAU_ROWS[1] * 256  # kept plateau cells on both sides of a cut


def nan_counts(k):
    return sorted({0, max(k - 1, 0), k, k + 1, 6000})


def nan_heads(seed, count, H=128, W=128):
    """One class, tie-free logits in [-15, 3] with `count` NaN cells at random positions (a NaN also suppresses its 8
    neighbours)"""
    rng = np.random.default_rng(seed)
    heat, wh, reg = tie_free_heads(seed, 1, 1, H, W)
    heat[0, 0].reshape(-1)[rng.choice(H * W, count, replace=False)] = np.nan
    return heat[0], wh[0], reg[0]


@pytest.mark.parametrize("k", (1, 100, 1024))
def test_nan_generator(k):
    """With more than K NaNs, the final cut key is the NaN key and the K first NaNs in flat order are the answer."""
    for count in nan_counts(k):
        heat, wh, reg = nan_heads(count + k, count)
        got = CO.decode(heat, wh, reg, k)
        check_both(got, heat, wh, reg, k, (k, count))
        if count == 0:
            check_f64(got, heat, wh, reg, k)
        cuts, final = cut_schedule(heat[0], k)
        if count > k:
            assert final == 1 << 32
            assert np.isnan(got[:, 4]).all()
        if count > LIST_CAP:
            assert cuts


def lowbyte_logits():
    """(near-1 logits, near-0.5 logits).  Near 1: x = -ln(j 2^-23), j = 1..40, so E = expf(-x) lies a relative 2^-20 or
    less from j 2^-23: any expf within a few ulp gives 1 + E = 1 + j 2^-23 exactly, and the sigmoids are every other float
    below 1, alike in their top 3 key bytes on every implementation.  Near 0.5: x = i 2^-22, i = -20..20, sigmoids up to four
    floats apart around 0.5, some equal; which floats depends on the expf (the device's are read back)."""
    j = np.arange(1, 41)
    near1 = (-np.log(j * 2.0 ** -23)).astype(np.float32)
    half = (np.arange(-20, 21) * 2.0 ** -22).astype(np.float32)
    return near1, half


def lowbyte_heads(seed, H=256, W=256):
    """One class: background logits far below (tie-free in [-30, -16], so their keys differ in the top byte), the near-1 and
    near-0.5 logits on an isolated lattice, each used three times so that equal low bytes also meet across strips and cuts"""
    rng = np.random.default_rng(seed)
    heat = rng.permutation(np.linspace(-30.0, -16.0, H * W)).astype(np.float32).reshape(H, W)
    near1, half = lowbyte_logits()
    vals = np.concatenate([near1, half, np.float32([1.0, 2.0, -1.0, 6.0])])
    lattice = [(y, x) for y in range(1, H - 1, 3) for x in range(1, W - 1, 3)]
    pick = rng.choice(len(lattice), 3 * vals.size, replace=False)
    for v, p in zip(np.tile(vals, 3), pick):
        heat[lattice[p]] = v
    wh, reg = _boxes(rng, 1, H, W)
    return heat[None], wh, reg


# K within the 129 cells above 0.5 (3 x 40 near 1, then 6, 2, 1 three times each), whose order every expf agrees on
LOWBYTE_ROBUST_K = (1, 20, 41, 60, 100, 120, 129)


def test_lowbyte_generator():
    """the near-1 sigmoids are every other float below 1 in numpy's float32 and in float64 rounded once, and share their top
    three key bytes; the decode follows the oracle and the definition where K stays above 0.5, and the definition on given
    sigmoids equals the definition"""
    near1, half = lowbyte_logits()
    s = sigmoid32(near1)
    assert np.array_equal(s, sigmoid64(near1).astype(np.float32))
    b = s.view(np.uint32)
    assert np.all(np.diff(b.astype(np.int64)) == -2) and len(set((b >> 8).tolist())) == 1
    h = sigmoid32(half).view(np.uint32).astype(np.int64)
    assert np.all(np.diff(h) >= 0) and np.all(np.diff(h) <= 4) and np.unique(h).size >= 35
    heat, wh, reg = lowbyte_heads(1)
    for k in LOWBYTE_ROBUST_K:
        check_both(CO.decode(heat, wh, reg, k), heat, wh, reg, k, k)
    for k in (20, 129, 300, 500):
        assert_dets(definition_from_sig(sigmoid32(heat), wh, reg, k), definition_decode(heat, wh, reg, k))


# ------------------------------------------------------------------ fewer than K candidates ----------------------------
# logits <= -104, and in (-103, -88.8) where expf(-x) overflows (torch.sigmoid's too), give a sigmoid of 0; in
# (-88.7, -87.3) the sigmoid is a positive subnormal, so a candidate
TINY_LOGITS = np.float32([-104.0, -120.0, -95.0, -89.0, -88.0, -87.5])


def sparse_heads(seed, k, npos, where, H=32, W=32):
    """All logits -inf (every cell a zero cell) but npos cells of logit 1 (each a peak, the plateau test being <=) placed
    before the first K zero cells ("before": flat indices 0..npos-1), among them (spread over the first K cells) or after
    them (the last npos cells); "tiny": no such cell, but TINY_LOGITS at random cells"""
    rng = np.random.default_rng(seed)
    HW = H * W
    heat = np.full(HW, -np.inf, np.float32)
    pos = {"before": np.arange(npos), "among": np.linspace(0, k - 1, npos).astype(int) if npos else np.arange(0),
           "after": np.arange(HW - npos, HW), "tiny": np.arange(0)}[where]
    pos = np.unique(pos)
    heat[pos] = np.float32(1.0)
    if where == "tiny":
        heat[rng.choice(HW, 6, replace=False)] = TINY_LOGITS
    wh, reg = _boxes(rng, 1, H, W)
    return heat.reshape(1, H, W), wh, reg


def sparse_cases():
    out = []
    for k in (1, 37, 1024):  # 1024 = H * W
        for npos in sorted({0, 1, k - 1}):
            out += [(k, npos, w) for w in ("before", "among", "after")]
        out.append((k, 0, "tiny"))
    return out


def test_sparse_generator():
    """-104, -120, -95 and -89 give 0 and -88, -87.5 a positive subnormal, in numpy and in torch; the oracle and the
    definition agree on every case, K = H * W included"""
    torch = pytest.importorskip("torch")
    x = TINY_LOGITS
    s = sigmoid32(x)
    assert np.array_equal(s == 0, torch.sigmoid(torch.from_numpy(x)).numpy() == 0)
    assert (s[:4] == 0).all() and (s[4:] > 0).all() and (s[4:] < np.finfo(np.float32).tiny).all()
    for k, npos, where in sparse_cases():
        heat, wh, reg = sparse_heads(k + npos, k, npos, where)
        check_both(CO.decode(heat, wh, reg, k), heat, wh, reg, k, (k, npos, where))


# ------------------------------------------------------------------ select kernel --------------------------------------
SELECT_K = (1, 2, 31, 32, 33, 511, 512, 513, 1000, 1023, 1024)


def class_tie_heads(seed, k, kind, Cn=4, H=32, W=32):
    """Tie-free background in [-15, -3]; "ties": A = k - 2 larger logits spread over the classes, and the logit 0.5 at the
    same cell of every class, so the cut falls inside that 4-way tie and the two smaller classes win; "nan": NaNs at
    cells of classes 1..3 (some the same cell in several classes) and larger logits in class 0"""
    rng = np.random.default_rng(seed)
    heat = rng.permutation(np.linspace(-15.0, -3.0, Cn * H * W)).astype(np.float32).reshape(Cn, H, W)
    lattice = [(y, x) for y in range(2, H - 1, 4) for x in range(2, W - 1, 4)]
    tie = lattice[len(lattice) // 2]
    spots = [p for p in lattice if p != tie]
    if kind == "ties":
        heat[:, tie[0], tie[1]] = np.float32(0.5)
        A = k - 2
        for i, v in enumerate(rng.permutation(np.linspace(1.0, 3.0, A))):
            heat[i % Cn, spots[i // Cn % len(spots)][0], spots[i // Cn % len(spots)][1]] = np.float32(v)
    else:
        for i, p in enumerate(spots[:k // 2]):
            heat[1 + i % 3, p[0], p[1]] = np.nan
            if i % 4 == 0:
                heat[1 + (i + 1) % 3, p[0], p[1]] = np.nan
        heat[0, spots[-1][0], spots[-1][1]] = np.float32(4.0)
    wh, reg = _boxes(rng, Cn, H, W)
    return heat, wh, reg, tie


def test_class_tie_generator():
    for k in (7, 100):
        heat, wh, reg, tie = class_tie_heads(k, k, "ties")
        got = CO.decode(heat, wh, reg, k)
        check_both(got, heat, wh, reg, k, k)
        at = got[got[:, 4] == sigmoid32(np.float32(0.5))]
        assert at[:, 5].tolist() == [0.0, 1.0]
        heat, wh, reg, _ = class_tie_heads(k, k, "nan")
        got = CO.decode(heat, wh, reg, k)
        check_both(got, heat, wh, reg, k, k)
        assert len(set(got[np.isnan(got[:, 4]), 5].tolist())) == 3


def test_select_generators_are_tie_free():
    """the tie-free maps of the select tests, the one-million-candidate one included, have no ambiguous peak test near
    their top K"""
    for Cn, H, W, k, seed in ((3, 48, 48, 1024, 1), (1, 40, 40, 1024, 2), (1024, 32, 32, 1024, 3)):
        heat, wh, reg = tie_free_heads(seed, 1, Cn, H, W)
        assert decode64(heat[0], k)[2] == 0


# ------------------------------------------------------------------ pre-process ----------------------------------------
PRE_NETS = (1, 2, 3, 255, 384, 511, 513, 1024, 2048)


def pre_sizes(net):
    """(w, h) frames for one net: an upscale, a downscale, L == net, L == 2 net (OpenCV's 2x path), 1 x 1, and w == 1 (the
    broadcast column); L = max(w, h, 3)"""
    s = {(max(1, net // 2 - 1), max(1, net // 3)), (net + net // 2 + 1, net // 2 + 1), (1, 1), (1, max(5, net // 2 + 3)),
         (max(1, net // 2), 2 * net)}
    if net >= 3:
        s.add((net, max(1, net - 7)))
    return sorted(s)


def float_fractions_exact(net, L):
    """whether every source coordinate (d + 0.5) L / net - 0.5 of a net-side resize of L samples is the same in float and in
    double: then the float64 resize's fractions do not depend on the precision they are computed in"""
    d = np.arange(net)
    f = (d + 0.5) * (1.0 / (net / L)) - 0.5
    return bool(np.all(f.astype(np.float32).astype(np.float64) == f))


def _cv2_pre(cv2, img, net):
    h, w = img.shape[:2]
    L_ = max(h, w, 3)
    canvas = np.zeros((L_, L_, 3))
    canvas[:h, :w if w > 1 else L_] = img  # a one-pixel-wide frame fills its rows, as numpy broadcasts it
    return ((cv2.resize(canvas, (net, net)) / 255. - 0.5) / 0.5).astype(np.float32).transpose(2, 0, 1)


@pytest.mark.parametrize("net", [n for n in PRE_NETS if n <= 1024])
@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_cv2_at_other_nets(net, ipp):
    """CO.preprocess(img, net) equals cv2.resize of the float64 canvas to net x net, then the normalisation, bit for bit,
    on every frame of pre_sizes whose coordinates are exact in float (pitched rows read the same).  At 512 that is every
    frame; the others are test_preprocess_oracle_differs_from_cv2_on_inexact_coordinates."""
    cv2 = pytest.importorskip("cv2")
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        rng = np.random.default_rng(net)
        for w, h in pre_sizes(net):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            got = CO.preprocess(img, net)
            pitched = np.zeros((h, w + 5, 3), np.uint8)[:, 2:w + 2]
            pitched[...] = img
            assert np.array_equal(CO.preprocess(pitched, net), got)
            if float_fractions_exact(net, max(w, h, 3)):
                assert np.array_equal(got, _cv2_pre(cv2, img, net)), (net, w, h)
    finally:
        cv2.ipp.setUseIPP(old)


@pytest.mark.xfail(strict=True, reason="cv2 4.13's float64 INTER_LINEAR computes its fractions in double where the oracle "
                                       "and the kernel take OpenCV's float geometry; they differ where (d + 0.5) L / net is "
                                       "not exact in float")
@pytest.mark.parametrize("net,w,h", [(384, 191, 128), (255, 1, 1), (513, 300, 300)])
def test_preprocess_oracle_differs_from_cv2_on_inexact_coordinates(net, w, h):
    cv2 = pytest.importorskip("cv2")
    assert not float_fractions_exact(net, max(w, h, 3))
    img = np.random.default_rng(net + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert np.array_equal(CO.preprocess(img, net), _cv2_pre(cv2, img, net))
