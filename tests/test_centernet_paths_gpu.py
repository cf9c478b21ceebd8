"""The CenterNet decode and pre-process (tensorrtx_b200/csrc/centernet.cu) on every path: strip seams, list cuts, NaN counts
around K, keys that differ in the low byte, fewer than K candidates, the select kernel at every K class and at one million
candidates, frame rows past one 64-frame launch, and the pre-process at other nets.

Each decode case is compared with the C oracle and the definition (classes, cells and boxes exact, scores within rtol 2e-6)
and, on tie-free maps, with the float64 reference of tests/test_centernet_paths_cpu.py: cells exact except near-tie ranks,
scores within the bound of logist's float error.  Each float64 case prints its largest error, its bound and the excused
ranks (run with -s).  Every output buffer is sentinel-filled, and the floats around it must keep their sentinel."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import centernet as CO
from tensorrtx_b200 import plugins as P

from test_centernet_cpu import assert_dets, tie_free_heads
from test_centernet_paths_cpu import (CUT_K, LOWBYTE_ROBUST_K, PRE_NETS, SELECT_K, check_both, check_f64, class_tie_heads,
                                      cut_schedule, definition_from_sig, flat_of, logist_bound, lowbyte_heads, nan_counts,
                                      nan_heads, plateau_heads, pre_sizes, rising_heads, seam_heads, seam_k, seam_sizes,
                                      sigmoid32, sigmoid64, sparse_cases, sparse_heads)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = float(np.float32(-3.5e37))  # a float32 value, so that the buffers compare equal to it


def _sentinel(shape):
    """(a tensor of `shape` inside a sentinel-filled buffer one float past its start, the buffer)"""
    n = int(np.prod(shape))
    buf = torch.full((n + 2,), SENT, device=DEV)
    return buf[1:1 + n].view(*shape), buf


def _decode(heat, wh, reg, k, sizes=None, thresh=0.5, net=512, down=4):
    """the device decode of heat [B, C, H, W] into sentinel-filled dets (and rows) -> numpy dets (, rows); every float of
    dets and rows is written, and none around them"""
    B = heat.shape[0]
    t = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV) for a in (heat, wh, reg)]
    dets, dbuf = _sentinel((B, k, 6))
    rows, rbuf = _sentinel((B, 1 + 6 * k)) if sizes is not None else (None, None)
    P.centernet_decode(*t, k, image_sizes=sizes, score_thresh=thresh, net=net, down=down, out=dets, rows_out=rows)
    torch.cuda.synchronize()
    for buf in (dbuf, rbuf):
        if buf is not None:
            assert buf[0].item() == SENT and buf[-1].item() == SENT
            assert not (buf[1:-1] == SENT).any()
    return dets.cpu().numpy() if rows is None else (dets.cpu().numpy(), rows.cpu().numpy())


def _f64(tag, dets, heat, wh, reg, k):
    e, b, x = check_f64(dets, heat, wh, reg, k)
    print(f"{tag}: max |GPU - f64| {e:.3e}, bound {b:.3e}, {x} near-tie ranks excused")


# ------------------------------------------------------------------ strip seams ----------------------------------------
@pytest.mark.parametrize("W,H", seam_sizes(), ids=lambda v: str(v))
def test_strip_seams(W, H):
    """Larger neighbours straight and diagonally across every seam, their mirrors and equal pairs, at columns 0, W - 1 and
    between: every planted peak is found, no planted loser is, and the dets follow all three references."""
    heat, wh, reg, peaks, dead = seam_heads(W * 1031 + H, 2, H, W)
    k = seam_k(H, W, len(peaks))
    got = _decode(heat[None], wh[None], reg[None], k)[0]
    check_both(got, heat, wh, reg, k, (W, H))
    _f64(f"seams W{W} H{H} K{k}", got, heat, wh, reg, k)
    zero = np.zeros_like(wh)
    cells = set(flat_of(_decode(heat[None], zero[None], zero[None], k)[0], H, W).tolist())
    assert peaks <= cells and not (dead & cells)


# ------------------------------------------------------------------ cuts -----------------------------------------------
@pytest.mark.parametrize("k", CUT_K)
def test_cuts_on_rising_strips(k):
    """Every strip beats the last, so the list is cut at least 3 times (the schedule model counts them)."""
    heat, wh, reg = rising_heads(k)
    assert len(cut_schedule(heat[0], k)[0]) >= 3
    got = _decode(heat[None], wh[None], reg[None], k)[0]
    check_both(got, heat, wh, reg, k, k)
    _f64(f"rising K{k}", got, heat, wh, reg, k)


@pytest.mark.parametrize("k", CUT_K)
def test_cut_key_plateau_on_both_sides_of_a_cut(k):
    """The final cut key is a plateau's, with plateau cells before and after a cut: the kept ones are the earliest in flat
    order."""
    heat, wh, reg, kept = plateau_heads(k, k)
    got = _decode(heat[None], wh[None], reg[None], k)[0]
    check_both(got, heat, wh, reg, k, k)
    zero = np.zeros_like(wh)
    z = _decode(heat[None], zero[None], zero[None], k)[0]
    at_p = flat_of(z, 256, 256)[z[:, 4] == z[-1, 4]]
    assert np.array_equal(np.sort(at_p), kept)


@pytest.mark.parametrize("k", CUT_K)
def test_nan_counts_around_k(k):
    """0, K - 1, K, K + 1 and 6000 (> 5120, the list's capacity) NaN cells: the first K NaNs in flat order win once there
    are more than K, and the cut key is then the NaN key."""
    for count in nan_counts(k):
        heat, wh, reg = nan_heads(count + k, count)
        got = _decode(heat[None], wh[None], reg[None], k)[0]
        check_both(got, heat, wh, reg, k, (k, count))
        if count == 0:
            _f64(f"nan K{k} count 0", got, heat, wh, reg, k)
        if count > k:
            assert np.isnan(got[:, 4]).all()


def test_keys_that_differ_in_the_low_byte():
    """Sigmoids every other float below 1 and one to four floats apart around 0.5, each three times, among keys that
    differ in the top byte.  The device's own sigmoids of the planted cells are read back (reg = wh = 0 put each box at its
    cell); every K must then equal the definition on those sigmoids bit for bit, and where K stays above 0.5 also the oracle.
    The near-1 sigmoids must equal numpy's bit for bit; all lie within the float64 bound."""
    heat, wh, reg = lowbyte_heads(1)
    _, H, W = heat.shape
    zero = np.zeros_like(wh)
    probe = _decode(heat[None], zero[None], zero[None], 255)[0]
    cells = flat_of(probe, H, W)
    s_dev = sigmoid32(heat).reshape(-1)
    s_dev[cells] = probe[:, 4]
    s64 = sigmoid64(heat).reshape(-1)[cells]
    err = np.abs(probe[:, 4].astype(np.float64) - s64)
    assert np.all(err <= logist_bound(s64))
    near1 = s64 > 0.9999
    assert np.array_equal(probe[near1, 4], sigmoid32(heat).reshape(-1)[cells][near1])
    diff = int((probe[:, 4] != sigmoid32(heat).reshape(-1)[cells]).sum())
    print(f"low byte: max |GPU - f64| {err.max():.3e}, bound {logist_bound(s64).max():.3e}, {diff} of 255 planted sigmoids "
          f"differ from numpy's")
    s_dev = s_dev.reshape(heat.shape)
    for k in (1, 20, 41, 60, 100, 120, 129, 150, 200, 254, 255):
        got = _decode(heat[None], wh[None], reg[None], k)[0]
        assert np.array_equal(got, definition_from_sig(s_dev, wh, reg, k), equal_nan=True), k
        if k in LOWBYTE_ROBUST_K:
            check_both(got, heat, wh, reg, k, k)


# ------------------------------------------------------------------ fewer than K candidates ----------------------------
@pytest.mark.parametrize("k,npos,where", sparse_cases(), ids=lambda v: str(v))
def test_fewer_than_k_candidates(k, npos, where):
    """0, 1 and K - 1 candidates before, among and after the first K zero cells, K = H * W, and logits whose sigmoid is 0
    or a positive subnormal: the zero-cell merge."""
    heat, wh, reg = sparse_heads(k + npos, k, npos, where)
    got = _decode(heat[None], wh[None], reg[None], k)[0]
    check_both(got, heat, wh, reg, k, (k, npos, where))


# ------------------------------------------------------------------ select kernel --------------------------------------
@pytest.mark.parametrize("k", SELECT_K)
def test_select_every_k_class(k):
    """K around the warp, 512 and the bitonic sort's power-of-two padding, up to 1024, on two images."""
    heat, wh, reg = tie_free_heads(k, 2, 3, 48, 48)
    got = _decode(heat, wh, reg, k)
    for b in range(2):
        check_both(got[b], heat[b], wh[b], reg[b], k, (k, b))
        _f64(f"select K{k} b{b}", got[b], heat[b], wh[b], reg[b], k)


@pytest.mark.parametrize("k", (1, 100, 1024))
def test_select_one_class(k):
    """C = 1: the select kernel's cn_select takes all n = K candidates."""
    heat, wh, reg = tie_free_heads(2, 1, 1, 40, 40)
    got = _decode(heat, wh, reg, k)[0]
    check_both(got, heat[0], wh[0], reg[0], k, k)
    _f64(f"one class K{k}", got, heat[0], wh[0], reg[0], k)


def test_select_one_million_candidates():
    """C = 1024 classes of 32 x 32 at K = 1024: the select kernel takes the best 1024 of 1 048 576 candidates (the C oracle
    and float64; the numpy definition is left out for time)."""
    k = 1024
    heat, wh, reg = tie_free_heads(3, 1, 1024, 32, 32)
    got = _decode(heat, wh, reg, k)[0]
    assert_dets(got, CO.decode(heat[0], wh[0], reg[0], k))
    _f64("one million", got, heat[0], wh[0], reg[0], k)


@pytest.mark.parametrize("kind", ("ties", "nan"))
@pytest.mark.parametrize("k", (7, 100))
def test_select_ties_and_nans_across_classes(kind, k):
    """An equal value at the same cell of four classes, cut inside the tie: the smaller classes win.  NaNs over three
    classes."""
    heat, wh, reg, _ = class_tie_heads(k, k, kind)
    got = _decode(heat[None], wh[None], reg[None], k)[0]
    check_both(got, heat, wh, reg, k, (kind, k))
    if kind == "ties":
        assert got[got[:, 4] == sigmoid32(np.float32(0.5)), 5].tolist() == [0.0, 1.0]


# ------------------------------------------------------------------ frame rows -----------------------------------------
NET_DOWN = ((384, 2), (1024, 8), (640, 4))
THRESH = ("0.5", "0", "-1", "1", "score")


def _frame_sizes(B, seed):
    """B distinct (w, h): 1 x 1, 2 x 1 (L = 3), portrait frames, a 4000-pixel-wide frame, the rest random"""
    rng = np.random.default_rng(seed)
    sizes = [(1, 1), (2, 1), (300, 1000), (4000, 300), (1, 9), (720, 1280)]
    seen = set(sizes)
    while len(sizes) < B:
        s = (int(rng.integers(1, 2000)), int(rng.integers(1, 2000)))
        if s not in seen:
            seen.add(s)
            sizes.append(s)
    return sizes[:B]


def _frame_heads(B, seed):
    """small tie-free maps with a few NaN cells in each frame, and one saturated cell (score exactly 1) in every third"""
    heat, wh, reg = tie_free_heads(seed, B, 2, 16, 16)
    for b in range(B):
        heat[b, b % 2, 3 + b % 5, 4] = np.nan
        heat[b, 1, 12, 2 + b % 7] = np.nan
        if b % 3 == 0:
            heat[b, 0, 9, 9] = 40.0
    return heat, wh, reg


@pytest.mark.parametrize("thresh", THRESH)
@pytest.mark.parametrize("B", (63, 64, 65, 130))
def test_frame_rows_past_one_launch(B, thresh):
    """Rows of B frames of distinct sizes, over one, two or three 64-frame launches, at score_thresh 0.5, 0, -1, 1 and a
    value equal to a score, with NaN scores present, at (net, down) other than (512, 4): equal bit for bit to CO.rows of
    the device's own dets, zeros past the count (over the sentinel)."""
    k = 40
    net, down = NET_DOWN[(B + THRESH.index(thresh)) % len(NET_DOWN)]
    sizes = _frame_sizes(B, B)
    heat, wh, reg = _frame_heads(B, B + 1)
    if thresh == "score":
        t = float(_decode(heat, wh, reg, k)[0, 9, 4])
        assert t == t and t > 0
    else:
        t = float(thresh)
    dets, rows = _decode(heat, wh, reg, k, sizes, t, net, down)
    for b in range(B):
        if b % 16 == 0:
            check_both(dets[b], heat[b], wh[b], reg[b], k, b)
        want = CO.rows(dets[b], *sizes[b], down=down, net=net, thresh=np.float32(t))
        assert np.array_equal(rows[b], want), (b, sizes[b])


def test_frames_130_equal_single_frame_calls():
    """The dets and rows of a 130-frame call equal 130 one-frame calls, frame by frame."""
    B, k, net, down = 130, 40, 384, 2
    sizes = _frame_sizes(B, 7)
    heat, wh, reg = _frame_heads(B, 8)
    dets, rows = _decode(heat, wh, reg, k, sizes, 0.5, net, down)
    for b in range(B):
        d1, r1 = _decode(heat[b:b + 1], wh[b:b + 1], reg[b:b + 1], k, sizes[b:b + 1], 0.5, net, down)
        assert np.array_equal(dets[b], d1[0], equal_nan=True), b
        assert np.array_equal(rows[b], r1[0]), b


# ------------------------------------------------------------------ pre-process ----------------------------------------
def _frames(rng, sizes, pitched):
    """u8 BGR frames on the device; frame i is pitched (5 spare pixels per row) behind an odd base where pitched(i)"""
    hosts, devs = [], []
    for i, (w, h) in enumerate(sizes):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        pad, off = (5, 3) if pitched(i) else (0, 0)
        flat = torch.zeros(h * (w + pad) * 3 + off, dtype=torch.uint8, device=DEV)
        view = flat[off:].view(h, w + pad, 3)[:, :w]
        view.copy_(torch.from_numpy(img))
        hosts.append(img)
        devs.append(view)
    return hosts, devs


def _preprocess(devs, net):
    out, buf = _sentinel((len(devs), 3, net, net))
    P.centernet_preprocess(devs, out=out, net=net)
    torch.cuda.synchronize()
    assert buf[0].item() == SENT and buf[-1].item() == SENT
    return out.cpu().numpy()


@pytest.mark.parametrize("net", PRE_NETS)
def test_preprocess_other_nets(net):
    """An upscale, a downscale, L == net, L == 2 net, 1 x 1 and a one-pixel-wide frame, every other one pitched behind an
    odd base: bit for bit with CO.preprocess(img, net), into an output one float past its buffer's start."""
    rng = np.random.default_rng(net)
    sizes = pre_sizes(net)
    hosts, devs = _frames(rng, sizes, lambda i: i % 2 == 1)
    got = _preprocess(devs, net)
    for i, img in enumerate(hosts):
        assert np.array_equal(got[i], CO.preprocess(img, net)), (net, sizes[i])


def test_preprocess_65_frames_at_384():
    """65 mixed frames at net 384 take two launches; each equals the oracle."""
    rng = np.random.default_rng(65)
    sizes = [(int(w), int(h)) for w, h in rng.integers(1, 900, (65, 2))]
    sizes[63], sizes[64] = (1, 700), (768, 384)
    hosts, devs = _frames(rng, sizes, lambda i: i % 3 == 0)
    got = _preprocess(devs, 384)
    for i, img in enumerate(hosts):
        assert np.array_equal(got[i], CO.preprocess(img, 384)), (i, sizes[i])
