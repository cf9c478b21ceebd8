"""RefineDet on the device: trtx_refinedet_postprocess_enqueue against the reference's own arithmetic -- the line-by-line
transcription of refinedet/refinedet.cpp:600-791 in oracle/refinedet.py run on CUDA, i.e. the same ATen kernels and CUDA's
double exp -- bit for bit, and trtx_refinedet_preprocess_enqueue and the frame rows against the CPU oracle
(oracle/refinedet_oracle.c, pinned to cv2 and to the transcription by tests/test_refinedet_cpu.py)."""

import numpy as np
import pytest
import torch

from oracle import refinedet as RO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
NET, PN, CN = RO.NET, RO.num_priors(), RO.NUM_CLASSES
SENTINEL = 0x7FBADBAD  # a quiet NaN with a payload
FRAMES = [(1920, 1080), (1280, 720), (320, 320), (1, 1), (2, 2), (17, 4000), (4000, 17), (731, 1299), (640, 480)]


def _dev_heads(h, dev):
    return [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in h]


def _want(h, b, dev, max_det=None, **kw):
    """The transcription on CUDA for frame b, in the device's dets layout."""
    res = RO.reference_postprocess(*[x[b] for x in h], device=dev, **kw)
    return RO.as_dets(res, (CN - 1) * RO.TOP_K if max_det is None else max_det)


def _sentinel_call(h, dev, sizes=None, **kw):
    """The post-process into outputs filled with a NaN of a payload the device never writes, with such a sentinel on each
    side; returns the host outputs after checking that the sentinels are untouched and every element was written."""
    B = h[0].shape[0]
    max_det = kw.get("max_det") or (CN - 1) * kw.get("top_k", RO.TOP_K)
    n = B * (1 + 6 * max_det)
    big = torch.full((2, n + 2), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)
    out, rows = big[0, 1:1 + n].view(B, -1), big[1, 1:1 + n].view(B, -1)
    P.refinedet_postprocess(*_dev_heads(h, dev), sizes, out=out, rows_out=rows if sizes else None, **kw)
    bits = big.view(torch.int32).cpu().numpy()
    assert (bits[:, 0] == SENTINEL).all() and (bits[:, -1] == SENTINEL).all()
    assert not (bits[0, 1:1 + n] == SENTINEL).any()
    if sizes:
        assert not (bits[1, 1:1 + n] == SENTINEL).any()
    got = big.cpu().numpy()
    return got[0, 1:1 + n].reshape(B, -1), got[1, 1:1 + n].reshape(B, -1)


# ------------------------------------------------------------------ post-process vs the CUDA transcription --------------
@pytest.mark.parametrize("B,objects,check", [(1, 50, (0,)), (7, 50, range(7)), (70, 8, (0, 1, 33, 63, 64, 69))])
def test_postprocess_equals_cuda_transcription(dev, B, objects, check):
    """Tie-free seeded heads with planted objects per class, on 1, 7 and 70 frames (the rows take two launches), equal the
    reference's libtorch arithmetic bit for bit, rows past the count zeroed; the frame rows equal the driver loop over
    them for frames of mixed sizes."""
    h = RO.heads(B, seed=10 + B, objects=objects)
    sizes = [FRAMES[b % len(FRAMES)] for b in range(B)]
    dets, rows = _sentinel_call(h, dev, sizes)
    for b in check:
        want = _want(h, b, dev)
        assert want[0] > 0
        assert np.array_equal(dets[b], want), b
        assert np.array_equal(rows[b], RO.rows(want, *sizes[b])), (b, sizes[b])
    for b in range(B):
        assert np.array_equal(rows[b], RO.rows(dets[b], *sizes[b])), b


def test_dense_classes_top_k_cut_and_max_det(dev):
    """More than 1000 candidates in classes 1 and 2 (the top_k cut), and max_det truncation of the concatenated rows."""
    h = RO.heads(2, seed=5, objects=40, dense=2500)
    assert ((h[3][0, :, 1] > np.float32(0.01)) & (h[1][0, :, 1] > np.float32(0.01))).sum() > 1000
    dets, _ = _sentinel_call(h, dev)
    for b in range(2):
        assert np.array_equal(dets[b], _want(h, b, dev)), b
    for max_det in (1, 100, 1500):
        dets, rows = _sentinel_call(h, dev, [(1280, 720), (333, 777)], max_det=max_det)
        for b, wh in enumerate([(1280, 720), (333, 777)]):
            want = _want(h, b, dev, max_det=max_det)
            assert want[0] == max_det
            assert np.array_equal(dets[b], want), (b, max_det)
            assert np.array_equal(rows[b], RO.rows(want, *wh)), (b, max_det)


def test_empty_frames(dev):
    """A frame with no score above the threshold and a frame where the ARM filter removes every prior give no rows; the
    frame between them is unaffected."""
    h = list(RO.heads(3, seed=8, objects=20))
    h[3][0] = np.float32(0.005)
    h[1][2, :, 1] = np.float32(0.001)
    dets, rows = _sentinel_call(h, dev, [(640, 480)] * 3)
    assert dets[0, 0] == 0 and dets[2, 0] == 0 and (dets[[0, 2]] == 0).all() and (rows[[0, 2]] == 0).all()
    assert np.array_equal(dets[1], _want(h, 1, dev))


@pytest.mark.parametrize("head", ["arm_loc", "arm_conf", "odm_loc", "odm_conf"])
def test_nan_and_inf_in_each_head(dev, head):
    """NaN, +inf and -inf (and logits whose exp overflows the float range) in one head, at candidates of several classes,
    some of them the class's highest score, follow the ATen ops: NaN corners, NaN IoUs that suppress, NaN or inf scores
    that the ARM filter turns into NaN, an inf score ranked first; the frame rows convert NaN and inf to INT_MIN and
    RoiCorrect repairs them."""
    h = list(RO.heads(2, seed=21, objects=30))
    k = ("arm_loc", "arm_conf", "odm_loc", "odm_conf").index(head)
    rng = np.random.default_rng(99)
    for b in range(2):
        for c in (1, 5, 24):
            cand = np.flatnonzero(h[3][b, :, c] > 0.3)
            top = cand[np.argmax(h[3][b, cand, c])]
            ps = [top] + rng.choice(cand[cand != top], 6, replace=False).tolist()
            vals = [np.nan, np.inf, -np.inf, np.nan, 500.0, -500.0, np.inf]
            if k == 3:  # one +inf score per class, the highest: no tie
                vals = [np.inf, np.nan, -np.inf, np.nan, 5.0, -5.0, np.nan]
            for p, v in zip(ps, vals):
                if k == 3:
                    h[3][b, p, c] = v
                elif k == 1:
                    h[1][b, p, 1] = v
                else:
                    h[k][b, p, rng.integers(0, 4)] = v
    sizes = [(1280, 720), (97, 1001)]
    dets, rows = _sentinel_call(h, dev, sizes)
    for b in range(2):
        want = _want(h, b, dev)
        assert np.array_equal(dets[b], want, equal_nan=True), (head, b)
        assert np.array_equal(rows[b], RO.rows(want, *sizes[b])), (head, b)


def test_tie_order_lower_prior_first(dev):
    """Equal scores rank by prior index, at the top_k cut too: with zero offsets (boxes are the priors, exp(0) = 1) the
    device equals the oracle, which sorts by (score descending, prior ascending), bit for bit."""
    B = 2
    arm_loc = np.zeros((B, PN, 4), np.float32)
    odm_loc = np.zeros((B, PN, 4), np.float32)
    arm_conf = np.full((B, PN, 2), 0.5, np.float32)
    rng = np.random.default_rng(4)
    odm_conf = np.zeros((B, PN, CN), np.float32)
    odm_conf[..., 1:] = rng.choice(np.array([0.005, 0.2, 0.5, 0.7], np.float32), (B, PN, CN - 1))
    h = (arm_loc, arm_conf, odm_loc, odm_conf)
    for top_k in (10, 333, 1000):
        dets, _ = _sentinel_call(h, dev, top_k=top_k, max_det=3000)
        for b in range(B):
            want = RO.postprocess(*[x[b] for x in h], top_k=top_k, max_det=3000)
            assert np.array_equal(dets[b], want), (top_k, b)
    assert dets[0, 0] > 0


def test_rejected_calls_write_nothing(dev):
    h = _dev_heads(RO.heads(2, seed=2, objects=5), dev)
    out = torch.full((2, 1 + 6 * 24000), 3.0, dtype=torch.float32, device=dev)
    rows = torch.full_like(out, 4.0)
    for kw, sizes, err in (({"nms_thresh": float("nan")}, None, "INVALID"), ({"top_k": 1025, "max_det": 24000}, None,
                                                                               "UNSUPPORTED"),
                           ({}, [(64, 48), (0, 48)], "INVALID"), ({}, [(64, 48), (64, (1 << 24) + 1)], "UNSUPPORTED")):
        with pytest.raises(L.TrtxError, match=err):
            P.refinedet_postprocess(*h, sizes, out=out, rows_out=rows if sizes else None, **kw)
    ws = torch.empty(16, dtype=torch.uint8, device=dev)
    with pytest.raises(L.TrtxError, match="WORKSPACE"):
        P.refinedet_postprocess(*h, out=out, workspace=ws)
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (rows == 4.0).all()


# ------------------------------------------------------------------ pre-process -----------------------------------------
def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra + 1 bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def test_preprocess_equals_oracle(dev):
    """Pitched frames at odd bases, a frame cropped out of a larger one, 1080p, 1 x 1 and other sizes in one call, into a
    NaN-filled dst with sentinels, equal the oracle bit for bit; the frames are not written."""
    rng = np.random.default_rng(1)
    frames = [_frame(rng, w, h, dev, 3 * (i % 4)) for i, (w, h) in enumerate(FRAMES)]
    big = torch.from_numpy(rng.integers(0, 256, (900, 1700, 3), dtype=np.uint8)).to(dev)
    frames.append(big[123:123 + 611, 77:77 + 1001])  # cropped: pitch 3 * 1700, base inside the row
    before = [_host(f) for f in frames]
    n = len(frames) * 3 * NET * NET
    buf = torch.full((n + 2,), float("nan"), dtype=torch.float32, device=dev)
    P.refinedet_preprocess(frames, out=buf[1:1 + n].view(len(frames), 3, NET, NET))
    got = buf.cpu().numpy()
    assert np.isnan(got[0]) and np.isnan(got[-1])
    planes = got[1:1 + n].reshape(-1, 3, NET, NET)
    for i, f in enumerate(frames):
        assert np.array_equal(planes[i], RO.preprocess(before[i])), i
        assert np.array_equal(_host(f), before[i])


def test_preprocess_70_frames_other_net(dev):
    """70 frames take two launches; another square side."""
    rng = np.random.default_rng(2)
    frames = [_frame(rng, 40 + 29 * i, 30 + 17 * i, dev, i % 5) for i in range(70)]
    for net in (320, 512):
        out = P.refinedet_preprocess(frames, net=net).cpu().numpy()
        for i in (0, 1, 63, 64, 69):
            assert np.array_equal(out[i], RO.preprocess(_host(frames[i]), net)), (net, i)


# ------------------------------------------------------------------ end to end -------------------------------------------
def test_graph_capture_and_replay(dev):
    """Both calls captured in one CUDA graph and replayed on new frames and new heads give the new results."""
    B = 3
    rng = np.random.default_rng(9)
    sizes = [(1920, 1080), (1280, 720), (810, 1080)]
    frames = [_frame(rng, w, h, dev, 7) for w, h in sizes]
    h0 = RO.heads(B, seed=30, objects=20)
    hd = _dev_heads(h0, dev)
    inp = torch.empty((B, 3, NET, NET), dtype=torch.float32, device=dev)
    dets = torch.empty((B, 1 + 6 * 24000), dtype=torch.float32, device=dev)
    rows = torch.empty_like(dets)
    ws = torch.empty(int(L.load().trtx_refinedet_workspace_size(
        L.RefinedetParams(NET, CN, 0.01, 0.01, 0.45, 1000, 24000, 0.2), B)), dtype=torch.uint8, device=dev)
    P.refinedet_preprocess(frames, out=inp)
    P.refinedet_postprocess(*hd, sizes, workspace=ws, out=dets, rows_out=rows)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.refinedet_preprocess(frames, out=inp)
        P.refinedet_postprocess(*hd, sizes, workspace=ws, out=dets, rows_out=rows)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    h1 = RO.heads(B, seed=31, objects=20)
    for t, x in zip(hd, h1):
        t.copy_(torch.from_numpy(x))
    g.replay()
    torch.cuda.synchronize()
    pre, d, r = inp.cpu().numpy(), dets.cpu().numpy(), rows.cpu().numpy()
    for b in range(B):
        assert np.array_equal(pre[b], RO.preprocess(_host(frames[b])))
        want = _want(h1, b, dev)
        assert np.array_equal(d[b], want), b
        assert np.array_equal(r[b], RO.rows(want, *sizes[b])), b
