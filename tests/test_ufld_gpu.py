"""UFLD on the device: trtx_ufld_preprocess_enqueue and trtx_ufld_postprocess_enqueue against the CPU oracle
(oracle/ufld_oracle.c, pinned to cv2, to the driver's own argmax and softmax_mul and to its loop by tests/test_ufld_cpu.py),
bit for bit."""

import numpy as np
import pytest
import torch

from oracle import ufld as UO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
NET_W, NET_H = UO.NET_W, UO.NET_H
MIXED = [(1920, 1080), (1280, 720), (800, 288), (1600, 576), (640, 480), (3840, 2160), (1, 1), (1, 300), (300, 1),
         (17, 4000), (731, 1299)]
TUSIMPLE = np.array(UO.TUSIMPLE_ROW_ANCHOR, np.int32)


def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra + 1 bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def _probs(B, shape=UO.SHAPE, seed=0):
    """[B, C, H, W]: frame 0 the edge cells in its first 16 rows, the others lane logits of different seeds."""
    Cn, H, W = shape
    p = np.stack([UO.lane_prob(Cn, H, W, seed=seed + b) for b in range(B)])
    p[0, :, :16] = UO.edge_cells(Cn, seed=seed)
    return p


def _post_check(prob, sizes, got, anchors=TUSIMPLE, **kw):
    for b, (w, h) in enumerate(sizes):
        want = UO.postprocess(prob[b], w, h, anchors, **kw)
        assert np.array_equal(got[b], want), (b, w, h)


# ------------------------------------------------------------------ pre-process ------------------------------------------
def test_preprocess_mixed_sizes_equals_oracle(dev):
    """One call over frames of mixed sizes (up- and downscaling, the identity, the exact 2x downscale, 1 x 1, 1 x N, N x 1,
    tall frames), pitch > 3 * width and odd bases, into a dst that is only 4-byte aligned, equals the oracle bit for bit;
    nothing around the output is written, and the frames are not."""
    rng = np.random.default_rng(1)
    frames = [_frame(rng, w, h, dev, 13 + 3 * (i % 3)) for i, (w, h) in enumerate(MIXED)]
    before = [_host(f) for f in frames]
    n = len(frames) * 3 * NET_H * NET_W
    big = torch.full((n + 8,), -7.0, dtype=torch.float32, device=dev)
    P.ufld_preprocess(frames, out=big[1:1 + n].view(len(frames), 3, NET_H, NET_W))
    got = big.cpu().numpy()
    for i, f in enumerate(frames):
        assert np.array_equal(got[1:1 + n].reshape(-1, 3, NET_H, NET_W)[i], UO.preprocess(before[i])), MIXED[i]
        assert np.array_equal(_host(f), before[i])
    assert got[0] == -7.0 and (got[1 + n:] == -7.0).all()


def test_preprocess_other_net_and_all_bytes(dev):
    """Another net size (odd width, rows not a multiple of the band) and a frame holding every byte value in every channel."""
    rng = np.random.default_rng(4)
    allb = torch.from_numpy(np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(16, 16, 3).copy()).to(dev)
    frames = [allb, _frame(rng, 999, 555, dev, 2)]
    out = P.ufld_preprocess(frames, net_w=321, net_h=243).cpu().numpy()
    for i, f in enumerate(frames):
        assert np.array_equal(out[i], UO.preprocess(_host(f), 321, 243)), i


def test_preprocess_70_frames_graph_replay(dev):
    """70 frames take two launches; the call captured in a CUDA graph and replayed on new frame contents gives the oracle's
    planes for those."""
    rng = np.random.default_rng(2)
    sizes = [(64 + 37 * i, 48 + 23 * i) for i in range(70)]
    frames = [_frame(rng, w, h, dev, i % 5) for i, (w, h) in enumerate(sizes)]
    out = torch.empty((70, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.ufld_preprocess(frames, out=out)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    g.replay()
    torch.cuda.synchronize()
    for i in (0, 1, 63, 64, 69):
        assert np.array_equal(out[i].cpu().numpy(), UO.preprocess(_host(frames[i]))), i


# ------------------------------------------------------------------ post-process -----------------------------------------
def test_postprocess_edge_cells_and_lanes(dev):
    """The edge cells (ties, the truncation quirk, NaN, +-inf, exp overflow and underflow, max_ind -1, "no lane" winners,
    values above the int range) and lanes with many, 3, 2 and no non-zero rows and a NaN expectation, on frames of mixed
    sizes and at the driver's 1280 x 720, equal the oracle; rows past the count are written as zeros over a sentinel."""
    B = 8
    prob = _probs(B)
    pd = torch.from_numpy(prob).to(dev)
    for sizes in (MIXED[:B], None):
        out = torch.full((B, 1 + 56 * 4 * 3), 9.0, dtype=torch.float32, device=dev)
        P.ufld_postprocess(pd, sizes, out=out)
        rows = out.cpu().numpy()
        _post_check(prob, sizes or [(1280, 720)] * B, rows)
        assert rows[:, 0].min() > 0
        lanes = set(rows[1, 1:1 + 3 * int(rows[1, 0])].reshape(-1, 3)[:, 2].tolist())
        assert lanes == {0.0, 1.0}, lanes


@pytest.mark.parametrize("shape", [(101, 56, 4), (201, 18, 4), (2, 3, 5), (51, 32, 32), (238, 56, 4)])
def test_postprocess_other_shapes_and_70_frames(dev, shape):
    """CULane's C = 201, H = 18, the smallest C, H * W = 1024 threads and (C - 1) * H * W at the shared-memory bound, with
    other anchors, col_sample_w and net sizes, on 1 and 70 frames of mixed sizes (two launches)."""
    Cn, H, W = shape
    anchors = np.arange(H, dtype=np.int32) * 7 + 3
    for B in (1, 70):
        rng = np.random.default_rng(100 + Cn + B)
        prob = rng.normal(0, 2, (B, Cn, H, W)).astype(np.float32)
        prob[:, Cn - 1] += rng.choice([-6.0, 6.0], (B, H, W)).astype(np.float32)
        sizes = [(17 + 61 * b, 9 + 37 * b) for b in range(B)]
        out = torch.full((B, 1 + H * W * 3), 9.0, dtype=torch.float32, device=dev)
        P.ufld_postprocess(torch.from_numpy(prob).to(dev), sizes, row_anchor=anchors.tolist(), col_sample_w=5, net_w=640,
                           net_h=200, out=out)
        _post_check(prob, sizes, out.cpu().numpy(), anchors, net_w=640, net_h=200, col_sample_w=5)


def test_rejected_calls_write_nothing(dev):
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 320, 180, dev, 5), _frame(rng, 64, 48, dev, 0)]
    out = torch.full((2, 3, 64, 4758), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.ufld_preprocess(frames, out=out, net_w=4758, net_h=64)
    descs = P._image_descs(frames)
    descs[1].pitch = 3 * 64 - 1
    assert L.load().trtx_ufld_preprocess_enqueue(descs, 2, 4758, 64, out.data_ptr(), None) == L.ERR_INVALID
    prob = torch.from_numpy(_probs(2)).to(dev)
    rows = torch.full((2, 1 + 56 * 4 * 3), 9.0, dtype=torch.float32, device=dev)
    for kw, sizes, err in (({"col_sample_w": 0}, [(64, 48)] * 2, "INVALID"), ({}, [(64, 48), (64, 0)], "INVALID"),
                           ({"net_h": 0}, [(64, 48)] * 2, "INVALID"), ({}, [(64, 48), (64, (1 << 24) + 1)], "UNSUPPORTED"),
                           ({"row_anchor": [64] * 55 + [50_000_000]}, [(64, 48)] * 2, "UNSUPPORTED")):
        with pytest.raises(L.TrtxError, match=err):
            P.ufld_postprocess(prob, sizes, out=rows, **kw)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):  # (C - 1) * H * W above the shared-memory bound
        P.ufld_postprocess(torch.zeros((2, 239, 56, 4), device=dev), [(64, 48)] * 2, out=rows)
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (rows == 9.0).all()


# ------------------------------------------------------------------ end to end -------------------------------------------
def test_end_to_end_chain_and_graph_replay(dev):
    """Frames -> pre-process, and a stand-in engine output `prob` -> post-process, captured together in a CUDA graph and
    replayed on new frames and a new prob, give the oracle's planes and rows for those."""
    B = 3
    rng = np.random.default_rng(9)
    sizes = [(1920, 1080), (1280, 720), (810, 1080)]
    frames = [_frame(rng, w, h, dev, 7) for w, h in sizes]
    pd = torch.from_numpy(_probs(B, seed=61)).to(dev)
    inp = torch.empty((B, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    rows = torch.empty((B, 1 + 56 * 4 * 3), dtype=torch.float32, device=dev)

    def check():
        pre, r = inp.cpu().numpy(), rows.cpu().numpy()
        for b in range(B):
            assert np.array_equal(pre[b], UO.preprocess(_host(frames[b])))
        _post_check(pd.cpu().numpy(), sizes, r)
        assert r[:, 0].min() > 0

    P.ufld_preprocess(frames, out=inp)
    P.ufld_postprocess(pd, sizes, out=rows)
    torch.cuda.synchronize()
    check()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.ufld_preprocess(frames, out=inp)
        P.ufld_postprocess(pd, sizes, out=rows)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    pd.copy_(torch.from_numpy(_probs(B, seed=62)))
    g.replay()
    torch.cuda.synchronize()
    check()
