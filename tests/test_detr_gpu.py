"""DETR on the device: trtx_detr_preprocess_enqueue and trtx_detr_postprocess_enqueue against the CPU oracle
(oracle/detr_oracle.c, pinned to cv2 and to the driver's loop by tests/test_detr_cpu.py), bit for bit."""

import numpy as np
import pytest
import torch

from oracle import detr as DO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
NET_W, NET_H = 1066, 800
MIXED = [(1920, 1080), (1280, 720), (640, 480), (1066, 800), (2132, 1600), (533, 400), (4000, 3000), (1, 1), (1, 500),
         (500, 1), (731, 1299)]


def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra + 1 bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def _outputs(B, Q, Cn, seed, planted=12):
    """Seeded softmax scores [B, Q, C] with `planted` confident objects per frame, and sigmoid boxes [B, Q, 4]."""
    rng = np.random.default_rng(seed)
    logits = rng.normal(0, 1, (B, Q, Cn)).astype(np.float32)
    logits[:, :, Cn - 1] += 3.0  # most queries: no object
    for b in range(B):
        qs = rng.choice(Q, min(planted, Q), replace=False)
        logits[b, qs, rng.integers(0, Cn - 1, len(qs))] += rng.uniform(4, 12, len(qs)).astype(np.float32)
    e = np.exp(logits - logits.max(-1, keepdims=True))
    scores = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    boxes = (1 / (1 + np.exp(-rng.normal(0, 1.5, (B, Q, 4))))).astype(np.float32)
    return scores, boxes


def _post_check(scores, boxes, sizes, got, thresh=np.float32(0.5)):
    for b, (w, h) in enumerate(sizes):
        want = DO.postprocess(scores[b], boxes[b], w, h, thresh)
        assert np.array_equal(got[b], want), (b, w, h)


# ------------------------------------------------------------------ pre-process ------------------------------------------
def test_preprocess_mixed_sizes_equals_oracle(dev):
    """One call over frames of mixed sizes (up- and down-scaling, the identity, the exact 2x downscale, 1 x N, N x 1), pitch >
    3 * width and odd bases, into a dst that is only 4-byte aligned, equals the oracle bit for bit; nothing around the output
    is written."""
    rng = np.random.default_rng(1)
    frames = [_frame(rng, w, h, dev, 13 + 3 * (i % 3)) for i, (w, h) in enumerate(MIXED)]
    n = len(frames) * 3 * NET_H * NET_W
    big = torch.full((n + 8,), -7.0, dtype=torch.float32, device=dev)
    P.detr_preprocess(frames, out=big[1:1 + n].view(len(frames), 3, NET_H, NET_W))
    got = big.cpu().numpy()
    for i, f in enumerate(frames):
        assert np.array_equal(got[1:1 + n].reshape(-1, 3, NET_H, NET_W)[i], DO.preprocess(_host(f))), MIXED[i]
    assert got[0] == -7.0 and (got[1 + n:] == -7.0).all()


def test_preprocess_other_net_and_all_bytes(dev):
    """Another net size (odd width, rows not a multiple of the band) and a frame holding every byte value in every channel."""
    rng = np.random.default_rng(4)
    allb = torch.from_numpy(np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(16, 16, 3).copy()).to(dev)
    frames = [allb, _frame(rng, 999, 555, dev, 2)]
    out = P.detr_preprocess(frames, net_w=321, net_h=243).cpu().numpy()
    for i, f in enumerate(frames):
        assert np.array_equal(out[i], DO.preprocess(_host(f), 321, 243)), i


def test_preprocess_70_frames_graph_replay(dev):
    """70 frames take two launches; the call captured in a CUDA graph and replayed on new frame contents gives the oracle's
    planes for those."""
    rng = np.random.default_rng(2)
    sizes = [(64 + 37 * i, 48 + 23 * i) for i in range(70)]
    frames = [_frame(rng, w, h, dev, i % 5) for i, (w, h) in enumerate(sizes)]
    out = torch.empty((70, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.detr_preprocess(frames, out=out)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    g.replay()
    torch.cuda.synchronize()
    for i in (0, 1, 63, 64, 69):
        assert np.array_equal(out[i].cpu().numpy(), DO.preprocess(_host(frames[i]))), i


# ------------------------------------------------------------------ post-process -----------------------------------------
def test_postprocess_planted_and_edge_queries(dev):
    """Seeded softmax outputs with planted objects on frames of mixed sizes, plus equal maxima, NaN scores and an all-NaN
    query, a score of exactly 0.5f, no-object winners, scores all below -1 and NaN / inf boxes, equal the oracle."""
    B, Q, Cn = 8, 100, 92
    scores, boxes = _outputs(B, Q, Cn, 5)
    s, bx = scores[0], boxes[0]
    s[:9] = 0.001
    s[0, 5] = s[0, 9] = 0.7
    s[1, :3] = np.nan
    s[1, 40] = 0.9
    s[2] = np.nan
    s[3, 7] = 0.5
    s[4, Cn - 1] = 0.95
    s[5] = -2.0
    s[6, 3] = 0.8
    bx[6] = (np.nan, 0.5, 0.2, 0.2)
    s[7, 4] = 0.8
    bx[7] = (0.5, np.inf, -np.inf, 0.2)
    s[8, 60:64] = 0.6  # four equal maxima
    sizes = MIXED[:B]
    rows = P.detr_postprocess(torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev), sizes).cpu().numpy()
    _post_check(scores, boxes, sizes, rows)
    r0 = rows[0, 1:1 + 6 * int(rows[0, 0])].reshape(-1, 6)
    assert {5, 40, 3, 4, 60} <= set(r0[:, 5].astype(int)) and not {7, Cn - 1} & set(r0[:, 5].astype(int))
    assert rows[:, 0].min() > 0
    for t in (-1.0, 0.0, 0.9):  # other thresholds, -1 the lowest accepted
        rows = P.detr_postprocess(torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev), sizes, score_thresh=t)
        _post_check(scores, boxes, sizes, rows.cpu().numpy(), np.float32(t))


@pytest.mark.parametrize("Q,Cn", [(100, 92), (1, 2), (300, 2), (37, 1000), (1500, 81), (2100, 33)])
def test_postprocess_other_sizes_and_70_frames(dev, Q, Cn):
    """Q and C other than 100 / 92 (one query, two classes, more queries than a pass of 1 024, more classes than lanes), 1
    and 70 mixed-size frames (two launches); rows past the count are written as zeros over a sentinel."""
    for B in (1, 70):
        scores, boxes = _outputs(B, Q, Cn, 100 + Q + B, planted=max(1, Q // 3))
        sizes = [(17 + 61 * b, 9 + 37 * b) for b in range(B)]
        out = torch.full((B, 1 + Q * 6), 9.0, dtype=torch.float32, device=dev)
        P.detr_postprocess(torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev), sizes, out=out)
        rows = out.cpu().numpy()
        _post_check(scores, boxes, sizes, rows)
        assert rows[:, 0].sum() > 0


def test_rejected_calls_write_nothing(dev):
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 320, 180, dev, 5), _frame(rng, 64, 48, dev, 0)]
    out = torch.full((2, 3, 64, 4758), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.detr_preprocess(frames, out=out, net_w=4758, net_h=64)
    descs = P._image_descs(frames)
    descs[1].pitch = 3 * 64 - 1
    assert L.load().trtx_detr_preprocess_enqueue(descs, 2, 4758, 64, out.data_ptr(), None) == L.ERR_INVALID
    scores, boxes = _outputs(2, 100, 92, 8)
    rows = torch.full((2, 601), 9.0, dtype=torch.float32, device=dev)
    sd, bd = torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev)
    for thresh, sizes in ((float("nan"), [(64, 48), (64, 48)]), (-1.5, [(64, 48), (64, 48)]), (0.5, [(64, 48), (64, 0)])):
        with pytest.raises(L.TrtxError, match="INVALID"):
            P.detr_postprocess(sd, bd, sizes, score_thresh=thresh, out=rows)
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (rows == 9.0).all()


# ------------------------------------------------------------------ end to end -------------------------------------------
def test_end_to_end_chain_and_graph_replay(dev):
    """Frames -> pre-process, and fixed seeded scores and boxes -> post-process, captured together in a CUDA graph and replayed
    on new frames, scores and boxes, give the oracle's planes and rows for those."""
    B, Q, Cn = 3, 100, 92
    rng = np.random.default_rng(9)
    sizes = [(1920, 1080), (1280, 720), (810, 1080)]
    frames = [_frame(rng, w, h, dev, 7) for w, h in sizes]
    s_np, b_np = _outputs(B, Q, Cn, 61)
    sd, bd = torch.from_numpy(s_np).to(dev), torch.from_numpy(b_np).to(dev)
    inp = torch.empty((B, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    rows = torch.empty((B, 1 + Q * 6), dtype=torch.float32, device=dev)

    def check():
        pre, r = inp.cpu().numpy(), rows.cpu().numpy()
        for b in range(B):
            assert np.array_equal(pre[b], DO.preprocess(_host(frames[b])))
        _post_check(sd.cpu().numpy(), bd.cpu().numpy(), sizes, r)
        assert r[:, 0].min() > 0

    P.detr_preprocess(frames, out=inp)
    P.detr_postprocess(sd, bd, sizes, out=rows)
    torch.cuda.synchronize()
    check()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.detr_preprocess(frames, out=inp)
        P.detr_postprocess(sd, bd, sizes, out=rows)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    s2, b2 = _outputs(B, Q, Cn, 62)
    sd.copy_(torch.from_numpy(s2))
    bd.copy_(torch.from_numpy(b2))
    g.replay()
    torch.cuda.synchronize()
    check()
