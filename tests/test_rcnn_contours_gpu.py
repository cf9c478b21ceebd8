"""Mask R-CNN instance outlines on the GPU (trtx_rcnn_contours_enqueue), entry for entry against the CPU oracle
(oracle_find_contours_external, pinned to cv2.findContours(RETR_EXTERNAL, CHAIN_APPROX_NONE) in
tests/test_rcnn_contours_cpu.py) run on each whole canvas, with the truncation rule applied to the oracle's full lists:
  - canvases from the real chain (rcnn_postprocess_frames on mixed sizes, rcnn_postprocess described as frames);
  - synthetic canvases with content only inside each row's paste rectangle r: noise, rings with islands, lines, components
    touching r's and the frame's edges; one 4096 x 3072 frame; empty-r and throwing rows;
  - small capacities; sentinels in every entry the call must not write; 70 frames (two launch blocks); graph replay;
    rejected calls and a too-small workspace, which write nothing."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from oracle import contours as CO
from oracle import rcnn_post as RP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
F = np.float32
SENT = -5
NET_W, NET_H = 1067, 800
MIXED = [(640, 480), (480, 640), (1280, 720), (1920, 1080), (800, 800), (3000, 200), (64, 48), (17, 23), (1, 600)]


def _chain_inputs(rng, frames, D, S):
    """BatchedNms-like outputs: boxes inside each frame's letterboxed rectangle and anywhere, edge cases at the end."""
    B = len(frames)
    boxes = np.empty((B, D, 4), F)
    for b, (w, h) in enumerate(frames):
        l, r, t, bt = RP.rcnn_letterbox_pads(w, h, NET_W, NET_H)
        cw, ch = NET_W - l - r, NET_H - t - bt
        n = D // 2
        x1, y1 = l + rng.uniform(-0.1, 0.9, n) * cw, t + rng.uniform(-0.1, 0.9, n) * ch
        boxes[b, :n] = np.stack([x1, y1, x1 + rng.uniform(0.01, 0.6, n) * cw + 0.5, y1 + rng.uniform(0.01, 0.6, n) * ch + 0.5], -1)
        x1, y1 = rng.uniform(-60, NET_W + 20, D - n), rng.uniform(-60, NET_H + 20, D - n)
        boxes[b, n:] = np.stack([x1, y1, x1 + rng.uniform(-10, 500, D - n), y1 + rng.uniform(-10, 400, D - n)], -1)
    edge = [[0, 0, 3, 3], [NET_W - 2, NET_H - 2, NET_W, NET_H], [-30, -30, NET_W + 30, NET_H + 30], [100, 100, 100, 100],
            [300, 300, 200, 250], [np.nan, 5, 50, 50], [5, 5, np.inf, 50], [1e30, 5, 2e30, 50]]
    boxes[:, D - len(edge):] = edge
    scores = rng.uniform(0.3, 1.0, (B, D)).astype(F)
    scores[:, D - len(edge):] = 0.95
    classes = rng.integers(0, 80, (B, D)).astype(F)
    # steep random logits, so the pastes often hold several components and holes
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 3))).astype(F)
    return scores, boxes, classes, masks


def _outputs(B, M, Cc, Pp, dev):
    return (torch.full((B, M, 2), SENT, dtype=torch.int32, device=dev),
            torch.full((B, M, Cc), SENT, dtype=torch.int32, device=dev),
            torch.full((B, M, Pp, 2), SENT, dtype=torch.int32, device=dev))


def _check(out, rows, canvases, M, D, Cc, Pp, frames):
    """Every slot against the oracle on the whole canvas; entries past the counts keep the sentinel."""
    counts, lengths, points = (t.cpu().numpy() for t in out)
    rows = rows.cpu().numpy()
    checked = 0
    for b, (w, h) in enumerate(frames):
        cv = canvases[b].cpu().numpy()
        n_kept = min(int(rows[b, 0]), D, M)
        for k in range(M):
            if k >= n_kept:
                assert tuple(counts[b, k]) == (0, 0), (b, k)
                assert (lengths[b, k] == SENT).all() and (points[b, k] == SENT).all(), (b, k)
                continue
            n, tot, ln, pt = CO.find_contours_external(np.ascontiguousarray(cv[k]))
            assert tuple(counts[b, k]) == (n, tot), (b, k, tuple(counts[b, k]), (n, tot))
            nl, npt = min(n, Cc), min(tot, Pp)
            np.testing.assert_array_equal(lengths[b, k, :nl], ln[:nl], err_msg=f"lengths {b} {k}")
            np.testing.assert_array_equal(points[b, k, :npt], pt[:npt], err_msg=f"points {b} {k}")
            assert (lengths[b, k, nl:] == SENT).all() and (points[b, k, npt:] == SENT).all(), (b, k)
            checked += n
    return checked


def _synthetic(rng, frames, D, M, kinds=("noise", "rings", "lines", "edges", "blob")):
    """rows [B, 1 + D*7] (count, boxes in frame pixels) and canvases whose content lies inside each row's paste rectangle
    only; the last two kept rows of each frame have an empty r and a non-finite box (the reference throws there)."""
    B = len(frames)
    rows = np.zeros((B, 1 + D * 7), F)
    canv = []
    for b, (w, h) in enumerate(frames):
        cnt = min(D, M) if b % 3 else max(min(D, M) - 2, 0)
        rows[b, 0] = cnt
        c = np.zeros((M, h, w), np.uint8)
        for k in range(cnt):
            kind = kinds[(b + k) % len(kinds)]
            if kind == "edges":                       # r reaches the frame's edges
                box = [rng.uniform(-5, 2), rng.uniform(-5, 2), w + rng.uniform(-1, 5), h + rng.uniform(-1, 5)]
            else:
                x1, y1 = rng.uniform(-3, w * 0.8), rng.uniform(-3, h * 0.8)
                box = [x1, y1, x1 + rng.uniform(0, w * 0.5), y1 + rng.uniform(0, h * 0.5)]
            if k == cnt - 1 and cnt >= 2:
                box = [50.0, 40.0, 20.0, 10.0] if b % 2 else [5.0, 5.0, 5.0 + w * 0.3, 5.0 + h * 0.3]
                if b % 2 == 0:
                    box[0] = np.nan
            if k == cnt - 2 and cnt >= 3:
                box = [w + 10.0, 5.0, w + 40.0, 30.0]     # r starts past the image: the reference throws
            rows[b, 1 + k * 7:1 + k * 7 + 4] = box
            rows[b, 1 + k * 7 + 4:1 + k * 7 + 7] = (0.9, 1.0, k)
            r = RP.rcnn_mask_rect(np.array(box, F), w, h)
            if r is None:
                continue
            x, y, rw, rh = r
            if kind == "noise":
                sub = (rng.random((rh, rw)) < rng.uniform(0.1, 0.9)) * rng.integers(1, 256, (rh, rw))
            elif kind == "rings":
                yy, xx = np.mgrid[:rh, :rw]
                cy, cx = rh / 2, rw / 2
                d = np.hypot((yy - cy) / max(rh, 1), (xx - cx) / max(rw, 1))
                sub = ((d > 0.25) & (d < 0.25 + rng.uniform(0.01, 0.1))) | (d < 0.08) | \
                      ((d > 0.15) & (d < 0.17)) | (d > 0.45)
                sub = sub * 255
            elif kind == "lines":
                sub = np.zeros((rh, rw), np.int64)
                sub[::max(rh // 5, 2), :] = 7
                sub[:, ::max(rw // 7, 2)] = 255
                for i in range(min(rh, rw)):
                    sub[i, i] = 1
            else:                                      # a blob, as the paste makes them, touching r's border
                m = (1 / (1 + np.exp(-rng.standard_normal((14, 14)) * 2))).astype(F)
                sub = (cv2.resize(m, (rw, rh), interpolation=cv2.INTER_LINEAR) > 0.5) * 255
                sub[0, :] = 255
            c[k, y:y + rh, x:x + rw] = sub.astype(np.uint8)
        canv.append(c)
    return rows, canv


def _call(rows_t, canv_t, frames, D, M, Cc, Pp, out=None, stream=None):
    return P.rcnn_contours(rows_t, canv_t, frames=frames, detections_per_im=D, max_masks=M, max_contours=Cc,
                           max_points=Pp, out=out, stream=stream)


def test_real_chain_mixed_sizes():
    rng = np.random.default_rng(1)
    dev = torch.device("cuda")
    D, M = 40, 12
    sc, bx, cl, mk = _chain_inputs(rng, MIXED, D, 14)
    t = [torch.from_numpy(a).to(dev) for a in (sc, bx, cl, mk)]
    rows, canv = P.rcnn_postprocess_frames(*t, frames=MIXED, net_w=NET_W, net_h=NET_H, max_masks=M)
    out = _outputs(len(MIXED), M, 16, 4096, dev)
    _call(rows, canv, MIXED, D, M, 16, 4096, out=out)
    torch.cuda.synchronize()
    assert _check(out, rows, canv, M, D, 16, 4096, MIXED) > 20


def test_real_chain_single_size_as_frames():
    rng = np.random.default_rng(2)
    dev = torch.device("cuda")
    D, M, w, h, B = 30, 10, 1280, 720, 3
    sc, bx, cl, mk = _chain_inputs(rng, [(w, h)] * B, D, 28)
    t = [torch.from_numpy(a).to(dev) for a in (sc, bx, cl, mk)]
    rows, canv = P.rcnn_postprocess(*t, img_w=w, img_h=h, net_w=NET_W, net_h=NET_H, max_masks=M)
    frames = [(w, h)] * B
    views = [canv[b] for b in range(B)]      # dense [B, M, h, w]: frames of equal size with pitch = img_w
    out = _outputs(B, M, 8, 2048, dev)
    _call(rows, views, frames, D, M, 8, 2048, out=out)
    torch.cuda.synchronize()
    assert _check(out, rows, views, M, D, 8, 2048, frames) > 10


@pytest.mark.parametrize("caps", [(64, 100000), (3, 50), (1, 1)])
def test_synthetic_canvases_and_truncation(caps):
    rng = np.random.default_rng(3)
    dev = torch.device("cuda")
    frames = [(640, 480), (97, 61), (1920, 1080), (33, 300), (5, 7), (400, 3)]
    D, M = 12, 8
    rows, canv = _synthetic(rng, frames, D, M)
    rows_t = torch.from_numpy(rows).to(dev)
    canv_t = [torch.from_numpy(c).to(dev) for c in canv]
    Cc, Pp = caps
    out = _outputs(len(frames), M, Cc, Pp, dev)
    _call(rows_t, canv_t, frames, D, M, Cc, Pp, out=out)
    torch.cuda.synchronize()
    assert _check(out, rows_t, canv_t, M, D, Cc, Pp, frames) > 100


def test_pitched_canvases_and_padding_bytes():
    """Bytes past img_w in a pitched row are not read: they hold 255 and do not reach the contours."""
    rng = np.random.default_rng(4)
    dev = torch.device("cuda")
    frames = [(301, 157), (64, 64)]
    D, M = 6, 6
    rows, canv = _synthetic(rng, frames, D, M)
    views = []
    for c in canv:
        m_, h, w = c.shape
        buf = torch.full((m_, h, w + 13), 255, dtype=torch.uint8, device=dev)
        buf[:, :, :w] = torch.from_numpy(c).to(dev)
        views.append(buf[:, :, :w])
    rows_t = torch.from_numpy(rows).to(dev)
    out = _outputs(len(frames), M, 32, 20000, dev)
    _call(rows_t, views, frames, D, M, 32, 20000, out=out)
    torch.cuda.synchronize()
    _check(out, rows_t, [torch.from_numpy(c) for c in canv], M, D, 32, 20000, frames)


def test_large_frame_full_mask():
    """A 4096 x 3072 frame whose mask covers the whole net input: r is the frame."""
    dev = torch.device("cuda")
    w, h, D, M = 4096, 3072, 4, 2
    sc = torch.tensor([[0.9, 0.95, 0.1, 0.1]], device=dev)
    bx = torch.tensor([[[0, 0, NET_W, NET_H], [100, 100, 600, 500], [0, 0, 1, 1], [0, 0, 1, 1]]], dtype=torch.float32,
                      device=dev)
    cl = torch.zeros((1, D), device=dev)
    rng = np.random.default_rng(5)
    mk = torch.from_numpy((1 / (1 + np.exp(-rng.standard_normal((1, D, 14, 14)) * 2))).astype(F)).to(dev)
    rows, canv = P.rcnn_postprocess_frames(sc, bx, cl, mk, frames=[(w, h)], net_w=NET_W, net_h=NET_H, max_masks=M)
    r0 = RP.rcnn_mask_rect(rows[0, 1:5].cpu().numpy(), w, h)
    assert r0 == (0, 0, w, h)
    out = _outputs(1, M, 64, 60000, dev)
    _call(rows, canv, [(w, h)], D, M, 64, 60000, out=out)
    torch.cuda.synchronize()
    assert _check(out, rows, canv, M, D, 64, 60000, [(w, h)]) >= 2


def test_seventy_frames_two_launch_blocks():
    rng = np.random.default_rng(6)
    dev = torch.device("cuda")
    frames = [(int(rng.integers(8, 200)), int(rng.integers(8, 200))) for _ in range(70)]
    D, M = 5, 4
    rows, canv = _synthetic(rng, frames, D, M)
    rows_t = torch.from_numpy(rows).to(dev)
    canv_t = [torch.from_numpy(c).to(dev) for c in canv]
    out = _outputs(70, M, 6, 300, dev)
    _call(rows_t, canv_t, frames, D, M, 6, 300, out=out)
    torch.cuda.synchronize()
    assert _check(out, rows_t, canv_t, M, D, 6, 300, frames) > 100


def test_graph_replay_is_identical():
    rng = np.random.default_rng(7)
    dev = torch.device("cuda")
    frames = [(320, 240), (123, 77), (640, 480)]
    D, M = 8, 6
    rows, canv = _synthetic(rng, frames, D, M)
    rows_t = torch.from_numpy(rows).to(dev)
    canv_t = [torch.from_numpy(c).to(dev) for c in canv]
    ref = _outputs(3, M, 10, 3000, dev)
    _call(rows_t, canv_t, frames, D, M, 10, 3000, out=ref)
    out = _outputs(3, M, 10, 3000, dev)
    lib = L.load()
    q = L.RcnnPostParams(0, 0, 0, 0, D, 1, M, 0.0)
    descs, _ = P._frames(frames, canv_t, M, dev, True)
    n = lib.trtx_rcnn_contours_workspace_size(C.byref(q), descs, 3)
    work = torch.empty(n, dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, 3, rows_t.data_ptr(), 10, 3000, out[0].data_ptr(),
                                            out[1].data_ptr(), out[2].data_ptr(), work.data_ptr(), n, s.cuda_stream)
    assert rc == 0
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
    _check(out, rows_t, canv_t, M, D, 10, 3000, frames)


def test_rejected_calls_write_nothing():
    rng = np.random.default_rng(8)
    dev = torch.device("cuda")
    frames = [(64, 48), (100, 90)]
    D, M = 4, 3
    rows, canv = _synthetic(rng, frames, D, M)
    rows_t = torch.from_numpy(rows).to(dev)
    canv_t = [torch.from_numpy(c).to(dev) for c in canv]
    out = _outputs(2, M, 4, 100, dev)
    lib = L.load()
    q = L.RcnnPostParams(0, 0, 0, 0, D, 1, M, 0.0)
    descs, _ = P._frames(frames, canv_t, M, dev, True)
    n = lib.trtx_rcnn_contours_workspace_size(C.byref(q), descs, 2)
    assert n > 0
    work = torch.empty(n + 64, dtype=torch.uint8, device=dev)
    ptrs = [rows_t.data_ptr(), 4, 100, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr()]
    st = torch.cuda.current_stream().cuda_stream
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, 2, *ptrs, work.data_ptr(), n - 1, st) == L.ERR_WORKSPACE
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, 2, *ptrs, work.data_ptr() + 8, n, st) == L.ERR_INVALID
    bad = (L.Frame * 2)(descs[0], descs[1])
    bad[1].pitch = bad[1].img_w - 1
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), bad, 2, *ptrs, work.data_ptr(), n, st) == L.ERR_INVALID
    bad[1].pitch, bad[1].masks_dev = descs[1].pitch, None
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), bad, 2, *ptrs, work.data_ptr(), n, st) == L.ERR_INVALID
    torch.cuda.synchronize()
    for t in out:
        assert (t == SENT).all()
    # the same arguments accepted afterwards
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, 2, *ptrs, work.data_ptr(), n, st) == 0
    torch.cuda.synchronize()
    _check(out, rows_t, canv_t, M, D, 4, 100, frames)
