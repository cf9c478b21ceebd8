"""Mask R-CNN post-process on the GPU (trtx_rcnn_postprocess_enqueue, the device form of rcnn/rcnn.cpp:516-550) against the
CPU oracle, bit for bit: the rows, and the u8 canvases of the pasted masks.  The oracle itself is pinned to cv2 and to the
reference's compiled preprocessImg in tests/test_rcnn_post_cpu.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import rcnn_post as RP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
F = np.float32
ROW_SENTINEL, CANVAS_SENTINEL = -7.0, 77


def calculate_size(img_w, img_h):
    """calculateSize, rcnn/rcnn.cpp:349-366 -> (INPUT_W, INPUT_H)."""
    ratio = F(800.0) / F(min(img_h, img_w))
    newh, neww = (F(800.0), F(ratio * F(img_w))) if img_h < img_w else (F(ratio * F(img_h)), F(800.0))
    if max(newh, neww) > 1333.0:
        ratio = F(1333.0) / F(max(newh, neww))
        newh, neww = F(newh * ratio), F(neww * ratio)
    return int(float(neww) + 0.5), int(float(newh) + 0.5)


def _inputs(rng, B, D, S, net_w, net_h):
    """BatchedNms-like outputs with every edge case: boxes in the padding, across the borders, degenerate, inverted,
    non-finite; scores exactly at the threshold and NaN."""
    x1 = rng.uniform(-60, net_w + 20, (B, D))
    y1 = rng.uniform(-60, net_h + 20, (B, D))
    boxes = np.stack([x1, y1, x1 + rng.uniform(-10, 500, (B, D)), y1 + rng.uniform(-10, 400, (B, D))], -1).astype(F)
    edge = [[0, 0, 3, 3], [net_w - 2, net_h - 2, net_w, net_h], [-30, -30, net_w + 30, net_h + 30], [100, 100, 100, 100],
            [300, 300, 200, 250], [np.nan, 5, 50, 50], [5, 5, np.inf, 50], [-np.inf, 5, 50, 50], [1e30, 5, 2e30, 50],
            [5, -3e9, 50, 4e9]]
    for b in range(B):
        boxes[b, 1:1 + len(edge)] = edge
    scores = rng.uniform(0.3, 1.0, (B, D)).astype(F)
    scores[:, 1:1 + len(edge)] = 0.95
    scores[:, 20] = F(0.6)          # exactly SCORE_THRESH: not kept
    scores[:, 21] = np.nan          # not kept
    scores[:, 22] = np.nextafter(F(0.6), F(1))
    classes = rng.integers(0, 80, (B, D)).astype(F)
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 2))).astype(F)
    return scores, boxes, classes, masks


def _oracle(scores, boxes, classes, masks, img_w, img_h, net_w, net_h, max_masks, canvas_fill):
    B, D = scores.shape
    rows = np.zeros((B, 1 + D * 7), F)
    canv = None if masks is None else np.full((B, max_masks, img_h, img_w), canvas_fill, np.uint8)
    for b in range(B):
        rows[b], _ = RP.rcnn_postprocess(scores[b], boxes[b], classes[b], None if masks is None else masks[b], img_w, img_h,
                                             net_w, net_h, 0.6, max_masks, None if canv is None else canv[b])
    return rows, canv


@pytest.mark.parametrize("img_w,img_h,max_masks", [(640, 480, 100), (637, 479, 100), (1920, 1080, 24), (640, 480, 13)])
def test_rcnn_postprocess_matches_oracle(dev, img_w, img_h, max_masks):
    B, D, S = 8, 100, 14
    net_w, net_h = calculate_size(img_w, img_h)
    rng = np.random.default_rng(img_w + img_h + max_masks)
    scores, boxes, classes, masks = _inputs(rng, B, D, S, net_w, net_h)
    scores[3] = 0.1                 # an image with no detection
    scores[5, 40:] = 0.2            # and one with a few
    rows = torch.full((B, 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    canv = torch.full((B, max_masks, img_h, img_w), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
    t = [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]
    got_rows, got_canv = P.rcnn_postprocess(*t, img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h, max_masks=max_masks,
                                            out=(rows, canv))
    torch.cuda.synchronize()
    got_rows, got_canv = got_rows.cpu().numpy(), got_canv.cpu().numpy()
    exp_rows, exp_canv = _oracle(scores, boxes, classes, masks, img_w, img_h, net_w, net_h, max_masks, CANVAS_SENTINEL)
    assert np.array_equal(got_rows, exp_rows, equal_nan=True)     # includes the zeroed slots past the count
    counts = exp_rows[:, 0].astype(int)
    assert counts[3] == 0 and 0 < counts[5] < 40 and counts.max() > min(max_masks, 40)
    for b in range(B):
        n = min(counts[b], max_masks)
        assert np.array_equal(got_canv[b, :n], exp_canv[b, :n]), b
        assert np.all(got_canv[b, n:] == CANVAS_SENTINEL)          # canvases past the count are not written
        assert (got_canv[b, :n] == 255).any() or n == 0


def test_rcnn_postprocess_rows_only_equals_full_mode(dev):
    B, D, S, img_w, img_h = 8, 100, 14, 640, 480
    net_w, net_h = calculate_size(img_w, img_h)
    scores, boxes, classes, masks = _inputs(np.random.default_rng(5), B, D, S, net_w, net_h)
    t = [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]
    full, _ = P.rcnn_postprocess(*t, img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h)
    rows = torch.full((B, 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    only, none = P.rcnn_postprocess(*t[:3], img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h, out=(rows, None))
    torch.cuda.synchronize()
    assert none is None
    assert torch.equal(torch.nan_to_num(full, nan=1234.0), torch.nan_to_num(only, nan=1234.0))
    exp, _ = _oracle(scores, boxes, classes, None, img_w, img_h, net_w, net_h, D, 0)
    assert np.array_equal(only.cpu().numpy(), exp, equal_nan=True)


def _ws(nbytes, dev):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=dev)


def test_rcnn_chain_b8_to_postprocess(dev):
    """RpnDecode -> RpnNms -> PredictorDecode -> BatchedNms (as in the b8 chain test), then MaskRcnnInference and the
    post-process, all on the device; the post-process equals the oracle run on the same device outputs."""
    B, A, H, W, pre, post, N, Cc, D, S = 8, 15, 50, 67, 6000, 1000, 1000, 80, 100, 14
    img_w, img_h = 640, 480
    net_w, net_h = calculate_size(img_w, img_h)
    assert (net_w, net_h) == (1067, 800)
    anchors = synth.rcnn_anchors()
    scores, deltas = synth.rpn_inputs(B, seed=31, A=A, H=H, W=W)
    d_s, d_b = torch.zeros((B, pre), device=dev), torch.zeros((B, pre, 4), device=dev)
    p1 = P.RpnDecodePlugin(pre, anchors, 16.0, net_h, net_w, H, W)
    assert p1.enqueue(B, [torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)], [d_s, d_b],
                      _ws(p1.getWorkspaceSize(B), dev)) == 0
    props = torch.zeros((B, post, 4), device=dev)
    assert P.RpnNmsPlugin(0.7, post, pre).enqueue(B, [d_s, d_b], [props], _ws(256, dev)) == 0
    cls_scores, box_deltas, _ = synth.predictor_inputs(B, seed=32, N=N, Ccls=Cc)
    os_, ob, oc = torch.zeros((B, N), device=dev), torch.zeros((B, N, 4), device=dev), torch.zeros((B, N), device=dev)
    assert P.PredictorDecodePlugin(N, net_h, net_w, (10.0, 10.0, 5.0, 5.0), Cc).enqueue(
        B, [torch.from_numpy(cls_scores).to(dev), torch.from_numpy(box_deltas).to(dev), props], [os_, ob, oc], _ws(256, dev)) == 0
    fs, fb, fc = torch.zeros((B, D), device=dev), torch.zeros((B, D, 4), device=dev), torch.zeros((B, D), device=dev)
    assert P.BatchedNmsPlugin(1, 0.5, D, N).enqueue(B, [os_, ob, oc], [fs, fb, fc], _ws(256, dev)) == 0
    logits = torch.from_numpy(np.random.default_rng(33).standard_normal((B, D, Cc, S, S), dtype=np.float32) * 2).to(dev)
    mk = torch.zeros((B, D, S, S), device=dev)
    assert L.load().trtx_mask_rcnn_inference(B, fc.data_ptr(), logits.data_ptr(), mk.data_ptr(), D, S, Cc,
                                             torch.cuda.current_stream().cuda_stream) == 0
    rows, canv = P.rcnn_postprocess(fs, fb, fc, mk, img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h)
    torch.cuda.synchronize()
    s_, b_, c_, m_ = (x.cpu().numpy() for x in (fs, fb, fc, mk))
    exp_rows, exp_canv = _oracle(s_, b_, c_, m_, img_w, img_h, net_w, net_h, D, 0)
    assert np.array_equal(rows.cpu().numpy(), exp_rows, equal_nan=True)
    counts = exp_rows[:, 0].astype(int)
    assert counts.min() > 0, counts
    got = canv.cpu().numpy()
    for b in range(B):
        assert np.array_equal(got[b], exp_canv[b]), b
    assert (got == 255).sum() > 1000


def test_rcnn_postprocess_invalid_arguments_raise(dev):
    s, bx, c = torch.zeros((2, 10), device=dev), torch.zeros((2, 10, 4), device=dev), torch.zeros((2, 10), device=dev)
    m = torch.zeros((2, 10, 40, 40), device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):      # mask_size beyond the shared-memory stage
        P.rcnn_postprocess(s, bx, c, m, img_w=64, img_h=48, net_w=100, net_h=80)
    with pytest.raises(ValueError):
        P.rcnn_postprocess(s, bx[:, :5], c, img_w=64, img_h=48, net_w=100, net_h=80)
    q = L.RcnnPostParams(100, 80, 64, 48, 10, 14, 10, 0.6)
    assert L.load().trtx_rcnn_postprocess_enqueue(C.byref(q), 2, s.data_ptr(), bx.data_ptr(), c.data_ptr(), m.data_ptr(),
                                                  s.data_ptr(), None, None) == L.ERR_INVALID
