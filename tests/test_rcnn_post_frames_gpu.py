"""Mask R-CNN post-process for frames of mixed sizes on the GPU (trtx_rcnn_postprocess_frames_enqueue), bit for bit against
  - the CPU oracle run per frame with that frame's size (oracle/rcnn_post.py, pinned to cv2 and to the reference's compiled
    preprocessImg in tests/test_rcnn_post_cpu.py);
  - B batch-1 calls of trtx_rcnn_postprocess_enqueue with offset pointers, which defines the per-frame semantics;
  - one call of trtx_rcnn_postprocess_enqueue for a batch of one size.
The wrapper passes img_w = img_h = 0 in the parameter block, so every call here also shows that the entry does not read them."""
import numpy as np
import pytest
import torch

from oracle import rcnn_post as RP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth
from tensorrtx_b200.pipeline import RcnnHeadChain

pytestmark = pytest.mark.gpu
F = np.float32
ROW_SENTINEL, CANVAS_SENTINEL = -7.0, 77
NET_W, NET_H = 1067, 800
# the sizes of a mixed batch, then tiny frames and extreme aspect ratios, where the pads and the ratios differ most
MIXED = [(640, 480), (480, 640), (1280, 720), (1920, 1080), (1333, 750), (800, 800), (3000, 200), (64, 48), (17, 23),
         (1, 600), (5000, 40)]


def _inputs(rng, frames, D, S):
    """BatchedNms-like outputs: half the boxes inside each frame's letterboxed rectangle (so every frame gets pastes), half
    anywhere in the network input, plus boxes in the padding, across the borders, degenerate, inverted and non-finite;
    scores exactly at the threshold and NaN."""
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
            [300, 300, 200, 250], [np.nan, 5, 50, 50], [5, 5, np.inf, 50], [-np.inf, 5, 50, 50], [1e30, 5, 2e30, 50],
            [5, -3e9, 50, 4e9]]
    boxes[:, D - len(edge):] = edge
    scores = rng.uniform(0.3, 1.0, (B, D)).astype(F)
    scores[:, D - len(edge):] = 0.95
    scores[:, 20] = F(0.6)          # exactly SCORE_THRESH: not kept
    scores[:, 21] = np.nan          # not kept
    scores[:, 22] = np.nextafter(F(0.6), F(1))
    classes = rng.integers(0, 80, (B, D)).astype(F)
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 2))).astype(F)
    return scores, boxes, classes, masks


def _oracle(scores, boxes, classes, masks, frames, max_masks):
    """Frame b through the oracle with its own size; canvases start as the sentinel, so untouched slots keep it."""
    B, D = scores.shape
    rows = np.zeros((B, 1 + D * 7), F)
    canv = []
    for b, (w, h) in enumerate(frames):
        c = None if masks is None else np.full((max_masks, h, w), CANVAS_SENTINEL, np.uint8)
        rows[b], _ = RP.rcnn_postprocess(scores[b], boxes[b], classes[b], None if masks is None else masks[b], w, h, NET_W,
                                         NET_H, 0.6, max_masks, c)
        canv.append(c)
    return rows, canv


def _pitched(frames, M, dev, pitch_extra=(0,), base_offset=(0,)):
    """Sentinel-filled buffers; frame b's canvases are a [M, h, w] view with pitch w + pitch_extra[b % ..] starting
    base_offset[b % ..] bytes into its buffer, 5 bytes before the buffer's end.  -> (views, [(buffer, offset, pitch)])."""
    views, bufs = [], []
    for b, (w, h) in enumerate(frames):
        pitch, off = w + pitch_extra[b % len(pitch_extra)], base_offset[b % len(base_offset)]
        buf = torch.full((off + M * h * pitch + 5,), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
        views.append(buf[off:off + M * h * pitch].view(M, h, pitch)[:, :, :w])
        bufs.append((buf, off, pitch))
    return views, bufs


def _run(t, frames, M, dev, canvases=None, masks=True):
    rows = torch.full((len(frames), 1 + t[0].shape[1] * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    if masks and canvases is None:
        canvases, _ = _pitched(frames, M, dev)
    rows, canv = P.rcnn_postprocess_frames(*(t if masks else t[:3]), frames=frames, net_w=NET_W, net_h=NET_H, max_masks=M,
                                           rows=rows, canvases=canvases)
    torch.cuda.synchronize()
    return rows.cpu().numpy(), None if canv is None else [c.cpu().numpy() for c in canv]


def _check_canvases(got, exp, rows, M, frames):
    pasted = 0
    for b in range(len(frames)):
        assert np.array_equal(got[b], exp[b]), (b, frames[b])     # slots at or past min(count, M) keep the sentinel in both
        n = min(int(rows[b, 0]), M)
        assert np.all(got[b][n:] == CANVAS_SENTINEL), b
        pasted += int((got[b][:n] == 255).any())
    return pasted


@pytest.fixture(scope="module")
def mixed(dev):
    D, S, M = 100, 14, 30
    frames = MIXED
    scores, boxes, classes, masks = _inputs(np.random.default_rng(7), frames, D, S)
    scores[2] = 0.1                 # a frame with no detection
    scores[4, 40:] = 0.2            # and one with a few
    t = [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]
    return dict(frames=frames, D=D, M=M, np=(scores, boxes, classes, masks), t=t)


def test_mixed_batch_equals_oracle_per_frame(dev, mixed):
    frames, M = mixed["frames"], mixed["M"]
    rows, canv = _run(mixed["t"], frames, M, dev)
    exp_rows, exp_canv = _oracle(*mixed["np"], frames, M)
    assert np.array_equal(rows, exp_rows, equal_nan=True)        # includes the zeroed rows past each count
    counts = exp_rows[:, 0].astype(int)
    assert counts[2] == 0 and 0 < counts[4] < 40 and (counts > M).sum() >= 5
    assert _check_canvases(canv, exp_canv, rows, M, frames) >= len(frames) - 1   # every frame with a detection pastes


def test_mixed_batch_equals_batch1_calls_of_the_single_size_entry(dev, mixed):
    frames, M, D = mixed["frames"], mixed["M"], mixed["D"]
    s, bx, c, m = mixed["t"]
    rows, canv = _run(mixed["t"], frames, M, dev)
    ref_rows = torch.full((len(frames), 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    ref_canv = []
    for b, (w, h) in enumerate(frames):
        cb = torch.full((1, M, h, w), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
        P.rcnn_postprocess(s[b:b + 1], bx[b:b + 1], c[b:b + 1], m[b:b + 1], img_w=w, img_h=h, net_w=NET_W, net_h=NET_H,
                           max_masks=M, out=(ref_rows[b:b + 1], cb))
        ref_canv.append(cb[0])
    torch.cuda.synchronize()
    assert np.array_equal(rows, ref_rows.cpu().numpy(), equal_nan=True)
    for b in range(len(frames)):
        assert np.array_equal(canv[b], ref_canv[b].cpu().numpy()), (b, frames[b])


@pytest.mark.parametrize("img_w,img_h", [(637, 479), (1920, 1080)])
def test_uniform_batch_equals_one_call_of_the_single_size_entry(dev, img_w, img_h):
    B, D, S, M = 8, 100, 14, 24
    frames = [(img_w, img_h)] * B
    scores, boxes, classes, masks = _inputs(np.random.default_rng(img_w), frames, D, S)
    t = [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]
    rows, canv = _run(t, frames, M, dev)
    ref_rows = torch.full((B, 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    ref_canv = torch.full((B, M, img_h, img_w), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
    P.rcnn_postprocess(*t, img_w=img_w, img_h=img_h, net_w=NET_W, net_h=NET_H, max_masks=M, out=(ref_rows, ref_canv))
    torch.cuda.synchronize()
    assert np.array_equal(rows, ref_rows.cpu().numpy(), equal_nan=True)
    ref_canv = ref_canv.cpu().numpy()
    for b in range(B):
        assert np.array_equal(canv[b], ref_canv[b]), b
    assert (ref_canv == 255).sum() > 1000


def test_odd_pitches_and_unaligned_bases_write_only_the_canvas_bytes(dev, mixed):
    frames, M = mixed["frames"], mixed["M"]
    views, bufs = _pitched(frames, M, dev, pitch_extra=(1, 13, 0, 13), base_offset=(0, 1, 3, 0, 7))
    rows, canv = _run(mixed["t"], frames, M, dev, canvases=views)
    exp_rows, exp_canv = _oracle(*mixed["np"], frames, M)
    assert np.array_equal(rows, exp_rows, equal_nan=True)        # rows past the count are zeroed, not left as the sentinel
    assert _check_canvases(canv, exp_canv, rows, M, frames) >= len(frames) - 1
    for b, (buf, off, pitch) in enumerate(bufs):
        w, h = frames[b]
        raw = buf.cpu().numpy()
        assert np.all(raw[:off] == CANVAS_SENTINEL) and np.all(raw[off + M * h * pitch:] == CANVAS_SENTINEL), b
        assert np.all(raw[off:off + M * h * pitch].reshape(M, h, pitch)[:, :, w:] == CANVAS_SENTINEL), b   # row padding
    assert any(p % 16 for _, _, p in bufs) and any(o % 16 for _, o, _ in bufs)


def test_rows_only_equals_full_mode(dev, mixed):
    frames, M = mixed["frames"], mixed["M"]
    full, _ = _run(mixed["t"], frames, M, dev)
    only, none = _run(mixed["t"], frames, M, dev, masks=False)
    assert none is None
    assert np.array_equal(only, full, equal_nan=True)
    exp_rows, _ = _oracle(*mixed["np"][:3], None, frames, M)
    assert np.array_equal(only, exp_rows, equal_nan=True)


def test_70_frames_span_two_launch_parameter_blocks(dev):
    sizes = [(64, 48), (17, 23), (640, 480), (1, 600), (333, 517), (5000, 40), (48, 64)]
    frames = [sizes[i % len(sizes)] for i in range(70)]
    D, S, M = 40, 14, 6
    np_in = _inputs(np.random.default_rng(70), frames, D, S)
    t = [torch.from_numpy(a).to(dev) for a in np_in]
    rows, canv = _run(t, frames, M, dev)
    exp_rows, exp_canv = _oracle(*np_in, frames, M)
    assert np.array_equal(rows, exp_rows, equal_nan=True)
    assert _check_canvases(canv, exp_canv, rows, M, frames) >= 60
    # a rejected call writes nothing, even when the bad frame is in the second block
    rows_t = torch.full((70, 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    views, _ = _pitched(frames, M, dev)
    bad = frames[:69] + [(0, 10)]
    views[69] = torch.full((M, 10, 0), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.rcnn_postprocess_frames(*t, frames=bad, net_w=NET_W, net_h=NET_H, max_masks=M, rows=rows_t, canvases=views)
    torch.cuda.synchronize()
    assert torch.all(rows_t == ROW_SENTINEL)
    assert all(bool(torch.all(v == CANVAS_SENTINEL)) for v in views)


def test_graph_capture_replays_equal_the_eager_call(dev, mixed):
    frames, M, D = mixed["frames"], mixed["M"], mixed["D"]
    eager_rows, eager_canv = _run(mixed["t"], frames, M, dev)
    rows = torch.full((len(frames), 1 + D * 7), ROW_SENTINEL, dtype=torch.float32, device=dev)
    canv, _ = _pitched(frames, M, dev, pitch_extra=(0, 13), base_offset=(0, 1))
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            P.rcnn_postprocess_frames(*mixed["t"], frames=frames, net_w=NET_W, net_h=NET_H, max_masks=M, rows=rows,
                                      canvases=canv)
    torch.cuda.synchronize()
    assert torch.all(rows == ROW_SENTINEL)                       # capture launches nothing
    for _ in range(2):
        rows.fill_(ROW_SENTINEL)
        for c in canv:
            c.fill_(CANVAS_SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(rows.cpu().numpy(), eager_rows, equal_nan=True)
        for b in range(len(frames)):
            assert np.array_equal(canv[b].cpu().numpy(), eager_canv[b]), b


def test_rcnn_head_chain_b8_to_mixed_frames(dev):
    """RcnnHeadChain (RpnDecode -> RpnNms -> PredictorDecode -> BatchedNms) on b8, MaskRcnnInference on synthetic mask
    logits, then the per-frame post-process on eight frame sizes; equal to the oracle run on the same device outputs."""
    B, Cc, D, S, M = 8, 80, 100, 14, 100
    frames = MIXED[:8]
    chain = RcnnHeadChain(B, synth.rcnn_anchors(), dev)
    rs, rd = synth.rpn_inputs(B, seed=41)
    cs, bd, _ = synth.predictor_inputs(B, seed=42)
    fs, fb, fc = chain.run_device(*(torch.from_numpy(x).to(dev) for x in (rs, rd, cs, bd)))
    logits = torch.from_numpy(np.random.default_rng(43).standard_normal((B, D, Cc, S, S), dtype=np.float32) * 2).to(dev)
    mk = torch.zeros((B, D, S, S), device=dev)
    assert L.load().trtx_mask_rcnn_inference(B, fc.data_ptr(), logits.data_ptr(), mk.data_ptr(), D, S, Cc,
                                             torch.cuda.current_stream().cuda_stream) == 0
    rows, canv = _run([fs, fb, fc, mk], frames, M, dev)
    np_out = tuple(x.cpu().numpy() for x in (fs, fb, fc, mk))
    exp_rows, exp_canv = _oracle(*np_out, frames, M)
    assert np.array_equal(rows, exp_rows, equal_nan=True)
    assert exp_rows[:, 0].min() > 0, exp_rows[:, 0]
    _check_canvases(canv, exp_canv, rows, M, frames)
    assert sum(int((c == 255).sum()) for c in canv) > 1000
