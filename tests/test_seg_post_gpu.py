"""YOLO segmentation post-process on the GPU (trtx_yolo_seg_postprocess_enqueue: process_mask + scale_mask + draw_mask_bbox's
mask selection in one call) against
  - the library's own kernels, bit for bit: trtx_process_mask_enqueue -> trtx_scale_mask_enqueue, thresholded inside the
    host trtx_get_rect rectangle (the main gate: the fused kernel evaluates the same expressions of the same inputs);
  - the CPU oracle (oracle/seg_post_oracle.c), equal except where the oracle's S lies within 2e-6 of 0.5 (CUDA vs glibc expf
    inside the sigmoid).
The oracle itself is pinned to cv2 and to the reference's compiled draw_mask_bbox in tests/test_seg_post_cpu.py."""
import numpy as np
import pytest
import torch

from oracle import seg_post as SP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
F = np.float32
ROW_SENTINEL, CANVAS_SENTINEL = -7.0, 77
MIXED = [(1920, 1080), (1080, 1920), (1280, 720), (640, 480), (480, 640), (640, 640), (333, 1001), (17, 1000)]


def _edge_boxes(variant):
    """Boxes inside the frame, across its borders, in the letterbox padding, degenerate, non-finite and huge."""
    if variant == L.YOLO_V8:  # l, t, r, b (process_mask reads them as x, y, w, h, like the reference)
        return [[100, 150, 300, 400], [-40, -30, 200, 180], [500, 560, 700, 690], [0, 0, 640, 640], [10, 5, 60, 70],
                [300, 2, 380, 30], [200, 200, 200, 200], [250, 260, 240, 250], [np.nan, 5, 50, 50], [5, 5, np.inf, 50],
                [-np.inf, 5, 50, 50], [1e30, 5, 2e30, 50]]
    return [[320, 320, 200, 250], [10, 20, 120, 100], [630, 620, 100, 90], [320, 320, 700, 700], [40, 8, 60, 30],
            [320, 600, 80, 60], [300, 300, 0, 0], [200, 200, -20, 30], [np.nan, 5, 50, 50], [5, 5, np.inf, 50],
            [-np.inf, 5, 50, 50], [1e30, 5, 50, 50]]


def _inputs(rng, variant, B, K, counts, R=39, off=7, n_rand=20, nan_coeff=False):
    proto = rng.standard_normal((B, 32, 160, 160)).astype(F)
    dets = np.zeros((B, 1 + K * R), F)
    edge = _edge_boxes(variant)
    for b in range(B):
        dets[b, 0] = counts[b]
        rows = dets[b, 1:].reshape(K, R)
        for i in range(K):
            if i < n_rand:
                if variant == L.YOLO_V8:
                    x, y = rng.uniform(-20, 600), rng.uniform(-20, 600)
                    rows[i, :4] = [x, y, x + rng.uniform(2, 300), y + rng.uniform(2, 300)]
                else:
                    rows[i, :4] = [rng.uniform(0, 640), rng.uniform(0, 640), rng.uniform(2, 300), rng.uniform(2, 300)]
            else:
                rows[i, :4] = edge[(i - n_rand) % len(edge)]
            rows[i, 4:6] = [rng.uniform(0.5, 1), rng.integers(0, 80)]
            rows[i, off:off + 32] = rng.standard_normal(32) * 0.6
        if nan_coeff:
            rows[0, off + 3] = np.nan
    return proto, dets


def _canvases(sizes, M, dev, odd_pitch=(), offset_base=()):
    """Sentinel-filled canvases; image b in odd_pitch gets pitch w + 3, image b in offset_base a base 1 byte off alignment."""
    out = []
    for b, (w, h) in enumerate(sizes):
        pitch = w + 3 if b in odd_pitch else w
        extra = 1 if b in offset_base else 0
        buf = torch.full((extra + M * h * pitch,), CANVAS_SENTINEL, dtype=torch.uint8, device=dev)
        out.append(buf[extra:].view(M, h, pitch)[:, :, :w])
    return out


def _composition(variant, proto_d, dets_d, dets, sizes, K, M, R=39, off=7):
    """process_mask -> scale_mask (the library's kernels), thresholded like draw_mask_bbox inside the host get_rect rect."""
    masks = P.process_mask(proto_d, dets_d, K, R, off, M, 640, 640, variant=variant)
    res = []
    for b, (w, h) in enumerate(sizes):
        n = min(max(int(dets[b, 0]), 0), K, M)
        c = np.zeros((n, h, w), np.uint8)
        if n:
            S = P.scale_mask(masks[b, :n].contiguous(), w, h)
            keep = (~(S <= 0.5)).cpu().numpy()
            rows = dets[b, 1:].reshape(K, R)
            for k in range(n):
                x, y, rw, rh = P.get_rect(w, h, rows[k, :4], variant=variant)
                x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + rw, w), min(y + rh, h)
                if x0 < x1 and y0 < y1:
                    c[k, y0:y1, x0:x1] = np.where(keep[k, y0:y1, x0:x1], 255, 0)
        res.append(c)
    return res


def _run(variant, proto_d, dets_d, sizes, K, M, canv, dev, R=39, off=7):
    rows = torch.full((len(sizes), 1 + K * 6), ROW_SENTINEL, dtype=torch.float32, device=dev)
    P.yolo_seg_postprocess(proto_d, dets_d, sizes, variant=variant, max_rows=K, row_floats=R, coeff_offset=off, max_masks=M,
                           rows_out=rows, canvases_out=canv)
    torch.cuda.synchronize()
    return rows.cpu().numpy(), [c.cpu().numpy() for c in canv]


def _check_rows(rows, dets, sizes, variant, K, R=39):
    for b, (w, h) in enumerate(sizes):
        n = min(max(int(dets[b, 0]), 0), K)
        assert rows[b, 0] == n
        src = dets[b, 1:].reshape(K, R)
        got = rows[b, 1:].reshape(K, 6)
        for i in range(n):
            assert tuple(int(v) for v in got[i, :4]) == P.get_rect(w, h, src[i, :4], variant=variant), (b, i, src[i, :4])
            assert np.array_equal(got[i, 4:6], src[i, 4:6])
        assert np.all(got[n:] == 0)                 # rows past the count are zeroed


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_mixed_batch_bit_exact_to_composition(dev, variant):
    """One b8 call over 8 frame sizes: 20 random boxes + the edge boxes per image, max_masks below the count, a count of 0,
    an odd pitch and a 1-byte-offset canvas base -> equal to the library's process_mask -> scale_mask, thresholded."""
    rng = np.random.default_rng(10 + variant)
    K, M = 40, 26
    counts = [32, 20, 0, 32, 26, 7, 32, 32]
    proto, dets = _inputs(rng, variant, len(MIXED), K, counts, nan_coeff=True)
    proto_d, dets_d = torch.from_numpy(proto).to(dev), torch.from_numpy(dets).to(dev)
    canv = _canvases(MIXED, M, dev, odd_pitch=(0, 6), offset_base=(1, 7))
    rows, got = _run(variant, proto_d, dets_d, MIXED, K, M, canv, dev)
    ref = _composition(variant, proto_d, dets_d, dets, MIXED, K, M)
    _check_rows(rows, dets, MIXED, variant, K)
    total = 0
    for b in range(len(MIXED)):
        n = ref[b].shape[0]
        assert np.array_equal(got[b][:n], ref[b]), (b, MIXED[b])
        assert np.all(got[b][n:] == CANVAS_SENTINEL)  # slots at or past min(count, max_masks) are untouched
        total += int((ref[b] == 255).sum())
    assert total > 100000  # the masks really select pixels
    # the non-finite and huge boxes whose get_rect is undefined get rect {0, 0, 0, 0} (and, in test_against_oracle, where
    # max_masks covers them, an all-zero canvas)
    src = dets[0, 1:].reshape(K, 39)
    undefined = [i for i in range(20, 32) if not np.all(np.isfinite(src[i, :4])) or np.abs(src[i, :4]).max() > 1e20]
    assert len(undefined) == 4
    assert sum(not rows[0, 1 + i * 6:1 + i * 6 + 4].any() for i in undefined) >= 3


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_against_oracle(dev, variant):
    """The CPU oracle: equal except where its S lies within 2e-6 of 0.5."""
    rng = np.random.default_rng(30 + variant)
    K, M = 32, 32
    sizes = MIXED
    counts = [32] * len(sizes)
    proto, dets = _inputs(rng, variant, len(sizes), K, counts)
    canv = _canvases(sizes, M, dev)
    rows, got = _run(variant, torch.from_numpy(proto).to(dev), torch.from_numpy(dets).to(dev), sizes, K, M, canv, dev)
    near_total = 0
    for b, (w, h) in enumerate(sizes):
        orows, ocanv, S = SP.seg_postprocess(variant, proto[b], dets[b], w, h, max_rows=K, max_masks=M, scaled=True)
        assert np.array_equal(rows[b], orows)
        src = dets[b, 1:].reshape(K, 39)
        for i in range(20, 32):
            if P.get_rect(w, h, src[i, :4], variant=variant) == (0, 0, 0, 0):
                assert not got[b][i].any()          # undefined or empty get_rect: nothing selected
        diff = got[b] != ocanv
        near = np.abs(S - 0.5) <= 2e-6
        assert not np.any(diff & ~near), (b, int((diff & ~near).sum()))
        near_total += int(diff.sum())
    print(f"variant {variant}: {near_total} pixels differ from the oracle, all with |S - 0.5| <= 2e-6")


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_rows_only_equal_host_get_rect(dev, variant):
    """Rows-only mode (proto NULL, every canvas NULL): 4000 random boxes x 8 frame sizes, each row equal to the host
    trtx_get_rect, conf and class copied, the tail zeroed."""
    rng = np.random.default_rng(50 + variant)
    K, R = 4000, 6
    B = len(MIXED)
    dets = np.zeros((B, 1 + K * R), F)
    for b in range(B):
        rows = dets[b, 1:].reshape(K, R)
        rows[:, :4] = rng.uniform(-100, 740, (K, 4))
        if variant == L.YOLO_V5:
            rows[:, 2:4] = rng.uniform(0, 400, (K, 2))
        rows[:, 4] = rng.uniform(0, 1, K)
        rows[:, 5] = rng.integers(0, 80, K)
        dets[b, 0] = K - 7 * b
    out = torch.full((B, 1 + K * 6), ROW_SENTINEL, dtype=torch.float32, device=dev)
    rows, canv = P.yolo_seg_postprocess(None, torch.from_numpy(dets).to(dev), MIXED, variant=variant, max_rows=K, row_floats=R,
                                        coeff_offset=0, max_masks=1, masks=False, rows_out=out)
    assert canv is None
    torch.cuda.synchronize()
    _check_rows(rows.cpu().numpy(), dets, MIXED, variant, K, R)


def test_70_images_two_launches(dev):
    """70 images (more than one launch of 64) of assorted small sizes: bit-exact to the composition."""
    rng = np.random.default_rng(70)
    sizes = [(int(rng.integers(8, 400)), int(rng.integers(8, 400))) for _ in range(70)]
    K, M = 12, 10
    counts = [int(rng.integers(0, 13)) for _ in range(70)]
    proto, dets = _inputs(rng, L.YOLO_V8, 70, K, counts, n_rand=8)
    proto_d, dets_d = torch.from_numpy(proto).to(dev), torch.from_numpy(dets).to(dev)
    canv = _canvases(sizes, M, dev, odd_pitch=(3, 66), offset_base=(65,))
    rows, got = _run(L.YOLO_V8, proto_d, dets_d, sizes, K, M, canv, dev)
    ref = _composition(L.YOLO_V8, proto_d, dets_d, dets, sizes, K, M)
    _check_rows(rows, dets, sizes, L.YOLO_V8, K)
    for b in range(70):
        n = ref[b].shape[0]
        assert np.array_equal(got[b][:n], ref[b]), (b, sizes[b])
        assert np.all(got[b][n:] == CANVAS_SENTINEL)


def test_decode_nms_seg_chain(dev, oracle):
    """trtx_yolo_decode_enqueue (is_seg) -> trtx_nms_enqueue (extra_floats = 32) -> the seg post-process: the kept counts
    equal the oracle chain's, the canvases equal the composition on the same NMS output and the CPU oracle (up to S
    within 2e-6 of 0.5)."""
    B, sizes = 4, [(1920, 1080), (640, 480), (1080, 1920), (333, 1001)]
    heads = synth.yolov8_heads(B, seed=21, extra=32, n_obj=20)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, True, False, False, (8, 16, 32))
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(h).to(dev) for h in heads], [out], ws) == 0
    K = 100
    comp = P.batch_nms(out, B, plug.output_elems(), 0.5, 0.45, det_floats=90, max_det=K, extra_floats=32, extra_offset=6)
    rng = np.random.default_rng(22)
    proto = (rng.standard_normal((B, 32, 160, 160)) * 0.5).astype(F)
    proto_d = torch.from_numpy(proto).to(dev)
    M = 40
    canv = _canvases(sizes, M, dev)
    rows, got = _run(L.YOLO_V8, proto_d, comp, sizes, K, M, canv, dev)
    dets = comp.cpu().numpy()
    ref_dec, _ = oracle.yolov8_decode(heads, is_seg=True)
    for b in range(B):
        res, _ = oracle.nms(0, ref_dec[b], 1000, 90, 0.5, 0.45)
        assert int(dets[b, 0]) == len(res) > 0
    ref = _composition(L.YOLO_V8, proto_d, comp, dets, sizes, K, M)
    _check_rows(rows, dets, sizes, L.YOLO_V8, K)
    for b, (w, h) in enumerate(sizes):
        n = ref[b].shape[0]
        assert np.array_equal(got[b][:n], ref[b])
        _, ocanv, S = SP.seg_postprocess(0, proto[b], dets[b], w, h, max_rows=K, max_masks=M, scaled=True)
        diff = got[b][:n] != ocanv[:n]
        assert not np.any(diff & ~(np.abs(S[:n] - 0.5) <= 2e-6))
        assert (got[b][:n] == 255).any()


def test_rejected_calls_write_nothing(dev):
    """Validation happens before the first launch: a rejected call leaves rows and canvases as they were."""
    K, M = 4, 2
    dets = torch.zeros((2, 1 + K * 39), device=dev)
    dets[:, 0] = 2
    proto = torch.zeros((2, 32, 160, 160), device=dev)
    rows = torch.full((2, 1 + K * 6), ROW_SENTINEL, device=dev)
    canv = _canvases([(64, 64), (1, 5000)], M, dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.yolo_seg_postprocess(proto, dets, [(64, 64), (1, 5000)], variant=0, max_rows=K, max_masks=M, rows_out=rows,
                               canvases_out=canv)
    torch.cuda.synchronize()
    assert torch.all(rows == ROW_SENTINEL) and torch.all(canv[0] == CANVAS_SENTINEL)
