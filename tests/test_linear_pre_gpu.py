"""The bilinear letterbox pre-process and the truncating get_rect rows of yolov3, yolov4, scaled-yolov4, yolov3-spp and RetinaFace
on the device: trtx_linear_preprocess_enqueue against the CPU oracle (oracle/linear_oracle.c, pinned to cv2 by
tests/test_linear_pre_cpu.py) bit for bit, and the rows-only mode of trtx_yolo_seg_postprocess_enqueue with TRTX_YOLO_V3 and
TRTX_RECT_YOLOV3_SPP against trtx_get_rect bit for bit, after the fused yolov3 decode + NMS too."""

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import linear as LO
from oracle import oracle as O
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
VARIANTS = [(L.LINEAR_YOLOV3, 608, 608), (L.LINEAR_RETINA, 640, 480), (L.LINEAR_YOLOV3, 512, 512)]
# up- and downscales, the identity, 1-pixel rectangle sides (2 x 1000 at 608), odd sizes, tall and wide, 4K
MIXED = [(1920, 1080), (1280, 720), (608, 608), (640, 480), (480, 640), (300, 200), (2, 1000), (1000, 2), (1, 3), (97, 301),
         (731, 1299), (3840, 2160), (2432, 600), (53, 77)]


def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra + 1 bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def _fits(w, h, net_w, net_h):
    """preprocess_img's rectangle is not empty (2 x 1000 at 640 x 480 is 0 pixels wide)."""
    r = (C.c_int * 4)()
    L.load().trtx_calib_letterbox_rect(w, h, net_w, net_h, r)
    return r[2] > 0 and r[3] > 0


def _expect(frames, variant, net_w, net_h, mx=608):
    return np.stack([LO.preprocess(_host(f), variant, net_w, net_h, mx)[0] for f in frames])


@pytest.mark.parametrize("variant,net_w,net_h", VARIANTS)
def test_mixed_sizes_pitched_cropped_equal_oracle(dev, variant, net_w, net_h):
    """One call over frames of mixed sizes, pitch > 3 * width at odd bases and a cropped view of a larger frame, into a dst
    that is only 4-byte aligned, equals the oracle bit for bit; nothing around the output is written, nor the frames."""
    rng = np.random.default_rng(1 + variant + net_h)
    sizes = [(w, h) for w, h in MIXED if _fits(w, h, net_w, net_h)]
    frames = [_frame(rng, w, h, dev, 5 + 3 * (i % 4)) for i, (w, h) in enumerate(sizes)]
    frames.append(_frame(rng, 1000, 700, dev, 0)[37:637, 101:901])  # a crop: 800 x 600 inside a 1000-wide pitch
    before = [_host(f) for f in frames]
    n = len(frames) * 3 * net_w * net_h
    big = torch.full((n + 8,), -7.0, dtype=torch.float32, device=dev)
    P.linear_preprocess(frames, variant, out=big[1:1 + n].view(len(frames), 3, net_h, net_w), net_w=net_w, net_h=net_h)
    got = big.cpu().numpy()
    exp = _expect(frames, variant, net_w, net_h)
    for i in range(len(frames)):
        assert np.array_equal(got[1:1 + n].reshape(-1, 3, net_h, net_w)[i], exp[i]), i
        assert np.array_equal(_host(frames[i]), before[i])
    assert got[0] == -7.0 and (got[1 + n:] == -7.0).all()


def test_spp_at_and_below_max(dev):
    """yolov3-spp: frames above MAX sharing the 608 x 352 canvas, frames below it sharing 320 x 224 (copied, not resized), and
    608 x 608 itself; each call binds one canvas."""
    rng = np.random.default_rng(8)
    for sizes in ([(1920, 1080), (1280, 720), (3840, 2160), (2432, 1368)], [(300, 200), (310, 210), (292, 194)],
                  [(608, 608), (1216, 1216), (700, 700)]):
        canvases = {P.yolov3spp_letterbox(w, h)[0] for w, h in sizes}
        assert len(canvases) == 1, canvases
        (cw, ch), = canvases
        frames = [_frame(rng, w, h, dev, i) for i, (w, h) in enumerate(sizes)]
        out = torch.full((len(frames), 3, ch, cw), -1.0, dtype=torch.float32, device=dev)
        P.linear_preprocess(frames, L.LINEAR_YOLOV3_SPP, out=out, net_w=cw, net_h=ch, max_size=608)
        assert np.array_equal(out.cpu().numpy(), _expect(frames, L.LINEAR_YOLOV3_SPP, cw, ch)), sizes


@pytest.mark.parametrize("variant,net_w,net_h", VARIANTS[:2])
def test_70_frames_two_launches_and_graph_replay(dev, variant, net_w, net_h):
    """70 frames take two launches; a graph-captured call replayed on overwritten frames gives the oracle's values for them."""
    rng = np.random.default_rng(9 + variant)
    fit = [(w, h) for w, h in MIXED if _fits(w, h, net_w, net_h)]
    sizes = [fit[i % len(fit)] if i % 5 else (1280, 720) for i in range(70)]
    sizes = [(w, h) if w * h <= 1280 * 720 else (w // 3, h // 3) for w, h in sizes]
    frames = [_frame(rng, w, h, dev, i % 7) for i, (w, h) in enumerate(sizes)]
    out = torch.empty((70, 3, net_h, net_w), dtype=torch.float32, device=dev)
    P.linear_preprocess(frames, variant, out=out, net_w=net_w, net_h=net_h)
    assert np.array_equal(out.cpu().numpy(), _expect(frames, variant, net_w, net_h))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.linear_preprocess(frames, variant, out=out, net_w=net_w, net_h=net_h)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    out.fill_(5.0)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), _expect(frames, variant, net_w, net_h))


def test_rejected_calls_write_nothing(dev):
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 320, 180, dev, 5) for _ in range(69)] + [_frame(rng, 1, 700, dev, 0)]
    out = torch.full((70, 3, 608, 608), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):  # frame 69's rectangle is empty: no launch for frames 0..63 either
        P.linear_preprocess(frames, L.LINEAR_YOLOV3, out=out)
    lib = L.load()
    descs = P._image_descs(frames[:2])
    assert lib.trtx_linear_preprocess_enqueue(7, descs, 2, 608, 608, 608, out.data_ptr(), None) == L.ERR_INVALID
    assert lib.trtx_linear_preprocess_enqueue(0, descs, 2, 608, 608, 608, out.data_ptr() + 2, None) == L.ERR_INVALID
    assert lib.trtx_linear_preprocess_enqueue(0, None, 2, 608, 608, 608, out.data_ptr(), None) == L.ERR_INVALID
    assert lib.trtx_linear_preprocess_enqueue(1, descs, 2, 608, 608, 608, None, None) == L.ERR_INVALID
    spp = [_frame(rng, 300, 200, dev, 0), _frame(rng, 250, 200, dev, 0)]  # canvases 320 x 224 and 256 x 224
    small = torch.full((2, 3, 224, 320), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.linear_preprocess(spp, L.LINEAR_YOLOV3_SPP, out=small, net_w=320, net_h=224)
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (small == 3.0).all()


# ------------------------------------------------------------------ rows ----------------------------------------------
SIZES = [(1920, 1080), (1080, 1920), (608, 608), (640, 480), (300, 200), (1, 7), (4000, 3000), (99, 331), (5, 70000)]


def _dets(rng, B, K, R, counts):
    """[B, 1 + K * R] rows (cx, cy, w, h, conf, class, keep) with negative, large and non-finite boxes among them."""
    d = np.zeros((B, 1 + K * R), np.float32)
    for b in range(B):
        rows = np.zeros((K, R), np.float32)
        rows[:, :2] = rng.uniform(-60, 700, (K, 2))
        rows[:, 2:4] = rng.uniform(0, 500, (K, 2))
        rows[:, 4] = rng.uniform(0, 1, K)
        rows[:, 5] = rng.integers(0, 80, K)
        rows[:, 6] = 1
        rows[: K // 10, :4] = rng.choice(np.array([np.nan, np.inf, -np.inf, 3e9, -2.5e9, 1e30], np.float32), (K // 10, 4))
        d[b, 0] = counts[b]
        d[b, 1:] = rows.reshape(-1)
    return d


def _check_rows(got, dets, sizes, variant, net, K, R):
    for b, (w, h) in enumerate(sizes):
        n = int(min(max(dets[b, 0], 0), K))
        assert got[b, 0] == n
        g = got[b, 1:].reshape(K, 6)
        src = dets[b, 1:].reshape(K, R)
        for i in range(n):
            assert tuple(int(v) for v in g[i, :4]) == P.get_rect(w, h, src[i, :4], net, net, variant), (b, i, src[i, :4])
            assert np.array_equal(g[i, 4:], src[i, 4:6])
        assert (g[n:] == 0).all()


@pytest.mark.parametrize("variant,net", [(L.YOLO_V3, 608), (L.YOLO_V3, 416), (L.RECT_YOLOV3_SPP, 608)])
def test_rows_equal_get_rect(dev, variant, net):
    """Frames of mixed sizes, a count above max_rows, an empty image and a negative count; undefined boxes give zeros."""
    rng = np.random.default_rng(40 + variant + net)
    B, K, R = len(SIZES), 300, 7
    counts = [K, 5000, 0, -3, 17, 1, K, 299, 64]
    dets = _dets(rng, B, K, R, counts)
    out = torch.full((B, 1 + K * 6), 9.0, dtype=torch.float32, device=dev)
    P.yolo_seg_postprocess(None, torch.from_numpy(dets).to(dev), SIZES, variant=variant, max_rows=K, row_floats=R,
                           max_masks=1, net_w=net, net_h=net, masks=False, rows_out=out)
    got = out.cpu().numpy()
    _check_rows(got, dets, SIZES, variant, net, K, R)
    zeros = sum(int((got[b, 1:].reshape(K, 6)[:max(0, min(counts[b], K)), 2:4] == 0).all(1).sum()) for b in range(B))
    assert zeros >= K // 10


def test_fused_decode_nms_then_rows_and_graph(dev):
    """Synthetic yolov3 heads through the fused decode + NMS, then the rows: the kept set is the oracle nms()'s, and each
    rectangle is trtx_get_rect of the kept box, for frames of different sizes; the two calls replay from a CUDA graph."""
    B, net = 3, 608
    heads = synth.yolov3_heads(B, seed=77, net_w=net, net_h=net)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    plug = P.YoloLayerPluginV3()
    plug.configure(hd)  # the grids of the heads, as the plugin's enqueue takes them
    orc, orc_idx = O.yolov3_decode(heads, [k.anchors for k in P.YOLOV3_KERNELS])
    fused = P.FusedYoloDecodeNms(plug, B, 0.5, 0.4, device=dev)
    sizes = [(1920, 1080), (500, 375), (720, 1280)]
    comp, idx = fused.enqueue(B, hd)
    K = (comp.shape[1] - 1) // 7
    rows = P.yolo_seg_postprocess(None, comp, sizes, variant=L.YOLO_V3, max_rows=K, row_floats=7, max_masks=1, net_w=net,
                                  net_h=net, masks=False)[0]
    c, ix, r = comp.cpu().numpy(), idx.cpu().numpy(), rows.cpu().numpy()
    same = 0
    for b, (w, h) in enumerate(sizes):
        res, src = O.nms(1, orc[b], 1000, 7, 0.5, 0.4)
        n = int(c[b, 0])
        assert n == len(res) and n > 5 and r[b, 0] == n
        assert np.array_equal(ix[b, :n], orc_idx[b][src])
        kept = c[b, 1:1 + n * 7].reshape(n, 7)
        got = r[b, 1:1 + n * 6].reshape(n, 6)
        for i in range(n):
            rect = P.get_rect(w, h, kept[i, :4], net, net, L.YOLO_V3)
            assert tuple(int(v) for v in got[i, :4]) == rect
            if np.array_equal(kept[i, :4], res[i, :4]):  # where the device box is the oracle's to the bit, so is the rect
                assert P.get_rect(w, h, res[i, :4], net, net, L.YOLO_V3) == rect
                same += 1
    assert same > 0
    g = torch.cuda.CUDAGraph()
    frames = [torch.from_numpy(synth.frames(1, seed=5 + b, h=h, w=w)[0]).to(dev) for b, (w, h) in enumerate(sizes)]
    pre = torch.empty((B, 3, net, net), dtype=torch.float32, device=dev)
    with torch.cuda.graph(g):
        P.linear_preprocess(frames, L.LINEAR_YOLOV3, out=pre, net_w=net, net_h=net)
        P.yolo_seg_postprocess(None, comp, sizes, variant=L.YOLO_V3, max_rows=K, row_floats=7, max_masks=1, net_w=net,
                               net_h=net, masks=False, rows_out=rows)
    rows.fill_(-1.0)
    pre.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(rows.cpu().numpy(), r)
    assert np.array_equal(pre.cpu().numpy(), _expect(frames, L.LINEAR_YOLOV3, net, net))
