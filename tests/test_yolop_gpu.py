"""YOLOP on the device: trtx_yolop_preprocess_enqueue and trtx_yolop_postprocess_enqueue against the CPU oracle
(oracle/yolop_oracle.c, pinned to cv2 and to YOLOP's compiled host code by tests/test_yolop_cpu.py), YOLOP's YoloLayer scan
against YOLOP's own compiled plugin kernel (oracle/_ref/libref_yolop.so, or tests/golden/ref_yolop_gpu.npz where it was not
built), and the NMS + rows against YOLOP's compiled nms() and get_rect."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import yolop as YO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_yolop_gpu")
GH = RefOutputs("ref_yolop_host")
ANCHORS = ((3, 9, 5, 11, 4, 20), (7, 18, 6, 39, 12, 31), (19, 50, 38, 81, 68, 157))  # strides 8, 16, 32
STRIDES = (32, 16, 8)  # the plugin's input order (yolop/common.hpp:354)
MIXED = [(1920, 1080), (1280, 720), (640, 360), (333, 517), (1, 300), (2000, 7), (641, 385), (96, 54)]


def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def _kernels():
    return [P.YoloKernel(640 // s, 384 // s, ANCHORS[{8: 0, 16: 1, 32: 2}[s]]) for s in STRIDES]


def _heads(B, seed, nc=1):
    """Synthetic heads [B, 3 * (5 + nc), gh * gw] in the plugin's order; objectness mostly below the 0.1 gate."""
    rng = np.random.default_rng(seed)
    out = []
    for s in STRIDES:
        g = (640 // s) * (384 // s)
        h = rng.normal(0, 1.5, (B, 3, 5 + nc, g)).astype(np.float32)
        h[:, :, 4] = rng.normal(-5.0, 1.5, (B, 3, g))
        out.append(np.ascontiguousarray(h.reshape(B, 3 * (5 + nc), g)))
    return out


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _sorted_rows(buf, b, F=6):
    n = int(buf[b, 0])
    r = buf[b, 1:1 + n * F].reshape(n, F)
    return r[np.lexsort(r.T[::-1])]


def test_preprocess_mixed_sizes_equals_oracle(dev):
    """One call over frames of mixed sizes, pitch > 3 * width and odd bases, equals the oracle bit for bit; nothing around the
    output is written."""
    rng = np.random.default_rng(1)
    frames = [_frame(rng, w, h, dev, 13 + 3 * (w + 1) * (i % 2)) for i, (w, h) in enumerate(MIXED)]
    assert all(f.stride(0) > 3 * f.shape[1] for f in frames)
    n = len(frames) * 3 * 384 * 640
    big = torch.full((n + 8,), -7.0, dtype=torch.float32, device=dev)
    P.yolop_preprocess(frames, out=big[1:1 + n].view(len(frames), 3, 384, 640))  # 4-byte but not 16-byte aligned
    got = big.cpu().numpy()
    for i, f in enumerate(frames):
        want, _ = YO.preprocess(_host(f))
        assert np.array_equal(got[1:1 + n].reshape(-1, 3, 384, 640)[i], want), MIXED[i]
    assert got[0] == -7.0 and (got[1 + n:] == -7.0).all()


def test_preprocess_70_frames_and_all_bytes(dev):
    """More than one launch (64 frames each); a frame holding every byte value in every channel."""
    rng = np.random.default_rng(2)
    frames = [_frame(rng, 64 + 7 * i, 48 + 3 * i, dev, 0) for i in range(70)]
    allb = torch.from_numpy(np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(16, 16, 3).copy()).to(dev)
    frames[5] = allb
    out = P.yolop_preprocess(frames).cpu().numpy()
    for i in (0, 5, 63, 64, 69):
        assert np.array_equal(out[i], YO.preprocess(_host(frames[i]))[0]), i


def test_scan_vs_reference_kernel(dev):
    """YOLOP's YoloLayer (1 class, grids 20 x 12 / 40 x 24 / 80 x 48, YOLOP's anchors, stride-32 input first) through
    YoloLayerPluginV7 equals YOLOP's compiled plugin kernel as a set of rows (the reference's order is atomicAdd arrival)."""
    lib = G.lib("libref_yolop.so")
    assert lib is None or lib.ref_yolop_det_floats() == 6
    B = 4
    heads = _heads(B, 31)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    plug = P.YoloLayerPluginV7(1, 640, 384, 1000, _kernels())
    out = torch.full((B, plug.output_elems()), -5.0, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    got = out.cpu().numpy()
    ref = None
    if lib is not None:
        ks = np.zeros((3, 8), np.float32)
        ki = ks.view(np.int32)
        for l, k in enumerate(_kernels()):
            ki[l, 0], ki[l, 1] = k.width, k.height
            ks[l, 2:] = k.anchors
        r = torch.zeros((B, 1 + 1000 * 6), dtype=torch.float32, device=dev)
        assert lib.ref_yolop_plugin_enqueue(1, 640, 384, 1000, ks.ctypes.data_as(C.c_void_p), 3, B, _ptrs(hd),
                                            C.c_void_p(r.data_ptr()), None) == 0
        ref = r.cpu().numpy()
    assert 100 < got[:, 0].min() and got[:, 0].max() < 1000
    for b in range(B):
        G.equal(f"scan.rows{b}", _sorted_rows(got, b), None if ref is None else _sorted_rows(ref, b))
    _close_to_oracle_decode(heads, got)


def _close_to_oracle_decode(heads, got):
    """The oracle's decode (host expf, so within float rounding of the device's) has the same rows."""
    orc, _ = O.yolov5_decode(heads, [ANCHORS[{8: 0, 16: 1, 32: 2}[s]] for s in STRIDES], strides=STRIDES, net_h=384, nc=1,
                             det_floats=6)
    assert np.array_equal(orc[:, 0], got[:, 0])
    for b in range(got.shape[0]):
        np.testing.assert_allclose(_sorted_rows(got, b), _sorted_rows(orc, b), rtol=1e-5, atol=1e-5)


def _nms_rows(plugin_out, B):
    return P.batch_nms(plugin_out, B, plugin_out.shape[1], 0.25, 0.45, box_format=L.BOX_CXCYWH, det_floats=6, max_det=1000)


def test_nms_and_rows_vs_reference(dev):
    """batch_nms (CXCYWH, greedy) then the rows of yolop_postprocess equal YOLOP's compiled nms() and get_rect on the plugin
    rows of each frame, frames of mixed sizes."""
    ref = GH.lib("libref_yolop_host.so")
    B = 4
    hd = [torch.from_numpy(h).to(dev) for h in _heads(B, 41)]
    plug = P.YoloLayerPluginV7(1, 640, 384, 1000, _kernels())
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    comp = _nms_rows(out, B)
    sizes = MIXED[:B]
    rows, canv = P.yolop_postprocess(comp, sizes, max_rows=1000, labels=False)
    assert canv is None
    got = rows.cpu().numpy()
    host = out.cpu().numpy()
    for b, (w, h) in enumerate(sizes):
        assert got[b, 0] > 0
        live = None
        if ref is not None:
            res = np.zeros(1000 * 6, np.float32)
            k = ref.ref_yolop_nms(C.c_void_p(host[b].ctypes.data), C.c_float(0.25), C.c_float(0.45), C.c_void_p(res.ctypes.data))
            live = np.zeros(1 + 1000 * 6, np.float32)
            live[0] = k
            for i in range(k):
                r = np.zeros(4, np.int32)
                bb = np.ascontiguousarray(res[6 * i:6 * i + 4])
                ref.ref_yolop_get_rect(w, h, C.c_void_p(bb.ctypes.data), C.c_void_p(r.ctypes.data))
                live[1 + 6 * i:1 + 6 * i + 6] = [*r, res[6 * i + 4], res[6 * i + 5]]
        G.equal(f"rows{b}", got[b], live)
        res_o, _ = O.nms(1, host[b], 1000, 6, np.float32(0.25), np.float32(0.45))
        assert np.array_equal(got[b], YO.rows(res_o, w, h, 1000))


def _maps(B, seed):
    rng = np.random.default_rng(seed)
    seg = (rng.random((B, 360, 640)) < 0.5).astype(np.int32)
    lane = (rng.random((B, 360, 640)) < 0.15).astype(np.int32) * rng.integers(1, 3, (B, 360, 640), dtype=np.int32)
    return seg, lane


def _pitched_canvases(sizes, dev, fill=0xAB, extra=19):
    bufs = [torch.full((h, w + extra + 1), fill, dtype=torch.uint8, device=dev) for w, h in sizes]
    return bufs, [b[:, 1:1 + w] for b, (w, _) in zip(bufs, sizes)]


def test_labels_mixed_sizes_equal_oracle(dev):
    """Label canvases of frames of mixed sizes (views of pitched buffers from odd bases) equal the oracle; the bytes past
    img_w and before the base stay untouched; frame b reads maps b; 70 frames take two launches."""
    for sizes in (MIXED, [(17 + 29 * i, 9 + 16 * i) for i in range(70)]):
        B = len(sizes)
        seg, lane = _maps(B, 50 + B)
        dets = torch.zeros((B, 1 + 20 * 7), dtype=torch.float32, device=dev)
        bufs, views = _pitched_canvases(sizes, dev)
        P.yolop_postprocess(dets, sizes, max_rows=20, seg=torch.from_numpy(seg).to(dev), lane=torch.from_numpy(lane).to(dev),
                            canvases_out=views)
        for b, (w, h) in enumerate(sizes):
            buf = bufs[b].cpu().numpy()
            assert np.array_equal(buf[:, 1:1 + w], YO.labels(seg[b], lane[b], w, h)), (w, h)
            assert (buf[:, 0] == 0xAB).all() and (buf[:, 1 + w:] == 0xAB).all(), (w, h)


def test_rejected_calls_write_nothing(dev):
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 320, 180, dev, 5), _frame(rng, 5000, 1, dev, 0)]  # the second: an empty letterbox rectangle
    out = torch.full((2, 3, 384, 640), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.yolop_preprocess(frames, out=out)
    assert (out == 3.0).all()
    B = 2
    seg, lane = (torch.from_numpy(m).to(dev) for m in _maps(B, 4))
    dets = torch.zeros((B, 1 + 10 * 7), dtype=torch.float32, device=dev)
    dets[:, 0] = 3
    dets[:, 7::7] = 1
    rows = torch.full((B, 1 + 10 * 6), 9.0, dtype=torch.float32, device=dev)
    bufs, views = _pitched_canvases([(64, 32), (64, 32)], dev)
    fr = (L.Frame * 2)()
    for b in range(2):
        fr[b].img_w, fr[b].img_h, fr[b].masks_dev, fr[b].pitch = 64, 32, views[b].data_ptr(), int(views[b].stride(0))
    fr[1].pitch = 63  # < img_w
    q = L.YolopPostParams(640, 384, 640, 360, 7)
    lib = L.load()
    assert lib.trtx_yolop_postprocess_enqueue(C.byref(q), fr, B, dets.data_ptr(), 10, seg.data_ptr(), lane.data_ptr(),
                                              rows.data_ptr(), None) == L.ERR_INVALID
    torch.cuda.synchronize()
    assert (rows == 9.0).all() and all((b == 0xAB).all() for b in bufs)


def test_end_to_end_chain_and_graph_replay(dev):
    """Frames -> pre-process, and heads -> scan -> NMS -> post-process with labels, equal to the oracle chain (the scan within
    float rounding of the oracle's decode, everything after it bit for bit from the scan's rows); the pre- and
    post-process captured in a CUDA graph and replayed on new frames, rows and maps give the oracle's outputs for those."""
    B = 3
    rng = np.random.default_rng(9)
    sizes = [(1920, 1080), (1280, 720), (810, 1080)]
    frames = [_frame(rng, w, h, dev, 7) for w, h in sizes]
    plug = P.YoloLayerPluginV7(1, 640, 384, 1000, _kernels())
    hd = [torch.from_numpy(h).to(dev) for h in _heads(B, 61)]
    seg_np, lane_np = _maps(B, 62)
    seg, lane = torch.from_numpy(seg_np).to(dev), torch.from_numpy(lane_np).to(dev)
    inp = torch.empty((B, 3, 384, 640), dtype=torch.float32, device=dev)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    rows = torch.empty((B, 1 + 1000 * 6), dtype=torch.float32, device=dev)
    canv = [torch.zeros((h, w), dtype=torch.uint8, device=dev) for w, h in sizes]
    comp = torch.empty((B, 1 + 1000 * 7), dtype=torch.float32, device=dev)

    def step(stream=None):
        P.yolop_preprocess(frames, out=inp, stream=stream)
        assert plug.enqueue(B, hd, [out], ws, stream) == 0
        comp.copy_(_nms_rows(out, B))
        P.yolop_postprocess(comp, sizes, max_rows=1000, seg=seg, lane=lane, rows_out=rows, canvases_out=canv, stream=stream)

    def check():
        pre = inp.cpu().numpy()
        scan = out.cpu().numpy()
        _close_to_oracle_decode([h.cpu().numpy() for h in hd], scan)
        r = rows.cpu().numpy()
        for b, (w, h) in enumerate(sizes):
            assert np.array_equal(pre[b], YO.preprocess(_host(frames[b]))[0])
            res, _ = O.nms(1, scan[b], 1000, 6, np.float32(0.25), np.float32(0.45))
            assert np.array_equal(r[b], YO.rows(res, w, h, 1000))
            assert np.array_equal(canv[b].cpu().numpy(), YO.labels(seg[b].cpu().numpy(), lane[b].cpu().numpy(), w, h))

    step()
    torch.cuda.synchronize()
    check()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.yolop_preprocess(frames, out=inp)
        P.yolop_postprocess(comp, sizes, max_rows=1000, seg=seg, lane=lane, rows_out=rows, canvases_out=canv)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    for h in hd:
        h.add_(0.25)
    seg.copy_(torch.from_numpy(_maps(B, 63)[0]))
    assert plug.enqueue(B, hd, [out], ws) == 0
    comp.copy_(_nms_rows(out, B))
    g.replay()
    torch.cuda.synchronize()
    check()
