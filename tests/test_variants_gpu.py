"""SURVEY 8f rank 4 + row a2: the older / other plugin variants through the same scan / pack / NMS kernels, each against
(1) the REFERENCE'S OWN plugin compiled into oracle/_ref (same GPU, same inputs; where it was not built, its outputs of an
H100 run stored in tests/golden/ref_gpu.npz) and (2) the CPU oracle:
  yolov7   6-float Detection rows            yolov7/plugin/yololayer.cu:152-200, yolov7/include/types.h:11-16
  yolov3   exp-wh, dual confidence, 7 floats yolov3-spp/yololayer.cu:148-191
  yolo26   NMS-free gatherKernel, AoS input  yolo26/plugin/yololayer.cu:178-245
  retinafaceAntiCov  16-float rows           retinafaceAntiCov/decode.cu:110-172
The references' slot order is atomicAdd arrival: rows are compared as canonically sorted sets."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_gpu")
ATOL = 1e-4
V3_ANCHORS = [k.anchors for k in P.YOLOV3_KERNELS]


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _canon(rows):
    if rows is None:
        return None
    return rows[np.lexsort(tuple(rows[:, k] for k in range(rows.shape[1] - 1, -1, -1)))]


def _rows(buf, b, F, n=None):
    if buf is None:
        return None
    n = int(buf[b, 0]) if n is None else n
    return buf[b, 1:1 + n * F].reshape(n, F)


# ------------------------------------------------------------------ yolov7: 6-float rows -----------------
def _v7_kernels():
    return [P.YoloKernel(640 // s, 640 // s, a) for s, a in zip((8, 16, 32), synth.V5_ANCHORS)]


def test_yolov7_6_float_rows_vs_reference_kernel_and_oracle(oracle, dev):
    lib = G.lib("libref_yolov7.so")
    assert lib is None or lib.ref_v7_det_floats() == 6
    B = 3
    heads = synth.yolov5_heads(B, seed=610)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    ref = None
    if lib is not None:
        ks = np.zeros((3, 8), np.float32)
        ki = ks.view(np.int32)
        for l, (s, a) in enumerate(zip((8, 16, 32), synth.V5_ANCHORS)):
            ki[l, 0], ki[l, 1] = 640 // s, 640 // s
            ks[l, 2:] = a
        ref = torch.zeros((B, 1 + 1000 * 6), dtype=torch.float32, device=dev)
        assert lib.ref_v7_plugin_enqueue(80, 640, 640, 1000, ks.ctypes.data_as(C.c_void_p), 3, B, _ptrs(hd),
                                         C.c_void_p(ref.data_ptr()), None) == 0
        ref = ref.cpu().numpy()
    plug = P.YoloLayerPluginV7(80, 640, 640, 1000, _v7_kernels())
    out = torch.full((B, plug.output_elems()), -5.0, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    got = out.cpu().numpy()
    orc, _ = oracle.yolov5_decode(heads, synth.V5_ANCHORS, det_floats=6)
    G.equal("v7_plugin.count", got[:, 0], None if ref is None else ref[:, 0])
    assert np.array_equal(orc[:, 0], got[:, 0]) and got[:, 0].min() > 100
    for b in range(B):
        G.close(f"v7_plugin.{b}", _canon(_rows(got, b, 6)), _canon(_rows(ref, b, 6)), rtol=3e-7, atol=0)  # FMA contraction
        np.testing.assert_allclose(_rows(got, b, 6), _rows(orc, b, 6), atol=ATOL, rtol=2e-6)                  # anchor order
        assert np.all(got[b, 1 + int(got[b, 0]) * 6:] == -5.0)   # nothing written past the rows
    # serialization layout of yolov7/plugin/yololayer.cu:62-77 round-trips
    q = P.YoloLayerPluginV7.deserialize(plug.serialize())
    assert q.serialize() == plug.serialize() and len(plug.serialize()) == plug.getSerializationSize()


# ------------------------------------------------------------------ yolov3 / v3-spp / v4 -----------------
@pytest.mark.parametrize("net,B", [((608, 608), 2), ((416, 352), 3)])
def test_yolov3_vs_reference_kernel_and_oracle(oracle, dev, net, B):
    lib = G.lib("libref_yolov3.so")
    assert lib is None or (lib.ref_v3_det_floats() == 7 and lib.ref_v3_num_classes() == 80)
    heads = synth.yolov3_heads(B, seed=620 + B, net_w=net[0], net_h=net[1])
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    ref = None
    if lib is not None:
        gh = (C.c_int * 3)(*[h.shape[2] for h in heads])
        gw = (C.c_int * 3)(*[h.shape[3] for h in heads])
        ref = torch.zeros((B, 1 + 1000 * 7), dtype=torch.float32, device=dev)
        assert lib.ref_v3_plugin_enqueue(B, gh, gw, _ptrs(hd), C.c_void_p(ref.data_ptr())) == 0
        ref = ref.cpu().numpy()
    plug = P.YoloLayerPluginV3()
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    assert plug.enqueue(hd, [out]) == 0
    got = out.cpu().numpy()
    orc, orc_idx = oracle.yolov3_decode(heads, V3_ANCHORS)
    key = f"v3_plugin.{net[0]}x{net[1]}"
    G.equal(key + ".count", got[:, 0], None if ref is None else ref[:, 0])
    assert np.array_equal(orc[:, 0], got[:, 0]) and got[:, 0].min() > 50
    n_class_gated = 0
    for b in range(B):
        r, g = _canon(_rows(ref, b, 7)), _canon(_rows(got, b, 7))
        G.equal(f"{key}.{b}.conf_class", g[:, 4:], None if r is None else r[:, 4:])      # both confidences and the class: bit-exact
        # same expf; FMA contraction of the reference build
        G.close(f"{key}.{b}.box", g[:, :4], None if r is None else r[:, :4], rtol=3e-7, atol=0)
        np.testing.assert_allclose(_rows(got, b, 7), _rows(orc, b, 7), atol=ATOL, rtol=2e-6)
        n_class_gated += int((_rows(got, b, 7)[:, 6] < 0.5).sum())
    assert n_class_gated > 0
    # fused decode + NMS == oracle nms() of yolov3-spp.cpp:77-120 (cxcywh IoU, det_confidence order): variant 1 on 7-float rows
    fused = P.FusedYoloDecodeNms(plug, B, 0.5, 0.4, device=dev)
    comp, idx = fused.enqueue(B, hd)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(1, orc[b], 1000, 7, 0.5, 0.4)
        n = int(comp[b, 0])
        assert n == len(res) and n > 5
        assert np.array_equal(idx[b, :n], orc_idx[b][src])
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=2e-6)
    q = P.YoloLayerPluginV3.deserialize(plug.serialize())
    assert q.serialize() == plug.serialize() and len(plug.serialize()) == plug.getSerializationSize()


# ------------------------------------------------------------------ yolo26 gather -------------------------
@pytest.mark.parametrize("obb", [False, True])
def test_yolo26_gather_vs_reference_kernel_and_oracle(oracle, dev, obb):
    lib = G.lib("libref_yolo26.so")
    assert lib is None or lib.ref_v26_det_floats() == 90
    nc, A, K, B = (15, 21504, 300, 3) if obb else (80, 8400, 300, 3)
    rows = synth.yolo26_rows(B, seed=630 + int(obb), nc=nc, anchors=A, obb=obb)
    rd = torch.from_numpy(rows).to(dev)
    plug = P.YoloLayerPlugin26(nc, 17, K, not obb, False, False, obb, A, conf_thresh=0.3)
    out = torch.full((B, plug.output_elems()), 7.0, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [rd], [out], ws) == 0
    got = out.cpu().numpy()
    orc, orc_idx = oracle.yolo26_gather(rows, nc=nc, obb=obb, max_out=K, conf_thresh=0.3)
    assert np.array_equal(got, orc)          # pure gather: every float of the buffer, ascending anchor order, zeros elsewhere
    assert 30 < got[:, 0].min() <= got[:, 0].max() <= K
    # the reference decodes image 0 of the batch only (yololayer.cu:185): one image at a time against it
    for b in range(B):
        ref = None
        if lib is not None:
            ref = torch.full((1, 1 + K * 90), 3.0, dtype=torch.float32, device=dev)
            assert lib.ref_v26_plugin_enqueue(nc, 17, K, int(not obb), int(obb), A, C.c_float(0.3), C.c_void_p(rd[b].data_ptr()),
                                              C.c_void_p(ref.data_ptr()), None) == 0
            ref = ref.cpu().numpy()
            assert np.all(ref[0, 1 + int(ref[0, 0]) * 90:] == 0)   # the reference clears its whole buffer
        key = f"v26_plugin.{int(obb)}.{b}"
        G.equal(key + ".count", got[b, :1], None if ref is None else ref[0, :1])
        G.equal(key, _canon(_rows(got, b, 90)), _canon(_rows(ref, 0, 90)))
    q = P.YoloLayerPlugin26.deserialize(plug.serialize())
    assert q.serialize() == plug.serialize() and len(plug.serialize()) == 24


def test_yolo26_gather_overflow_unaligned_and_empty(oracle, dev):
    # more candidates than max_detections (count clamped, first K in anchor order), a channel count that is not a multiple of
    # 4 (scalar load path), an anchor count that is not a multiple of 32, and an image without candidates
    nc, A, K, B = 3, 1000 + 13, 50, 2
    rows = synth.yolo26_rows(B, seed=640, nc=nc, anchors=A, n_obj=200)
    rows[1, :, 4:] = 0.01
    plug = P.YoloLayerPlugin26(nc, 17, K, True, False, False, False, A, conf_thresh=0.3)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(rows).to(dev)], [out], ws) == 0
    got = out.cpu().numpy()
    orc, _ = oracle.yolo26_gather(rows, nc=nc, max_out=K, conf_thresh=0.3)
    assert orc[0, 0] > K and got[0, 0] == K and got[1, 0] == 0
    assert np.array_equal(got[:, 1:], orc[:, 1:])


# ------------------------------------------------------------------ retinafaceAntiCov ---------------------
def test_anticov_decode_vs_reference_kernel_and_oracle(oracle, dev):
    lib = G.lib("libref_anticov.so")
    assert lib is None or (lib.ref_anticov_input_h(), lib.ref_anticov_input_w(), lib.ref_anticov_det_floats()) == (640, 640, 16)
    B = 3
    heads = synth.anticov_heads(B, seed=650)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    plug = P.DecodePlugin(640, 640, anticov=True)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    got = out.cpu().numpy()
    orc, _ = oracle.anticov_decode(heads)
    assert np.array_equal(got[:, 0], orc[:, 0]) and got[:, 0].min() > 50
    for b in range(B):
        np.testing.assert_allclose(_rows(got, b, 16), _rows(orc, b, 16), atol=ATOL, rtol=2e-6)
        # the reference is batch 1 only (no image offset): image by image
        ref = None
        if lib is not None:
            one = [h[b:b + 1].contiguous() for h in hd]
            ref = torch.zeros((1, plug.output_elems()), dtype=torch.float32, device=dev)
            assert lib.ref_anticov_plugin_enqueue(_ptrs(one), C.c_void_p(ref.data_ptr())) == 0
            ref = ref.cpu().numpy()
        G.equal(f"anticov_plugin.{b}.count", got[b, :1], None if ref is None else ref[0, :1])
        # same expf, same contraction: bit-exact
        G.equal(f"anticov_plugin.{b}", _canon(_rows(got, b, 16)), _canon(_rows(ref, 0, 16)))
    # NMS of retinafaceAntiCov.cpp:92-127 = the retinaface host nms() on 16-float rows (landmarks + mask conf ride along)
    comp, idx = P.batch_nms(out, B, plug.output_elems(), P.float_le_threshold(0.1), 0.4, det_floats=16, box_format=L.BOX_RETINA,
                            extra_floats=11, extra_offset=5, max_det=1000, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(2, got[b], plug.total_priors, 16, 0.1, 0.4)
        n = int(comp[b, 0])
        assert n == len(res) and np.array_equal(idx[b, :n], src)
        rows = comp[b, 1:1 + n * 18].reshape(n, 18)
        assert np.array_equal(rows[:, :5], res[:, :5]) and np.array_equal(rows[:, 7:], res[:, 5:])
