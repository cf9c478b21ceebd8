"""The yolov3 family's decode on the device (TRTX_YOLO_V3_NET: yolov3, yolov3-tiny; TRTX_YOLO_V4: yolov4; TRTX_YOLO_V4_CSP:
scaled-yolov4), each against
(1) that driver's OWN compiled YoloLayer kernel (oracle/_ref/libref_v3f_<driver>.so, same GPU, same inputs; where it was not
    built, its outputs stored in tests/golden/ref_v3f_gpu.npz): count, class, both confidences and the box, bit for bit,
    after a canonical sort (the reference's row order is atomicAdd arrival);
(2) the CPU oracle's decode + that driver's NMS parameters, through every entry point: the plugin decode, the fused
    decode + NMS and the split scan + NMS, fp32 and fp16 heads;
and the TensorRT creators enqueued through tests/trt_adapter_v3_family_check.cpp --gpu.
Other grids (non-square, odd cell counts, two levels), class counts, scan routes and edge logits: the family's rows of
tests/test_yolo_scan_paths_gpu.py, against the same drivers' kernels built from a blob."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

from oracle import v3family as V
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

from test_yolov3_family_cpu import DRIVERS, LIBNAME, _build_check

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_v3f_gpu")
ATOL = 1e-4


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _canon(rows):
    return rows[np.lexsort(tuple(rows[:, k] for k in range(rows.shape[1] - 1, -1, -1)))]


def _rows(buf, b, n=None):
    n = int(buf[b, 0]) if n is None else n
    return buf[b, 1:1 + n * 7].reshape(n, 7)


def _heads(d, B, seed):
    """Seeded heads at the driver's compiled-in shapes: objectness N(-9, 3) (some 1 % of the anchors pass the gate, a few
    per image pass the NMS threshold), class logits N(-5, 2) (the best class probability spans the class gate and 0.5)."""
    rng = np.random.default_rng(seed)
    out = []
    for w, h, _ in d["kernels"]:
        x = rng.normal(-5.0, 2.0, size=(B, 3, 85, h, w)).astype(np.float32)
        x[:, :, 4] = rng.normal(-9.0, 3.0, size=(B, 3, h, w))
        out.append(x.reshape(B, 3 * 85, h, w))
    return out


def _oracle(oracle, driver, heads, max_out=1000):
    d = P.V3_FAMILY_DRIVERS[driver]
    return V.decode(heads, [a for _, _, a in d["kernels"]], box_mode=d["variant"], net=d["net"], max_out=max_out)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("driver", DRIVERS)
def test_plugin_rows_equal_driver_kernel(oracle, dev, driver, B):
    lib = G.lib(f"libref_v3f_{LIBNAME[driver]}.so")
    d = P.V3_FAMILY_DRIVERS[driver]
    heads = _heads(d, B, seed=800 + B + 10 * d["variant"])
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    plug = P.YoloLayerPluginV3Net.for_driver(driver)
    ref = None
    if lib is not None:
        wh = (C.c_int * 2)()
        lib.ref_v3f_net(wh)
        assert (tuple(wh), lib.ref_v3f_num_classes(), lib.ref_v3f_max_out(), lib.ref_v3f_det_floats()) == \
            (d["net"], d["classes"], d["max_out"], 7)
        buf = (C.c_ubyte * 256)()
        n = lib.ref_v3f_serialize(buf, 256)
        assert bytes(buf[:n]) == plug.serialize()      # the reference constructor's own blob
        rt = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
        assert lib.ref_v3f_plugin_enqueue(B, _ptrs(hd), C.c_void_p(rt.data_ptr())) == 0
        ref = rt.cpu().numpy()
    out = torch.full((B, plug.output_elems()), -5.0, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    got = out.cpu().numpy()
    orc, _ = _oracle(oracle, driver, heads)
    key = f"{driver}.b{B}"
    G.equal(key + ".count", got[:, 0], None if ref is None else ref[:, 0])
    assert np.array_equal(orc[:, 0], got[:, 0]) and 20 < got[:, 0].min() and got[:, 0].max() < 1000
    n_class_gated = 0
    for b in range(B):
        g = _canon(_rows(got, b))
        r = None if ref is None else _canon(_rows(ref, b))
        G.equal(f"{key}.{b}", g, r)                  # box, det_confidence, class, class_confidence: bit for bit
        np.testing.assert_allclose(_rows(got, b), _rows(orc, b), atol=ATOL, rtol=2e-6)   # ascending anchor order
        assert np.all(got[b, 1 + int(got[b, 0]) * 7:] == -5.0)
        n_class_gated += int((_rows(got, b)[:, 6] < 0.5).sum())
    assert n_class_gated > 0                          # rows whose class confidence sits between the gate and 0.5


@pytest.mark.parametrize("driver", DRIVERS)
def test_every_entry_point_equals_oracle_decode_and_driver_nms(oracle, dev, driver):
    d = P.V3_FAMILY_DRIVERS[driver]
    B = 3
    heads = _heads(d, B, seed=820 + d["variant"])
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    orc, orc_idx = _oracle(oracle, driver, heads)
    results = {}
    for dtype in (L.F32, L.F16):
        hx = hd if dtype == L.F32 else [h.half() for h in hd]
        plug = P.YoloLayerPluginV3Net.for_driver(driver, in_dtype=dtype)
        out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
        ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
        assert plug.enqueue(B, hx, [out], ws) == 0
        fused = P.FusedYoloDecodeNms(plug, B, d["conf_thresh"], d["nms_thresh"], device=dev)
        assert fused.q.box_format == L.BOX_CXCYWH
        comp, idx = fused.enqueue(B, hx)
        comp, idx = comp.clone().cpu().numpy(), idx.clone().cpu().numpy()
        fused.enqueue_scan(B, hx)
        comp2, idx2 = fused.enqueue_nms(B, hx)
        assert np.array_equal(comp, comp2.cpu().numpy()) and np.array_equal(idx, idx2.cpu().numpy())
        results[dtype] = (out.cpu().numpy(), comp, idx)
    # fp16 heads = the fp32 decode of the widened halves
    wide = [h.half().float() for h in hd]
    plug = P.YoloLayerPluginV3Net.for_driver(driver)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, wide, [out], ws) == 0
    fused = P.FusedYoloDecodeNms(plug, B, d["conf_thresh"], d["nms_thresh"], device=dev)
    comp_w, idx_w = fused.enqueue(B, wide)
    assert np.array_equal(results[L.F16][0], out.cpu().numpy())
    assert np.array_equal(results[L.F16][1], comp_w.cpu().numpy()) and np.array_equal(results[L.F16][2], idx_w.cpu().numpy())
    got, comp, idx = results[L.F32]
    assert comp[:, 0].sum() > 20
    for b in range(B):
        res, src = oracle.nms(1, orc[b], 1000, 7, d["conf_thresh"], d["nms_thresh"])
        n = int(comp[b, 0])
        assert n == len(res) and n > 0
        assert np.array_equal(idx[b, :n], orc_idx[b][src])
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=2e-6)
        # the NMS over the plugin buffer keeps the same rows as the fused call
        pc, pi = P.batch_nms(torch.from_numpy(got[b:b + 1]).to(dev), 1, got.shape[1], d["conf_thresh"], d["nms_thresh"],
                             box_format=L.BOX_CXCYWH, det_floats=7, max_det=1000, return_index=True)
        assert np.array_equal(pc.cpu().numpy()[0, :1 + n * 7], comp[b, :1 + n * 7])


@pytest.mark.parametrize("driver", ["yolov3", "scaled-yolov4"])
def test_more_candidates_than_max_out_keeps_the_first_in_anchor_order(oracle, dev, driver):
    d = P.V3_FAMILY_DRIVERS[driver]
    B, K = 2, 60
    heads = _heads(d, B, seed=840)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    kern = [P.YoloKernel(w, h, a) for w, h, a in d["kernels"]]
    plug = P.YoloLayerPluginV3Net(d["classes"], kern, d["net"][0], d["net"][1], d["variant"], maxOut=K)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    got = out.cpu().numpy()
    full, _ = _oracle(oracle, driver, heads)
    orc, _ = _oracle(oracle, driver, heads, max_out=K)
    assert full[:, 0].min() > K and np.all(got[:, 0] == K)
    for b in range(B):
        np.testing.assert_allclose(_rows(got, b), _rows(orc, b, K), atol=ATOL, rtol=2e-6)
    fused = P.FusedYoloDecodeNms(plug, B, d["conf_thresh"], d["nms_thresh"], device=dev)
    comp, idx = fused.enqueue(B, hd)
    comp = comp.cpu().numpy()
    for b in range(B):
        res, _ = oracle.nms(1, orc[b], K, 7, d["conf_thresh"], d["nms_thresh"])
        assert int(comp[b, 0]) == len(res)


def test_family_creators_enqueue_on_gpu(tmp_path, dev):
    exe = _build_check(tmp_path)
    r = subprocess.run([str(exe), "--gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "gpu enqueue ok" in r.stdout
