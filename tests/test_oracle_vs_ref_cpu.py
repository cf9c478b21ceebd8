"""Pins the oracle's NMS restatements against the REFERENCE's OWN host code: oracle/_ref/libref_*_host.so are
built by oracle/Makefile from the reference's {yolov8,yolov5}/src/postprocess.cpp and retinaface/common.hpp,
compiled where they lie (with header shims for the OpenCV / TensorRT includes those files pull in).
Where oracle/_ref was not built, the reference's outputs come from tests/golden/ref_host_calls.npz (oracle/golden.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle.golden import RefOutputs
from tensorrtx_b200 import synth

G = RefOutputs("ref_host_calls")


def _fn(lib, name):
    return None if lib is None else getattr(lib, name)


def _ref_nms(fn, buf, F, *thr):
    if fn is None:
        return None
    out = np.zeros((buf.shape[0] // F + 1) * F, np.float32)
    b = np.ascontiguousarray(buf, np.float32)
    n = fn(b.ctypes.data_as(C.c_void_p), *[C.c_float(t) for t in thr], out.ctypes.data_as(C.c_void_p))
    return out[:n * F].reshape(n, F).copy()


@pytest.mark.parametrize("seed", range(4))
def test_v8_nms_equals_reference(oracle, seed):
    lib = G.lib("libref_yolov8_host.so")
    assert lib is None or lib.ref_v8_det_floats() == 90
    heads = synth.yolov8_heads(2, seed=100 + seed)
    out, _ = oracle.yolov8_decode(heads)
    for b in range(2):
        mine, _ = oracle.nms(0, out[b], 1000, 90, 0.5, 0.45)
        ref = _ref_nms(_fn(lib, "ref_v8_nms"), out[b], 90, 0.5, 0.45)
        G.equal(f"v8_nms.{seed}.{b}", mine, ref)  # same rows, same order (class asc, conf desc), bit for bit
        assert len(mine) > 20


def _obb_plugin_rows(oracle, seed, B=2):
    heads = synth.yolov8_heads(B, seed=seed, nc=15, extra=1, n_obj=40)
    out, _ = oracle.yolov8_decode(heads, nc=15, is_obb=True)
    return out


@pytest.mark.parametrize("seed", range(3))
def test_v8_nms_obb_equals_reference(oracle, seed):
    """nms_obb + probiou (mixed float/double C++ promotions): identical rows in identical order."""
    lib = G.lib("libref_yolov8_host.so")
    out = _obb_plugin_rows(oracle, 130 + seed)
    for b in range(out.shape[0]):
        for thr in (0.5, 0.2):
            mine, _ = oracle.nms(3, out[b], 1000, 90, 0.3, thr)
            ref = _ref_nms(_fn(lib, "ref_v8_nms_obb"), out[b], 90, 0.3, thr)
            G.equal(f"v8_nms_obb.{seed}.{b}.{thr}", mine, ref)
            assert len(mine) > 10 and len(mine) < int(out[b, 0])


def test_v8_nms_ties_broken_by_bbox0_like_reference(oracle):
    lib = G.lib("libref_yolov8_host.so")
    rng = np.random.default_rng(1)
    n = 400
    buf = np.zeros(1 + 1000 * 90, np.float32)
    rows = buf[1:1 + n * 90].reshape(n, 90)
    xy = rng.uniform(0, 600, (n, 2))
    wh = rng.uniform(10, 60, (n, 2))
    rows[:, :2], rows[:, 2:4] = xy, xy + wh
    rows[:, 4] = np.round(rng.uniform(0.5, 1.0, n), 2)  # many equal confidences, distinct bbox[0]
    rows[:, 5] = rng.integers(0, 3, n)
    buf[0] = n
    mine, _ = oracle.nms(0, buf, 1000, 90, 0.5, 0.45)
    G.equal("v8_nms_ties", mine, _ref_nms(_fn(lib, "ref_v8_nms"), buf, 90, 0.5, 0.45))


def test_v8_batch_nms_and_thresholds(oracle):
    lib = G.lib("libref_yolov8_host.so")
    heads = synth.yolov8_heads(3, seed=7)
    out, _ = oracle.yolov8_decode(heads)
    res, cnt = None, None
    if lib is not None:
        res = np.zeros((3, 1000, 90), np.float32)
        cnt = np.zeros(3, np.int32)
        lib.ref_v8_batch_nms(np.ascontiguousarray(out).ctypes.data_as(C.c_void_p), 3, out.shape[1], C.c_float(0.3),
                             C.c_float(0.6), res.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), 1000)
    for b in range(3):
        mine, _ = oracle.nms(0, out[b], 1000, 90, 0.3, 0.6)
        G.equal(f"v8_batch_nms.{b}", mine, None if lib is None else res[b, :cnt[b]])


@pytest.mark.parametrize("seed", range(3))
def test_v5_nms_equals_reference(oracle, seed):
    lib = G.lib("libref_yolov5_host.so")
    assert lib is None or lib.ref_v5_det_floats() == 38
    heads = synth.yolov5_heads(1, seed=200 + seed, n_obj=200)
    out, _ = oracle.yolov5_decode(heads, synth.V5_ANCHORS)
    mine, _ = oracle.nms(1, out[0], 1000, 38, 0.5, 0.45)
    G.equal(f"v5_nms.{seed}", mine, _ref_nms(_fn(lib, "ref_v5_nms"), out[0], 38, 0.5, 0.45))
    assert len(mine) > 50


@pytest.mark.parametrize("seed", range(3))
def test_retina_nms_equals_reference(oracle, seed):
    lib = G.lib("libref_retina_host.so")
    heads = synth.retina_heads(1, seed=300 + seed, in_h=480, in_w=640, n_obj=60)
    out, _ = oracle.retina_decode(heads, in_h=480, in_w=640)
    tp = oracle.retina_total_priors(480, 640)
    mine, _ = oracle.nms(2, out[0], tp, 15, 0.1, 0.4)
    G.equal(f"retina_nms.{seed}", mine, _ref_nms(_fn(lib, "ref_retina_nms"), out[0], 15, 0.4))
    assert len(mine) > 20


def test_retina_conf_threshold_is_a_double_compare(oracle):
    """`output[..] <= 0.1` compares against the DOUBLE 0.1: conf == 0.1f (> 0.1) is kept (common.hpp:113)."""
    lib = G.lib("libref_retina_host.so")
    tp = oracle.retina_total_priors(480, 640)
    buf = np.zeros(1 + tp * 15, np.float32)
    buf[0] = 3
    for i, c in enumerate([np.float32(0.1), np.nextafter(np.float32(0.1), np.float32(0)), np.float32(0.5)]):
        buf[1 + i * 15:1 + i * 15 + 4] = [100 * i, 0, 100 * i + 50, 50]
        buf[1 + i * 15 + 4] = c
    mine, _ = oracle.nms(2, buf, tp, 15, 0.1, 0.4)
    G.equal("retina_conf_double", mine, _ref_nms(_fn(lib, "ref_retina_nms"), buf, 15, 0.4))
    assert len(mine) == 2


@pytest.mark.parametrize("variant,libname,fn", [(0, "libref_yolov8_host.so", "ref_v8_get_rect"),
                                                (1, "libref_yolov5_host.so", "ref_v5_get_rect")])
def test_get_rect_equals_reference(oracle, variant, libname, fn):
    """get_rect (box in 640x640 network pixels -> cv::Rect in the original image): the reference's compiled host code vs
    the oracle vs the library's host function trtx_get_rect -- identical integers on 4000 boxes and 8 image sizes."""
    from tensorrtx_b200 import plugins as P
    lib = G.lib(libname)
    rng = np.random.default_rng(50 + variant)
    orc, mine, refs = [], [], []
    for (w, h) in ((1920, 1080), (1080, 1920), (640, 640), (1280, 720), (333, 777), (4000, 3000), (641, 640), (50, 60)):
        for _ in range(500):
            if variant == 0:
                x1, y1 = rng.uniform(-30, 650, 2)
                bb = np.array([x1, y1, x1 + rng.uniform(-5, 400), y1 + rng.uniform(-5, 400)], np.float32)
            else:
                bb = np.array([rng.uniform(-30, 670), rng.uniform(-30, 670), rng.uniform(0, 500), rng.uniform(0, 500)], np.float32)
            if lib is not None:
                ref = np.zeros(4, np.int32)
                getattr(lib, fn)(w, h, bb.ctypes.data_as(C.c_void_p), ref.ctypes.data_as(C.c_void_p))
                refs.append(ref)
            orc.append(oracle.get_rect(variant, w, h, bb))
            mine.append(P.get_rect(w, h, bb, variant=variant))
    ref = np.array(refs) if lib is not None else None
    G.equal(f"get_rect.{variant}", np.array(orc, np.int32), ref)
    G.equal(f"get_rect.{variant}", np.array(mine, np.int32), ref)


SIZES = ((1920, 1080), (1080, 1920), (640, 640), (1280, 720), (333, 777), (4000, 3000), (641, 640), (50, 60))


def test_get_rect_adapt_landmark_equals_reference():
    """get_rect_adapt_landmark (yolov8/src/postprocess.cpp:38-69, pose models): box AND the 17 keypoints mapped back to the
    original image -- the library's host function against the reference's compiled code, identical integers and identical
    keypoint bits on 300 boxes x 8 image sizes."""
    from tensorrtx_b200 import plugins as P
    lib = G.lib("libref_yolov8_host.so")
    rng = np.random.default_rng(70)
    rects, lmks, ref_rects, ref_lmks = [], [], [], []
    for (w, h) in SIZES:
        for _ in range(300):
            x1, y1 = rng.uniform(-30, 650, 2)
            bb = np.array([x1, y1, x1 + rng.uniform(-5, 400), y1 + rng.uniform(-5, 400)], np.float32)
            lmk = rng.uniform(-20, 660, 51).astype(np.float32)
            lmk[2::3] = rng.uniform(0, 1, 17).astype(np.float32)
            if lib is not None:
                ref_l, ref_r = lmk.copy(), np.zeros(4, np.int32)
                lib.ref_v8_get_rect_adapt_landmark(w, h, bb.copy().ctypes.data_as(C.c_void_p), ref_l.ctypes.data_as(C.c_void_p),
                                                   ref_r.ctypes.data_as(C.c_void_p))
                ref_rects.append(ref_r), ref_lmks.append(ref_l)
            rect, mapped = P.get_rect_adapt_landmark(w, h, bb, lmk)
            rects.append(rect), lmks.append(np.asarray(mapped, np.float32))
    G.equal("v8_lmk.rects", np.array(rects, np.int32), np.array(ref_rects) if lib is not None else None)
    G.equal("v8_lmk.points", np.array(lmks), np.array(ref_lmks) if lib is not None else None)


def test_scale_mask_rect_and_process_decode_rows_equal_reference():
    """scale_mask's crop of the 640x640 mask and its target size (postprocess.cpp:207-226; read back from the OpenCV shim) and
    process_decode_ptr_host (:131-147) -- the library's host functions against the reference's compiled code."""
    from tensorrtx_b200 import _lib as L
    ref = G.lib("libref_yolov8_host.so")
    lib = L.load()
    mine_r, ref_r = [], []
    for w in list(range(37, 2000, 97)) + [640, 641, 1920, 1080]:
        for h in (48, 479, 480, 640, 1080, 1920, 3000):
            mine = (C.c_int * 4)()
            assert lib.trtx_scale_mask_rect(640, 640, w, h, mine) == 0
            mine_r.append(list(mine) + [w, h])
            if ref is not None:
                r6 = np.zeros(6, np.int32)
                ref.ref_v8_scale_mask_rect(w, h, r6.ctypes.data_as(C.c_void_p))
                ref_r.append(r6)
    G.equal("scale_mask_rect", np.array(mine_r, np.int32), np.array(ref_r) if ref is not None else None)
    rng = np.random.default_rng(71)
    K = 200
    buf = np.zeros(1 + K * 7, np.float32)
    buf[0] = K
    rows = buf[1:].reshape(K, 7)
    rows[:, :6] = rng.uniform(0, 640, (K, 6)).astype(np.float32)
    rows[:, 6] = rng.integers(0, 2, K)
    out_mine = np.zeros((K, 6), np.float32)
    n = lib.trtx_process_decode_ptr_host(buf.ctypes.data_as(C.POINTER(C.c_float)), 7, K, out_mine.ctypes.data_as(C.POINTER(C.c_float)))
    out_ref = None
    if ref is not None:
        out_ref = np.zeros((K, 6), np.float32)
        n_ref = ref.ref_v8_process_decode_ptr_host(buf.ctypes.data_as(C.c_void_p), 7, K, out_ref.ctypes.data_as(C.c_void_p))
        assert n == n_ref
    assert n == int(rows[:, 6].sum())
    G.equal("process_decode_ptr_host", out_mine, out_ref)


def test_process_decode_ptr_host_obb_equals_reference():
    """process_decode_ptr_host_obb (yolov8/src/postprocess.cpp:273-290): kept rows of the oriented-box compact buffer (8-float rows,
    angle in column 7) -- the library's host function against the reference's compiled code."""
    from tensorrtx_b200 import _lib as L
    ref = G.lib("libref_yolov8_host.so")
    lib = L.load()
    rng = np.random.default_rng(72)
    for elem in (8, 9):
        K = 150
        buf = np.zeros(1 + K * elem, np.float32)
        buf[0] = K
        rows = buf[1:].reshape(K, elem)
        rows[:, :] = rng.uniform(-3, 640, (K, elem)).astype(np.float32)
        rows[:, 6] = rng.integers(0, 3, K)                  # keep flags 0, 1, 2: only == 1 is kept
        out_mine = np.zeros((K, 7), np.float32)
        n = lib.trtx_process_decode_ptr_host_obb(buf.ctypes.data_as(C.POINTER(C.c_float)), elem, K, out_mine.ctypes.data_as(C.POINTER(C.c_float)))
        out_ref = None
        if ref is not None:
            out_ref = np.zeros((K, 7), np.float32)
            n_ref = ref.ref_v8_process_decode_ptr_host_obb(buf.ctypes.data_as(C.c_void_p), elem, K, out_ref.ctypes.data_as(C.c_void_p))
            assert n == n_ref
        assert n == int((rows[:, 6] == 1).sum()) and n > 20
        G.equal(f"process_decode_ptr_host_obb.{elem}", out_mine, out_ref)
    assert lib.trtx_process_decode_ptr_host_obb(buf.ctypes.data_as(C.POINTER(C.c_float)), 7, K, out_mine.ctypes.data_as(C.POINTER(C.c_float))) < 0


def test_retina_get_rect_adapt_landmark_equals_reference():
    """RetinaFace's get_rect_adapt_landmark (retinaface/common.hpp:65-89: box corners truncated to int, 5 landmark pairs mapped in
    place) -- the library's host function against the reference's compiled code: identical integers and landmark bits on 250 faces
    x 8 image sizes, for the 640x640 network of BASELINE config 3 and the 480x640 one the reference compiles in."""
    from tensorrtx_b200 import _lib as L
    ref = G.lib("libref_retina_host.so")
    lib = L.load()
    rng = np.random.default_rng(73)
    rects, lmks, ref_rects, ref_lmks = [], [], [], []
    for (in_w, in_h) in ((640, 640), (640, 480)):
        for (w, h) in SIZES:
            for _ in range(250):
                x1, y1 = rng.uniform(-30, in_w + 10), rng.uniform(-30, in_h + 10)
                bb = np.array([x1, y1, x1 + rng.uniform(-5, 400), y1 + rng.uniform(-5, 400)], np.float32)
                lmk = rng.uniform(-20, 660, 10).astype(np.float32)
                if ref is not None:
                    l_ref, r_ref = lmk.copy(), np.zeros(4, np.int32)
                    ref.ref_retina_get_rect_adapt_landmark(w, h, in_w, in_h, bb.copy().ctypes.data_as(C.c_void_p),
                                                           l_ref.ctypes.data_as(C.c_void_p), r_ref.ctypes.data_as(C.c_void_p))
                    ref_rects.append(r_ref), ref_lmks.append(l_ref)
                l_mine, r_mine = lmk.copy(), (C.c_int * 4)()
                assert lib.trtx_retina_get_rect_adapt_landmark(in_w, in_h, w, h, bb.ctypes.data_as(C.POINTER(C.c_float)),
                                                               l_mine.ctypes.data_as(C.POINTER(C.c_float)), r_mine) == 0
                rects.append(list(r_mine)), lmks.append(l_mine)
    G.equal("retina_lmk.rects", np.array(rects, np.int32), np.array(ref_rects) if ref is not None else None)
    G.equal("retina_lmk.points", np.array(lmks), np.array(ref_lmks) if ref is not None else None)
