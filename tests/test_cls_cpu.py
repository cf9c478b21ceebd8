"""YOLO classification pre- and post-process on the CPU: the oracle (oracle/cls_oracle.c) against cv2 4.13 (IPP on and off) and
against the cls drivers' own compiled batch_preprocess, softmax and topk (oracle/_ref/libref_cls_<driver>.so, or
tests/golden/ref_cls_host.npz where they were not built), and the argument checks of trtx_cls_preprocess_enqueue and
trtx_cls_postprocess_enqueue."""
import ctypes as C

import numpy as np
import pytest

from oracle import cls as CO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

G = RefOutputs("ref_cls_host")
F = np.float32
V8, V5 = 0, 1
V8_DRIVERS = ("yolov8", "yolo11", "yolo26")
SOFTMAX_DRIVERS = ("yolov8", "yolo11", "yolov5")


def _pitched(img, extra=7):
    """The same pixels read through an odd pitch from a base one byte into the allocation."""
    h, w = img.shape[:2]
    buf = np.zeros((h, w * 3 + extra), np.uint8)
    buf[:, 1:w * 3 + 1] = img.reshape(h, w * 3)
    return np.lib.stride_tricks.as_strided(buf[:, 1:], (h, w, 3), (w * 3 + extra, 3, 1))


# ------------------------------------------------------------------ pre-process: values ------------------------
def test_convert_to_is_one_float_product():
    """convertTo(CV_32F, 1 / 255.0) -- here cv2.normalize(NORM_MINMAX, 0, 1, CV_32F) over all 256 bytes, which is that
    convertTo -- is (float)u * (float)(1 / 255.0), and not (float)(u / 255.0)."""
    cv2 = pytest.importorskip("cv2")
    u = np.arange(256, dtype=np.uint8).reshape(16, 16)
    got = cv2.normalize(u, None, 0, 1, cv2.NORM_MINMAX, cv2.CV_32F)
    assert np.array_equal(got.reshape(-1), np.arange(256, dtype=F) * F(1 / 255.0))
    assert int((np.arange(256, dtype=F) * F(1 / 255.0) != (np.arange(256) / 255.0).astype(F)).sum()) > 0


V8_SIZES = [(640, 480, 224, 224), (480, 640, 224, 224), (224, 224, 224, 224), (300, 224, 224, 224), (224, 301, 224, 224),
            (448, 600, 224, 224), (896, 448, 224, 224), (100, 80, 224, 224), (1, 1, 224, 224), (1, 7, 224, 224),
            (9, 1, 224, 224), (1920, 1080, 224, 224), (1081, 1920, 224, 224), (333, 517, 160, 96), (64, 64, 96, 160)]


def _v8_sweep(n=60, seed=31):
    rng = np.random.default_rng(seed)
    return V8_SIZES + [(int(w), int(h), 224, 224) for w, h in rng.integers(1, 1300, (n, 2))]


@pytest.mark.parametrize("ipp", [True, False])
def test_v8_oracle_equals_cv2(ipp):
    """crop + cv2.resize + cvtColor(BGR2RGB) + convertTo, planar: the oracle's planes are the convertTo values of cv2's bytes.
    Covers m == net (a plain copy in OpenCV), m == 2 net (OpenCV's 2x fast path), upscales, 1 x 1, 1 x N and odd w - m."""
    cv2 = pytest.importorskip("cv2")
    lut = np.arange(256, dtype=F) * F(1 / 255.0)
    rng = np.random.default_rng(32 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for (w, h, nw, nh) in _v8_sweep():
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            m = min(w, h)
            top, left = (h - m) // 2, (w - m) // 2
            re = cv2.resize(img[top:top + m, left:left + m], (nw, nh), interpolation=cv2.INTER_LINEAR)
            rgb = cv2.cvtColor(re, cv2.COLOR_BGR2RGB)
            got = CO.cls_preprocess(_pitched(img), V8, nw, nh)
            assert got is not None and got[1] == (left, top, m, m), (w, h)
            assert np.array_equal(got[0], lut[rgb].transpose(2, 0, 1)), (w, h, nw, nh)
    finally:
        cv2.ipp.setUseIPP(old)


def _v5_norm_table():
    """The oracle's V5 value of every byte in every plane: a 256-pixel image of grey levels 0..255 letterboxed at scale 1."""
    img = np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(1, 256, 3)
    out, rect = CO.cls_preprocess(img, V5, 256, 1)
    assert rect == (0, 0, 256, 1)
    return out[:, 0, :]


def test_v5_normalization_equals_driver_loop():
    """The V5 value of all 3 x 256 bytes equals yolov5_cls.cpp's own loop, ((float)u / 255.0 - mean) / std in double."""
    table = _v5_norm_table()
    ref = G.lib("libref_cls_yolov5.so")
    live = None
    if ref is not None:
        bgr = np.repeat(np.arange(256, dtype=np.uint8), 3)
        live = np.full((3, 256), np.nan, np.float32)
        ref.ref_cls_v5_normalize(C.c_void_p(bgr.ctypes.data), 256, C.c_void_p(live.ctypes.data))
    G.equal("v5_normalize", table, live)
    mean, std = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
    assert np.array_equal(table, ((np.arange(256.0)[None, :] / 255.0 - mean[:, None]) / std[:, None]).astype(F))


@pytest.mark.parametrize("ipp", [True, False])
def test_v5_oracle_equals_calibrator_letterbox(ipp):
    """V5 = preprocess_img's letterbox (trtx_calib_letterbox_host, pinned to cv2 in test_calibrator_cpu.py) with the mean / std
    values in place of / 255: the same bytes, the same rectangle."""
    cv2 = pytest.importorskip("cv2")
    lib = L.load()
    lut = np.arange(256, dtype=F) * F(1 / 255.0)
    table = _v5_norm_table()
    rng = np.random.default_rng(41 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        sizes = [(640, 480), (480, 640), (224, 224), (448, 448), (112, 100), (1, 1), (3, 2), (1920, 1080), (641, 479)]
        sizes += [(int(w), int(h)) for w, h in rng.integers(1, 1300, (40, 2))]
        for (w, h) in sizes:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            p = _pitched(img)
            got = CO.cls_preprocess(p, V5, 224, 224)
            cal = np.full((3, 224, 224), -1.0, np.float32)
            rc = lib.trtx_calib_letterbox_host(C.c_void_p(p.ctypes.data), w, h, p.strides[0], 224, 224,
                                               C.c_void_p(cal.ctypes.data))
            if got is None:
                assert rc == L.ERR_UNSUPPORTED, (w, h)
                continue
            assert rc == 0
            rect = (C.c_int * 4)()
            lib.trtx_calib_letterbox_rect(w, h, 224, 224, rect)
            assert got[1] == tuple(rect), (w, h)
            u = np.searchsorted(lut, cal)                                   # the letterboxed RGB bytes
            assert np.array_equal(lut[u], cal)
            assert np.array_equal(got[0], table[np.arange(3)[:, None, None], u]), (w, h)
    finally:
        cv2.ipp.setUseIPP(old)


def test_v5_empty_rectangle():
    """1 x 5000 letterboxes to width 0: cv::resize throws, the oracle refuses."""
    assert CO.cls_preprocess(np.zeros((5000, 1, 3), np.uint8), V5, 224, 224) is None


# ------------------------------------------------------------------ pre-process: crop geometry ------------------
def _geometry_cases():
    cases = []
    for w, h in ((640, 480), (480, 640), (224, 224), (1, 1), (1, 5000), (5000, 1), (3, 2), (641, 479), (1920, 1080),
                 (1080, 1920), (448, 224), (225, 224), (224, 227)):
        cases += [(w, h, 224, 224), (w, h, 160, 96)]
    rng = np.random.default_rng(51)
    cases += [(int(w), int(h), 224, 224) for w, h in rng.integers(1, 4000, (280, 2))]
    cases += [(w, 480, 224, 224) for w in range(481, 501)]             # odd and even w - m
    return cases


def test_crop_geometry_equals_drivers():
    """The crop Rect and the resize size of the V8 drivers' batch_preprocess (yolov8, yolo11, yolo26), compiled, against the
    oracle's crop: the rectangle the device pre-process reads."""
    cases = _geometry_cases()
    assert len(cases) >= 300
    mine = []
    for (w, h, nw, nh) in cases:
        m = min(w, h)
        mine.append([(w - m) // 2, (h - m) // 2, m, m, nw, nh])
        got = CO.cls_preprocess(np.zeros((h, w, 3), np.uint8), V8, nw, nh) if w * h <= 1 << 20 else None
        if got is not None:
            assert got[1] == tuple(mine[-1][:4])
    mine = np.array(mine, np.int32)
    for drv in V8_DRIVERS:
        ref = G.lib(f"libref_cls_{drv}.so")
        live = None
        if ref is not None:
            live = np.zeros((len(cases), 6), np.int32)
            for i, (w, h, nw, nh) in enumerate(cases):
                ref.ref_cls_crop_geometry(w, h, nw, nh, C.c_void_p(live[i].ctypes.data))
        G.equal(f"crop_geometry_{drv}", mine, live)


# ------------------------------------------------------------------ post-process ---------------------------------
def _tie_free_logits(rng, b, n, scale):
    while True:
        x = (rng.standard_normal((b, n)) * scale).astype(F)
        if all(len(np.unique(r)) == n for r in x):
            return x


@pytest.mark.parametrize("drv", SOFTMAX_DRIVERS)
def test_softmax_topk_equal_drivers(drv):
    """The oracle's softmax and topk equal the driver's compiled ones bit for bit on tie-free rows of 1 000 classes."""
    rng = np.random.default_rng(61)
    x = _tie_free_logits(rng, 8, 1000, 3.0)
    res = CO.softmax(x)
    assert not np.isnan(res).any()
    idx = CO.topk(res, 5)
    ref = G.lib(f"libref_cls_{drv}.so")
    live_res = live_idx = None
    if ref is not None:
        live_res = np.zeros_like(x)
        live_idx = np.zeros((8, 5), np.int32)
        for r in range(8):
            xr = np.ascontiguousarray(x[r])
            ref.ref_cls_softmax(C.c_void_p(xr.ctypes.data), 1000, C.c_void_p(live_res[r].ctypes.data))
            assert ref.ref_cls_topk(C.c_void_p(live_res[r].ctypes.data), 1000, 5, C.c_void_p(live_idx[r].ctypes.data)) == 5
    G.equal(f"softmax_{drv}", res, live_res)
    G.equal(f"topk_{drv}", idx, live_idx)


def test_topk_raw_equals_yolo26():
    """yolo26 ranks the raw (sigmoid) output: the oracle's topk equals its compiled topk on tie-free rows, k = 1, 3, 5, n."""
    rng = np.random.default_rng(62)
    while True:
        x = (1 / (1 + np.exp(-rng.standard_normal((4, 1000)) * 2.0))).astype(F)
        if all(len(np.unique(r)) == 1000 for r in x):
            break
    ref = G.lib("libref_cls_yolo26.so")
    for k in (1, 3, 5, 1000, 1200):
        mine = CO.topk(x, k)
        live = None
        if ref is not None:
            live = np.zeros_like(mine)
            for r in range(4):
                xr = np.ascontiguousarray(x[r])
                assert ref.ref_cls_topk(C.c_void_p(xr.ctypes.data), 1000, k, C.c_void_p(live[r].ctypes.data)) == min(k, 1000)
        G.equal(f"topk_yolo26_k{k}", mine, live)


def test_tie_order_recorded():
    """On rows with ties the drivers' std::sort (unstable) may order equal values any way; the library keeps ascending index.
    The test records libstdc++'s order next to the library's, and checks both give the same value sequence."""
    rng = np.random.default_rng(63)
    x = rng.integers(0, 6, (4, 1000)).astype(F) / F(8)
    x[0, ::7] = -0.0
    x[0, 3::7] = 0.0
    mine = CO.topk(x, 1000)
    for r in range(4):
        vals = x[r, mine[r]]
        assert np.all(vals[:-1] >= vals[1:])
        for v in np.unique(vals):                                       # ties in ascending index (-0.0 == +0.0)
            pos = mine[r][vals == v]
            assert np.all(np.diff(pos) > 0)
    ref = G.lib("libref_cls_yolov8.so")
    live = None
    if ref is not None:
        live = np.zeros_like(mine)
        for r in range(4):
            xr = np.ascontiguousarray(x[r])
            ref.ref_cls_topk(C.c_void_p(xr.ctypes.data), 1000, 1000, C.c_void_p(live[r].ctypes.data))
    stdsort = G.array("topk_ties_libstdcxx", live)
    for r in range(4):
        assert np.array_equal(x[r, stdsort[r]], x[r, mine[r]])         # the same values in the same order
    assert not np.array_equal(stdsort, mine)                          # but not the same indices: std::sort is unstable


def test_oracle_topk_nan_inf_order():
    x = np.array([[1.0, np.nan, -np.inf, np.inf, -np.nan, -0.0, 0.0, 2.0]], F)
    x[0, 4] = -np.abs(np.float32(np.nan))                              # a NaN with the sign bit set
    assert np.signbit(x[0, 4]) and not np.signbit(x[0, 1])
    assert CO.topk(x, 8).tolist() == [[1, 3, 7, 0, 5, 6, 2, 4]]


# ------------------------------------------------------------------ argument validation ------------------------
def test_cls_preprocess_argument_validation():
    """Every descriptor is checked before anything is launched (the pointers here are never dereferenced)."""
    lib = L.load()

    def descs(*sizes, ptr=4096, pitch=None):
        d = (L.ImageDesc * len(sizes))()
        for i, (w, h) in enumerate(sizes):
            d[i].data_dev, d[i].width, d[i].height = ptr, w, h
            d[i].pitch = 3 * w if pitch is None else pitch
        return d

    inv, uns = L.ERR_INVALID, L.ERR_UNSUPPORTED
    ok = descs((640, 480), (480, 640))
    f = lib.trtx_cls_preprocess_enqueue
    for v in (V8, V5):
        assert f(v, None, 2, 224, 224, 4096, None) == inv
        assert f(v, ok, 0, 224, 224, 4096, None) == inv
        assert f(v, ok, -1, 224, 224, 4096, None) == inv
        assert f(v, ok, 2, 0, 224, 4096, None) == inv
        assert f(v, ok, 2, 224, -1, 4096, None) == inv
        assert f(v, ok, 2, 224, 224, None, None) == inv
        assert f(v, ok, 2, 224, 224, 4098, None) == inv                  # not a float address
        assert f(v, descs((640, 480), (640, 480), ptr=None), 2, 224, 224, 4096, None) == inv
        assert f(v, descs((640, 480), (0, 480)), 2, 224, 224, 4096, None) == inv
        assert f(v, descs((640, 480), pitch=1919), 1, 224, 224, 4096, None) == inv
        assert f(v, descs(*([(640, 480)] * 70 + [(640, -1)])), 71, 224, 224, 4096, None) == inv
    for v in (2, 3, -1, 7):
        assert f(v, ok, 2, 224, 224, 4096, None) == inv
    # V5: an empty letterbox rectangle (cv::resize throws), also behind valid images; rows wider than the shared-memory stage
    assert f(V5, descs((1, 5000)), 1, 224, 224, 4096, None) == uns
    assert f(V5, descs((640, 480), (5000, 1)), 2, 224, 224, 4096, None) == uns
    assert f(V5, descs((6000, 100)), 1, 6000, 100, 4096, None) == uns
    assert f(V8, descs((6000, 100)), 1, 6000, 100, 4096, None) == uns


def test_cls_postprocess_argument_validation():
    lib = L.load()
    f = lib.trtx_cls_postprocess_enqueue
    inv, uns = L.ERR_INVALID, L.ERR_UNSUPPORTED
    assert f(1, 2, 1000, None, 3, 4096, 4096, None, None) == inv
    assert f(1, 2, 1000, 4096, 3, None, 4096, None, None) == inv
    assert f(1, 2, 1000, 4096, 3, 4096, None, 4096, None) == inv
    assert f(1, 0, 1000, 4096, 3, 4096, 4096, None, None) == inv
    assert f(1, 2, 0, 4096, 3, 4096, 4096, None, None) == inv
    assert f(1, 2, 1000, 4096, 0, 4096, 4096, None, None) == inv
    assert f(2, 2, 1000, 4096, 3, 4096, 4096, None, None) == inv
    assert f(-1, 2, 1000, 4096, 3, 4096, 4096, None, None) == inv
    assert f(1, 2, 8193, 4096, 3, 4096, 4096, None, None) == uns
    assert f(0, 2, 100000, 4096, 3, 4096, 4096, None, None) == uns
