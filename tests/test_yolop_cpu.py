"""YOLOP on the CPU: the YoloLayer_TRT creator with YOLOP's and yolov7's fields (tests/trt_adapter_yolop_check.cpp under
AddressSanitizer), the oracle (oracle/yolop_oracle.c) against cv2 4.13 and against YOLOP's own compiled nms() and get_rect
(oracle/_ref/libref_yolop_host.so, or tests/golden/ref_yolop_host.npz where it was not built), the library's host
trtx_yolop_get_rect, and the argument checks of the YOLOP calls that reject before any launch."""
import ctypes as C
import shutil
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import oracle as O
from oracle import yolop as YO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

ROOT = Path(__file__).resolve().parents[1]
G = RefOutputs("ref_yolop_host")
F = np.float32
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
YOLOP_ANCHORS = ((3, 9, 5, 11, 4, 20), (7, 18, 6, 39, 12, 31), (19, 50, 38, 81, 68, 157))  # strides 8, 16, 32


# ------------------------------------------------------------------ TensorRT adapter ----------------------------------
def _adapter_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda = Path(nvcc).resolve().parents[1]
    exe = tmp_path / "trt_adapter_yolop_check"
    cmd = ["g++", "-std=c++14", "-O1", "-g", "-Wall", "-fsanitize=address", "-fno-omit-frame-pointer", "-I", str(ROOT / "include"),
           "-I", str(ROOT / "tests" / "mock_trt"), "-I", str(cuda / "include"), str(ROOT / "tests" / "trt_adapter_yolop_check.cpp"),
           "-o", str(exe), str(L.LIB_PATH), f"-Wl,-rpath,{L.LIB_PATH.parent}", "-L", str(cuda / "lib64"), "-lcudart",
           f"-Wl,-rpath,{cuda / 'lib64'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "--dump"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "trt adapter yolop check ok" in r.stdout, r.stdout + r.stderr
    return {ln.split()[1]: bytes.fromhex(ln.split()[2]) for ln in r.stdout.splitlines() if ln.startswith("blob ")}


def test_adapter_yolop_and_yolov7_fields_make_the_v7_plugin(tmp_path):
    """YOLOP's field collection (netdata declared 3 holding 4 ints, yolodata1..3 of ints, stride-32 kernel first) and yolov7's
    netinfo of 4 create the 6-float-row plugin: its blob equals YoloLayerPluginV7(...).serialize() and the reference's write()
    order (yolop/yololayer.cu:81-96: classCount, threadCount, kernelCount, netW, netH, maxOut, kernels).  yolov5's netinfo of 5
    and yolov8's combinedInfo give the blobs they gave before.  The check binary also round-trips every blob through both
    plugin forms, refuses malformed fields and blob lengths, and runs under AddressSanitizer."""
    from tensorrtx_b200 import plugins as P

    blobs = _adapter_check(tmp_path)
    grids = ((20, 12), (40, 24), (80, 48))  # the plugin's input order: stride 32, 16, 8
    kern = [P.YoloKernel(w, h, YOLOP_ANCHORS[2 - i]) for i, (w, h) in enumerate(grids)]
    assert blobs["yolop"] == P.YoloLayerPluginV7(1, 640, 384, 1000, kern).serialize()
    ref = struct.pack("<6i", 1, 256, 3, 640, 384, 1000) + b"".join(
        struct.pack("<2i6f", w, h, *YOLOP_ANCHORS[2 - i]) for i, (w, h) in enumerate(grids))
    assert blobs["yolop"] == ref
    v7k = [P.YoloKernel(80, 80, [12, 16, 19, 36, 40, 28]), P.YoloKernel(40, 40, [36, 75, 76, 55, 72, 146]),
           P.YoloKernel(20, 20, [142, 110, 192, 243, 459, 401])]
    assert blobs["yolov7"] == P.YoloLayerPluginV7(80, 640, 640, 1000, v7k).serialize()
    assert blobs["yolov5"] == P.YoloLayerPluginV5(80, 640, 640, 1000, False, v7k).serialize()
    assert blobs["yolov8"] == P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)).serialize()
    assert {len(b) % 4 for b in blobs.values()} == {0, 1, 3}


# ------------------------------------------------------------------ pre-process: values -------------------------------
def _all_bytes_image():
    return np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(16, 16, 3)


def _cv2_chain(img):
    """preprocess_img after the resize, in cv2: convertTo(CV_32FC3, 1.f / 255.f) -- cv2.normalize(NORM_MINMAX, 0, 1) of an image
    holding 0 and 255 is that convertTo -- then cv2.subtract and cv2.divide by the Scalars."""
    cv2 = pytest.importorskip("cv2")
    assert img.min() == 0 and img.max() == 255
    t = cv2.normalize(img, None, 0, 1, cv2.NORM_MINMAX, cv2.CV_32F)
    t = cv2.subtract(t, MEAN + (0.0,))
    return cv2.divide(t, STD + (1.0,), scale=1)


def test_values_equal_cv2_chain_on_all_768_bytes():
    """For every byte in every channel, cv2 4.13's convertTo / subtract / divide chain equals the oracle's
    s = (float)u * (1.f / 255.f) - (float)mean in float, then (float)((double)s / std); a float division differs."""
    assert F(1.0) / F(255.0) == F(1 / 255.0)
    got = _cv2_chain(_all_bytes_image()).reshape(256, 3)
    u = np.arange(256)
    for c in range(3):
        assert np.array_equal(got[:, c], np.array([YO.input_value(c, v) for v in u], np.float32)), c
    fdiv = np.array([(F(v) * F(1 / 255.0) - F(MEAN[0])) / F(STD[0]) for v in u], np.float32)
    assert (fdiv != got[:, 0]).any()


# ------------------------------------------------------------------ pre-process: the oracle -----------------------------
PRE_SIZES = [(1920, 1080), (1280, 720), (640, 384), (640, 360), (320, 180), (1000, 1000), (384, 640), (1, 1), (1, 300),
             (300, 1), (5000, 3), (2, 700), (1111, 333), (97, 1301), (4096, 2160), (643, 386)]


def _letterbox_rect(w, h, net_w=640, net_h=384):
    r = np.zeros(4, np.int32)
    L.load().trtx_calib_letterbox_rect(w, h, net_w, net_h, r.ctypes.data_as(C.POINTER(C.c_int)))
    return tuple(int(v) for v in r)


@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_cv2(ipp):
    """preprocess_img restated with cv2 (resize INTER_LINEAR of the 8-bit image into trtx_calib_letterbox_rect's rectangle on a
    114 canvas, then the chain above) and split into B, G, R planes equals the oracle bit for bit, up- and down-scaling,
    1 x N and N x 1; a pitched image reads the same."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for w, h in PRE_SIZES:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            got = YO.preprocess(img)
            x, y, rw, rh = _letterbox_rect(w, h)
            if rw <= 0 or rh <= 0:
                assert got is None, (w, h)
                continue
            canvas = np.full((384, 640, 3), 114, np.uint8)
            canvas[y:y + rh, x:x + rw] = cv2.resize(img, (rw, rh), interpolation=cv2.INTER_LINEAR)
            canvas[0, 0] = (0, 0, 0)  # 0 and 255 present, so that normalize is convertTo (the two pixels are excluded below)
            canvas[0, 1] = (255, 255, 255)
            want = _cv2_chain(canvas).transpose(2, 0, 1)
            assert got is not None and got[1] == (x, y, rw, rh), (w, h)
            keep = np.ones((384, 640), bool)
            keep[0, :2] = False
            assert np.array_equal(got[0][:, keep], want[:, keep]), (w, h, ipp)
            buf = np.zeros((h, 3 * w + 5), np.uint8)
            buf[:, :3 * w] = img.reshape(h, 3 * w)
            pitched = np.lib.stride_tricks.as_strided(buf, (h, w, 3), (3 * w + 5, 3, 1))
            assert np.array_equal(YO.preprocess(pitched)[0], got[0])
    finally:
        cv2.ipp.setUseIPP(old)


# ------------------------------------------------------------------ labels: the nearest index tables --------------------
def test_nearest_tables_equal_cv2_inter_nearest():
    """The oracle's labels are cv2.resize(INTER_NEAREST) of both int32 maps to the frame, then lane ? 2 : seg ? 1 : 0, on
    every pixel of 34 frame sizes (down- and up-scaling, 1 x N, N x 1, exact multiples)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    sizes = [(1920, 1080), (1280, 720), (640, 360), (320, 180), (1, 1), (1, 500), (500, 1), (1279, 719), (641, 361), (960, 540),
             (3840, 2160), (2, 2), (1919, 1081), (1000, 1000), (160, 90), (1280, 1080), (1366, 768), (427, 240)]
    sizes += [tuple(int(v) for v in s) for s in rng.integers(1, 2000, (16, 2))]
    seg = rng.integers(0, 2, (360, 640), dtype=np.int32)
    lane = (rng.random((360, 640)) < 0.2).astype(np.int32)
    for w, h in sizes:
        rs = cv2.resize(seg, (w, h), interpolation=cv2.INTER_NEAREST)
        rl = cv2.resize(lane, (w, h), interpolation=cv2.INTER_NEAREST)
        want = np.where(rl != 0, 2, np.where(rs != 0, 1, 0)).astype(np.uint8)
        assert np.array_equal(YO.labels(seg, lane, w, h), want), (w, h)
        idx = np.arange(640 * 360, dtype=np.int32).reshape(360, 640)
        r = cv2.resize(idx, (w, h), interpolation=cv2.INTER_NEAREST)
        assert np.array_equal(r // 640, np.broadcast_to(YO.nearest(h, 360)[:, None], (h, w))), (w, h)
        assert np.array_equal(r % 640, np.broadcast_to(YO.nearest(w, 640)[None, :], (h, w))), (w, h)


# ------------------------------------------------------------------ get_rect ----------------------------------------------
RECT_SIZES = [(1920, 1080), (1280, 720), (640, 384), (640, 360), (384, 640), (1, 1), (3000, 17), (17, 3000)]


def _boxes(n=2500, seed=7):
    rng = np.random.default_rng(seed)
    b = np.concatenate([rng.uniform(-50, 700, (n, 2)), rng.uniform(0, 400, (n, 2))], 1).astype(np.float32)
    special = np.array([[np.nan, 10, 5, 5], [10, np.inf, 5, 5], [-np.inf, 10, 5, 5], [10, 10, np.nan, 5], [3e9, 10, 5, 5],
                        [10, -3e9, 5, 5], [10, 10, 5e9, 5], [1e30, 1e30, 1e30, 1e30], [0, 0, 0, 0], [320, 192, 640, 384],
                        [-2.5, -0.5, 1, 1], [639.9, 383.9, 0.2, 0.2]], np.float32)
    return np.concatenate([b, special])


def test_get_rect_equals_compiled_reference():
    """trtx_yolop_get_rect and the oracle equal YOLOP's compiled get_rect (yolop/common.hpp:13-37, 640 x 384) on 2 512 boxes x
    8 frame sizes, NaN, infinite and out-of-int-range boxes included: INT_MIN where x86-64 converts such a value, wrapping
    widths."""
    lib = L.load()
    ref = G.lib("libref_yolop_host.so")
    boxes = _boxes()
    for w, h in RECT_SIZES:
        got = np.zeros((len(boxes), 4), np.int32)
        orc = np.zeros_like(got)
        r = (C.c_int * 4)()
        for i, b in enumerate(boxes):
            bb = (C.c_float * 4)(*b.tolist())
            assert lib.trtx_yolop_get_rect(640, 384, w, h, bb, r) == 0
            got[i] = list(r)
            orc[i] = YO.get_rect(w, h, b)
        assert np.array_equal(got, orc), (w, h)
        live = None
        if ref is not None:
            live = np.zeros_like(got)
            for i, b in enumerate(boxes):
                bb = np.ascontiguousarray(b, np.float32)
                ref.ref_yolop_get_rect(w, h, C.c_void_p(bb.ctypes.data), C.c_void_p(live[i].ctypes.data))
        G.equal(f"get_rect_{w}x{h}", got, live)
    assert (got == np.iinfo(np.int32).min).any()


# ------------------------------------------------------------------ NMS ------------------------------------------------
def test_oracle_nms_equals_compiled_reference():
    """oracle.nms(1, ...) over 6-float rows equals YOLOP's compiled nms() (conf 0.25, IoU 0.45) on tie-free rows: counts of
    0, 1, 300 and 1000 (its MAX_OUTPUT_BBOX_COUNT), one and three classes."""
    ref = G.lib("libref_yolop_host.so")
    if ref is not None:
        assert ref.ref_yolop_det_floats() == 6
    rng = np.random.default_rng(21)
    for n, nc in ((0, 1), (1, 1), (300, 1), (1000, 1), (1000, 3)):
        buf = np.zeros(1 + 1000 * 6, np.float32)
        rows = buf[1:].reshape(1000, 6)
        rows[:n, :2] = rng.uniform(0, 640, (n, 2))
        rows[:n, 2:4] = rng.uniform(4, 120, (n, 2))
        rows[:n, 4] = rng.permutation(n) / max(n, 1) * 0.99 + 0.005  # distinct confidences
        rows[:n, 5] = rng.integers(0, nc, n)
        buf[0] = n
        res, _ = O.nms(1, buf, 1000, 6, F(0.25), F(0.45))
        live = None
        if ref is not None:
            out = np.zeros(1000 * 6, np.float32)
            k = ref.ref_yolop_nms(C.c_void_p(buf.ctypes.data), C.c_float(0.25), C.c_float(0.45), C.c_void_p(out.ctypes.data))
            live = out[:k * 6].reshape(k, 6)
        G.equal(f"nms_{n}_{nc}", res[:, :6], live)


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_abi_and_rejected_arguments():
    lib = L.load()
    assert lib.trtx_abi_sizeof(10) == C.sizeof(L.YolopPostParams) == 20
    descs = (L.ImageDesc * 1)()
    descs[0].data_dev, descs[0].width, descs[0].height, descs[0].pitch = 16, 4, 4, 12
    assert lib.trtx_yolop_preprocess_enqueue(None, 1, 640, 384, 16, None) == L.ERR_INVALID
    assert lib.trtx_yolop_preprocess_enqueue(descs, 0, 640, 384, 16, None) == L.ERR_INVALID
    assert lib.trtx_yolop_preprocess_enqueue(descs, 1, 640, 384, None, None) == L.ERR_INVALID
    assert lib.trtx_yolop_preprocess_enqueue(descs, 1, 640, 384, 18, None) == L.ERR_INVALID  # dst not 4-byte aligned
    descs[0].pitch = 11
    assert lib.trtx_yolop_preprocess_enqueue(descs, 1, 640, 384, 16, None) == L.ERR_INVALID
    descs[0].width, descs[0].height, descs[0].pitch = 5000, 1, 15000
    assert lib.trtx_yolop_preprocess_enqueue(descs, 1, 640, 384, 16, None) == L.ERR_UNSUPPORTED  # empty rectangle
    q = L.YolopPostParams(640, 384, 640, 360, 7)
    fr = (L.Frame * 2)()
    fr[0].img_w, fr[0].img_h, fr[1].img_w, fr[1].img_h = 1920, 1080, 1280, 720
    call = lambda p=C.byref(q), f=fr, b=2, d=16, m=10, s=16, l_=16, r=16: lib.trtx_yolop_postprocess_enqueue(p, f, b, d, m, s, l_, r, None)
    assert call(p=None) == L.ERR_INVALID
    assert call(b=0) == L.ERR_INVALID
    assert call(d=None) == L.ERR_INVALID
    assert call(m=0) == L.ERR_INVALID
    assert call(r=None) == L.ERR_INVALID
    q.row_floats = 6
    assert call() == L.ERR_INVALID
    q.row_floats = 7
    fr[0].masks_dev, fr[0].pitch = 64, 1920  # canvases for one frame of two
    assert call() == L.ERR_INVALID
    fr[1].masks_dev, fr[1].pitch = 64, 1279  # pitch < img_w
    assert call() == L.ERR_INVALID
    fr[1].pitch = 1280
    assert call(s=None) == L.ERR_INVALID
    fr[0].img_w, fr[0].pitch = 200000, 200000  # the sx table does not fit in shared memory
    assert call() == L.ERR_UNSUPPORTED
