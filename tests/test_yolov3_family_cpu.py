"""The yolov3 family's decode and NMS on the CPU, and its YoloLayer_TRT creators (tests/trt_adapter_v3_family_check.cpp).

* The oracle's box modes (oracle/v3family.py, box_mode 4 / 5 / 6 = the library's TRTX_YOLO_V3_NET / V4 / V4_CSP) equal a
  numpy re-derivation of the reference expressions, with libm's expf as the oracle's exp: x, y, w, h of modes 4 and 5 and x,
  y of mode 6 bit for bit; mode 6's w, h (powf(2s, 2)) within 1 ulp of numpy's float32 (2s)*(2s), since the host powf
  need not round as a product does.
* Each driver's own compiled nms() (oracle/_ref/libref_v3f_nms_<driver>.so; where it was not built, the digests in
  tests/golden/ref_v3f_host.npz) keeps the same rows in the same order as the library's NMS semantics with the parameters of
  plugins.V3_FAMILY_DRIVERS, on rows whose det_confidence sits on each threshold.
* The creators' blobs equal the Python mirror's and those the drivers' own yololayer.h constants make."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import v3family as V
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

ROOT = Path(__file__).resolve().parents[1]
G = RefOutputs("ref_v3f_host")
DRIVERS = ("yolov3", "yolov4", "scaled-yolov4", "yolov3-tiny")
LIBNAME = {"yolov3": "yolov3", "yolov4": "yolov4", "scaled-yolov4": "csp", "yolov3-tiny": "tiny"}

_libm = C.CDLL("libm.so.6")
_libm.expf.restype = C.c_float
_libm.expf.argtypes = [C.c_float]


def _expf(x):
    return np.float32(_libm.expf(C.c_float(float(x))))


def _sig(x, f64):
    e = _expf(-np.float32(x))
    if f64:
        return np.float32(np.float64(1.0) / (np.float64(1.0) + np.float64(e)))
    return np.float32(np.float32(1.0) / (np.float32(1.0) + e))


def _heads(d, B, seed):
    rng = np.random.default_rng(seed)
    out = []
    for w, h, _ in d["kernels"]:
        x = rng.normal(-4.0, 3.0, size=(B, 3, 85, h, w)).astype(np.float32)
        x[:, :, 4] = rng.normal(-7.0, 2.0, size=(B, 3, h, w))   # objectness: ~1 % of the anchors pass
        out.append(x.reshape(B, 3 * 85, h, w))
    return out


def _ulps(a, b):
    ai = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    bi = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(ai - bi)


@pytest.mark.parametrize("driver", DRIVERS)
def test_oracle_box_modes_equal_numpy_restatement(oracle, driver):
    d = P.V3_FAMILY_DRIVERS[driver]
    mode, (nw, nh) = d["variant"], d["net"]
    B = 1
    heads = _heads(d, B, seed=700 + mode)
    anchors = [a for _, _, a in d["kernels"]]
    out, idx = V.decode(heads, anchors, box_mode=mode, net=(nw, nh))
    n = int(out[0, 0])
    assert 20 < n <= 1000
    rows = out[0, 1:1 + n * 7].reshape(n, 7)
    offs = np.cumsum([0] + [w * h * 3 for w, h, _ in d["kernels"]])
    f64 = mode in (L.YOLO_V4, L.YOLO_V4_CSP)
    wh_ulps = []
    for r, a in zip(rows, idx[0, :n]):
        l = int(np.searchsorted(offs, a, side="right") - 1)
        gw, gh, anc = d["kernels"][l]
        cell, k = divmod(int(a - offs[l]), 3)
        row, col = divmod(cell, gw)
        v = heads[l][0].reshape(3, 85, gh * gw)[k, :, cell]
        sx, sy = _sig(v[0], f64), _sig(v[1], f64)
        if mode == L.YOLO_V4_CSP:
            x = np.float32((np.float64(np.float32(col) + np.float32(2) * sx) - 0.5) * nw / gw)
            y = np.float32((np.float64(np.float32(row) + np.float32(2) * sy) - 0.5) * nh / gh)
            tw, th = np.float32(2) * _sig(v[2], f64), np.float32(2) * _sig(v[3], f64)
            w, h = np.float32(tw * tw) * np.float32(anc[2 * k]), np.float32(th * th) * np.float32(anc[2 * k + 1])
            wh_ulps.append(_ulps([r[2], r[3]], [w, h]).max())
        else:
            x = np.float32(np.float32(np.float32(col) + sx) * np.float32(nw)) / np.float32(gw)
            y = np.float32(np.float32(np.float32(row) + sy) * np.float32(nh)) / np.float32(gh)
            w, h = _expf(v[2]) * np.float32(anc[2 * k]), _expf(v[3]) * np.float32(anc[2 * k + 1])
            assert r[2] == w and r[3] == h
        assert r[0] == x and r[1] == y, (r[:2], x, y)
        # the gates and both confidences with this driver's Logist
        bp = _sig(v[4], f64)
        assert r[4] == bp and bp >= np.float32(0.1) and r[6] >= np.float32(0.1)
        assert r[6] == max(_sig(c, f64) for c in v[5:])
    if wh_ulps:
        assert max(wh_ulps) <= 1


def test_oracle_spp_mode_is_the_spp_oracle(oracle):
    from tensorrtx_b200 import synth
    heads = synth.yolov3_heads(1, seed=705, net_w=416, net_h=416)
    anchors = [k.anchors for k in P.YOLOV3_KERNELS]
    a, ia = oracle.yolov3_decode(heads, anchors)            # trtx_oracle.c's yolov3-spp decode
    b, ib = V.decode(heads, anchors, box_mode=L.YOLO_V3, strides=(32, 16, 8))
    assert np.array_equal(a, b) and np.array_equal(ia, ib)
    c, _ = V.decode(heads, anchors, box_mode=L.YOLO_V3_NET, net=(416, 416))
    n = int(a[0, 0])
    assert c[0, 0] == n
    ra, rc = a[0, 1:1 + 7 * n].reshape(n, 7), c[0, 1:1 + 7 * n].reshape(n, 7)
    assert np.array_equal(ra[:, 2:], rc[:, 2:])
    # `* INPUT_W / yoloWidth` is not `* stride` in float: some boxes differ
    assert (ra[:, :2] != rc[:, :2]).any(axis=1).mean() > 0.01


def _nms_rows(driver, seed):
    """A plugin buffer of 7-float rows: clusters of overlapping boxes over 4 classes, distinct confidences, and rows whose
    det_confidence is the threshold, the float below and the float above it."""
    d = P.V3_FAMILY_DRIVERS[driver]
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(40):
        cx, cy = rng.uniform(50, 550, 2)
        w, h = rng.uniform(20, 200, 2)
        cls = float(rng.integers(0, 4))
        for _ in range(int(rng.integers(1, 6))):
            rows.append([cx + rng.normal(0, 8), cy + rng.normal(0, 8), w * rng.uniform(0.8, 1.2), h * rng.uniform(0.8, 1.2),
                         rng.uniform(0.1, 1.0), cls, rng.uniform(0.1, 1.0)])
    thr = np.float32(0.4 if driver == "yolov3-tiny" else 0.5)
    for i, c in enumerate((thr, np.nextafter(thr, np.float32(0)), np.nextafter(thr, np.float32(1)))):
        rows.append([1000.0 + 300 * i, 1000.0, 50.0, 50.0, float(c), 1.0, 0.5])
    rows = np.asarray(rows, np.float32)
    rows = rows[rng.permutation(len(rows))]
    buf = np.zeros(1 + 1000 * 7, np.float32)
    buf[0] = len(rows)
    buf[1:1 + rows.size] = rows.reshape(-1)
    return buf


@pytest.mark.parametrize("driver", DRIVERS)
def test_library_nms_parameters_equal_driver_nms(oracle, driver):
    d = P.V3_FAMILY_DRIVERS[driver]
    lib = G.lib(f"libref_v3f_nms_{LIBNAME[driver]}.so")
    for seed in (710, 711):
        buf = _nms_rows(driver, seed)
        res, _ = oracle.nms(1, buf, 1000, 7, d["conf_thresh"], d["nms_thresh"])
        ref = None
        if lib is not None:
            out = np.zeros((1000, 7), np.float32)
            n = lib.ref_v3_nms(buf.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), 1000)
            ref = out[:n]
        G.equal(f"nms.{driver}.{seed}", res, ref)
        confs = res[:, 4]
        thr = np.float32(0.4 if driver == "yolov3-tiny" else 0.5)
        assert thr in confs if driver == "yolov3-tiny" else thr not in confs   # `<=` a double literal
        assert np.nextafter(thr, np.float32(1)) in confs and np.nextafter(thr, np.float32(0)) not in confs


def test_tiny_conf_thresh_is_the_float_below_0_4():
    t = np.float32(P.V3_FAMILY_DRIVERS["yolov3-tiny"]["conf_thresh"])
    assert t == np.nextafter(np.float32(0.4), np.float32(0))
    assert float(np.float32(0.4)) > 0.4 and float(t) <= 0.4   # 0.4f survives `(double)c <= 0.4`, the float below does not
    for d in ("yolov3", "yolov4", "scaled-yolov4"):
        assert P.V3_FAMILY_DRIVERS[d]["conf_thresh"] == 0.5 and P.V3_FAMILY_DRIVERS[d]["nms_thresh"] == 0.4


# ------------------------------------------------------------------ TensorRT creators ----------------------------------
def _build_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda = Path(nvcc).resolve().parents[1]
    exe = tmp_path / "trt_adapter_v3_family_check"
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-I", str(ROOT / "include"), "-I", str(ROOT / "tests" / "mock_trt"),
           "-I", str(cuda / "include"), str(ROOT / "tests" / "trt_adapter_v3_family_check.cpp"), "-o", str(exe),
           str(L.LIB_PATH), f"-Wl,-rpath,{L.LIB_PATH.parent}", "-L", str(cuda / "lib64"), "-lcudart", f"-Wl,-rpath,{cuda / 'lib64'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_family_creators_host_surface_and_blobs(tmp_path):
    exe = _build_check(tmp_path)
    r = subprocess.run([str(exe), "--dump"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "v3 family adapter check ok" in r.stdout
    blobs = {ln.split()[1]: bytes.fromhex(ln.split()[2]) for ln in r.stdout.splitlines() if ln.startswith("blob ")}
    assert set(blobs) == set(DRIVERS) | {"yolov3-spp"}
    for driver in DRIVERS:
        plug = P.YoloLayerPluginV3Net.for_driver(driver)
        assert blobs[driver] == plug.serialize() and len(plug.serialize()) == plug.getSerializationSize()
        d = P.V3_FAMILY_DRIVERS[driver]
        q = P.YoloLayerPluginV3Net.deserialize(blobs[driver], d["net"][0], d["net"][1], d["variant"])
        assert q.serialize() == blobs[driver] and q.params.variant == d["variant"]
        lib = G.lib(f"libref_v3f_{LIBNAME[driver]}_host.so")
        ref = None
        if lib is not None:
            buf = (C.c_ubyte * 256)()
            n = lib.ref_v3f_header_blob(buf, 256)
            ref = np.frombuffer(bytes(buf[:n]), np.uint8)
            v = (C.c_int * 4)()
            lib.ref_v3f_header_net(v)
            assert tuple(v) == (d["net"][0], d["net"][1], d["max_out"], 7)
        G.equal(f"blob.{driver}", np.frombuffer(blobs[driver], np.uint8), ref)
    assert blobs["yolov3-spp"] == P.YoloLayerPluginV3().serialize()
    with pytest.raises(L.TrtxError):
        P.YoloLayerPluginV3Net.deserialize(blobs["yolov3-spp"], 608, 608, L.YOLO_V3_NET)
