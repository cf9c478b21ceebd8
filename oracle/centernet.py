"""ctypes/numpy wrapper around oracle/libcenternet_oracle.so: the CPU oracle of the CenterNet pre-process (pre_process) and
decode (ctdet_decode and the driver's row loop), and the opener of the sample's own functions where oracle/_ref holds them.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
import subprocess
import sys
import types
from importlib.machinery import SourcelessFileLoader
from importlib.util import module_from_spec, spec_from_loader
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / "libcenternet_oracle.so"
REF_PYC = HERE / "_ref" / "ref_centernet.pyc"
NET, DOWN, K = 512, 4, 100
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = HERE / "centernet_oracle.c"
    if not LIB.exists() or LIB.stat().st_mtime < src.stat().st_mtime:  # recipe: oracle/centernet.mk
        subprocess.run(["make", "-C", str(HERE), "-f", "centernet.mk", str(LIB)], check=True, stdout=subprocess.DEVNULL)
    _lib = C.CDLL(str(LIB))
    _lib.oracle_centernet_rows.restype = C.c_int
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def preprocess(img, net: int = NET) -> np.ndarray:
    """pre_process of one u8 HWC BGR frame [h, w, 3] (rows may be pitched) -> [3, net, net] float32 planes B, G, R."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net, net), np.float32)
    load().oracle_centernet_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                       int(net), _vp(out))
    return out


def decode(heat, wh, reg, k: int = K) -> np.ndarray:
    """ctdet_decode of one image: heat [C, H, W], wh and reg [2, H, W] float32 -> dets [k, 6] float32."""
    h = np.ascontiguousarray(heat, np.float32)
    w = np.ascontiguousarray(wh, np.float32)
    r = np.ascontiguousarray(reg, np.float32)
    Cn, H, W = h.shape
    assert w.shape == (2, H, W) and r.shape == (2, H, W) and 0 < k <= H * W
    out = np.empty((k, 6), np.float32)
    load().oracle_centernet_decode(_vp(h), _vp(w), _vp(r), Cn, H, W, int(k), _vp(out))
    return out


def rows(dets, img_w: int, img_h: int, down: int = DOWN, net: int = NET, thresh=np.float32(0.5)) -> np.ndarray:
    """The driver loop over one frame's dets [K, 6] -> [1 + K*6]: the count of score > thresh, the scaled rows, zeros."""
    d = np.ascontiguousarray(dets, np.float32)
    out = np.empty(1 + d.shape[0] * 6, np.float32)
    load().oracle_centernet_rows(_vp(d), d.shape[0], int(img_w), int(img_h), int(down), int(net), C.c_float(thresh), _vp(out))
    return out


_ref = None


def reference():
    """The sample's module (pre_process, ctdet_decode) from oracle/_ref/ref_centernet.pyc, or None where it was not built.
    Its `import tensorrt` and `import common` meet stubs: the module level only builds a Logger and loads the plugins."""
    global _ref
    if _ref is not None or not REF_PYC.exists():
        return _ref
    trt = types.ModuleType("tensorrt")

    class Logger:
        WARNING = 2

        def __init__(self, *a):
            pass

    trt.Logger = Logger
    trt.init_libnvinfer_plugins = lambda *a: None
    saved = {n: sys.modules.get(n) for n in ("tensorrt", "common")}
    sys.modules["tensorrt"], sys.modules["common"] = trt, types.ModuleType("common")
    try:
        spec = spec_from_loader("ref_centernet", SourcelessFileLoader("ref_centernet", str(REF_PYC)))
        mod = module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    _ref = mod
    return _ref
