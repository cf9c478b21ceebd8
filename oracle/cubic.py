"""ctypes/numpy wrapper around oracle/libcubic_oracle.so: the CPU oracle of the bicubic letterbox pre-process of yolov3-tiny and
retinafaceAntiCov (preprocess_img with OpenCV's own 8-bit INTER_CUBIC, IPP off, and the drivers' plane loops).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "libcubic_oracle.so"
YOLOV3_TINY, ANTICOV = 0, 1  # TRTX_CUBIC_YOLOV3_TINY, TRTX_CUBIC_ANTICOV
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_cubic_input_value.restype = C.c_float
    _lib.oracle_cubic_preprocess.restype = C.c_int
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def _check(a):
    a = np.asarray(a)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    return a


def resize(img, dw: int, dh: int) -> np.ndarray:
    """cv::resize(img, Size(dw, dh), INTER_CUBIC) of a u8 HWC BGR image [h, w, 3] (rows may be pitched), IPP off -> [dh, dw, 3]."""
    a = _check(img)
    out = np.empty((dh, dw, 3), np.uint8)
    load().oracle_resize_cubic_u8(_vp(a), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]), int(dw), int(dh), _vp(out))
    return out


def input_value(variant: int, u: int) -> np.float32:
    """The engine input value of byte u."""
    return np.float32(load().oracle_cubic_input_value(int(variant), int(u)))


def preprocess(img, variant: int, net_w: int = 608, net_h: int = 608):
    """preprocess_img + the plane loop for one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> ([3, net_h, net_w] float32
    planes R, G, B, (x, y, w, h) of the pasted resize), or None where the reference throws."""
    a = _check(img)
    out = np.empty((3, net_h, net_w), np.float32)
    rect = (C.c_int * 4)()
    rc = load().oracle_cubic_preprocess(int(variant), _vp(a), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                        int(net_w), int(net_h), _vp(out), rect)
    return None if rc else (out, tuple(rect))
