"""ctypes/numpy wrapper around oracle/liblinear_oracle.so: the CPU oracle of the bilinear letterbox pre-process of yolov3,
yolov4, scaled-yolov4, yolov3-spp and RetinaFace (preprocess_img / letterbox with OpenCV's 8-bit INTER_LINEAR and the drivers'
plane loops), and of the truncating get_rect of yolov3, yolov4, scaled-yolov4, yolov3-tiny and yolov3-spp.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "liblinear_oracle.so"
YOLOV3, RETINA, YOLOV3_SPP = 0, 1, 2  # TRTX_LINEAR_*
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_linear_input_value.restype = C.c_float
    _lib.oracle_linear_preprocess.restype = C.c_int
    _lib.oracle_linear_get_rect.restype = C.c_int
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def input_value(variant: int, c: int, u: int) -> np.float32:
    """The engine input value of byte u in plane c."""
    return np.float32(load().oracle_linear_input_value(int(variant), int(c), int(u)))


def spp_letterbox(w: int, h: int, max_size: int = 608) -> tuple[int, ...]:
    """yolov3-spp's letterbox -> (canvas_w, canvas_h, x, y, w, h)."""
    g = (C.c_int * 6)()
    load().oracle_yolov3spp_letterbox(int(w), int(h), int(max_size), g)
    return tuple(g)


def preprocess(img, variant: int, net_w: int = 608, net_h: int = 608, max_size: int = 608):
    """The pre-process of one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> ([3, net_h, net_w] float32 planes, (x, y, w,
    h) of the pasted resize), or None where the reference throws (or an SPP canvas is not net_w x net_h)."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net_h, net_w), np.float32)
    rect = (C.c_int * 4)()
    rc = load().oracle_linear_preprocess(int(variant), _vp(a), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                         int(net_w), int(net_h), int(max_size), _vp(out), rect)
    return None if rc else (out, tuple(rect))


def get_rect(variant: int, net_w: int, net_h: int, img_w: int, img_h: int, bbox) -> tuple[tuple[int, ...], bool]:
    """get_rect of variant YOLOV3 (the yolov3 family, net_w x net_h) or YOLOV3_SPP (MAX = net_w) -> ((x, y, w, h), defined);
    (0, 0, 0, 0) where the reference is undefined."""
    b = (C.c_float * 4)(*[float(v) for v in bbox])
    r = (C.c_int * 4)()
    ok = load().oracle_linear_get_rect(int(variant), int(net_w), int(net_h), int(img_w), int(img_h), b, r)
    return tuple(r), bool(ok)
