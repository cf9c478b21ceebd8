"""ctypes/numpy wrapper around oracle/libdetr_oracle.so: the CPU oracle of the DETR pre- and post-process (preprocessImg with
the driver's plane loop, and the driver's per-query loop with its cv::Rect).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base


HERE = Path(__file__).resolve().parent
LIB = HERE / "libdetr_oracle.so"
NET_W, NET_H = 1066, 800  # INPUT_W, INPUT_H
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_detr_input_value.restype = C.c_float
    _lib.oracle_detr_postprocess.restype = C.c_int
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def input_value(c: int, u: int) -> np.float32:
    """The engine input value of byte u in plane c (0 = R, 1 = G, 2 = B)."""
    return np.float32(load().oracle_detr_input_value(int(c), int(u)))


def preprocess(img, net_w: int = NET_W, net_h: int = NET_H) -> np.ndarray:
    """preprocessImg + the plane loop for one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> [3, net_h, net_w] float32
    planes R, G, B."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net_h, net_w), np.float32)
    load().oracle_detr_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                  int(net_w), int(net_h), _vp(out))
    return out


def get_rect(img_w: int, img_h: int, box):
    """The driver's cv::Rect of one box (cx, cy, w, h) -> (x, y, w, h)."""
    b = np.ascontiguousarray(box, np.float32)
    r = np.zeros(4, np.int32)
    load().oracle_detr_get_rect(int(img_w), int(img_h), _vp(b), _vp(r))
    return tuple(int(v) for v in r)


def postprocess(scores, boxes, img_w: int, img_h: int, score_thresh=np.float32(0.5)) -> np.ndarray:
    """The driver's per-query loop over one frame: scores [Q, C], boxes [Q, 4] float32 -> rows [1 + Q*6]: the kept count,
    then (x, y, w, h, score, class) per kept query, zeros past the count."""
    s = np.ascontiguousarray(scores, np.float32)
    b = np.ascontiguousarray(boxes, np.float32)
    Q, Cn = s.shape
    assert b.shape == (Q, 4)
    out = np.empty(1 + Q * 6, np.float32)
    load().oracle_detr_postprocess(_vp(s), _vp(b), int(Q), int(Cn), C.c_float(score_thresh), int(img_w), int(img_h), _vp(out))
    return out
