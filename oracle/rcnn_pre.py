"""ctypes/numpy wrapper around oracle/librcnn_pre_oracle.so: the CPU oracle of the Mask R-CNN pre-process (preprocessImg,
rcnn/common.hpp:79-110, + the float widening of rcnn/rcnn.cpp:504-505).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "librcnn_pre_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_rcnn_preprocess.restype = C.c_int
    return _lib


def rcnn_preprocess(img, net_w, net_h):
    """preprocessImg (rcnn/common.hpp:79-110) + `data[i] = (float)img.data[i]` (rcnn.cpp:504-505) for one u8 HWC BGR image
    [h, w, 3] (rows may be pitched) -> ([net_h, net_w, 3] float32, (x, y, w, h) of the pasted image), or None where the
    reference throws (an empty resize)."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((net_h, net_w, 3), np.float32)
    rect = np.zeros(4, np.int32)
    rc = load().oracle_rcnn_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                       int(net_w), int(net_h), out.ctypes.data_as(C.c_void_p), rect.ctypes.data_as(C.c_void_p))
    return None if rc else (out, tuple(int(v) for v in rect))
