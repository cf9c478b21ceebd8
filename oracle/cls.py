"""ctypes/numpy wrapper around oracle/libcls_oracle.so: the CPU oracle of the YOLO classification pre- and post-process
(batch_preprocess, softmax and topk of the cls drivers).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "libcls_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_cls_preprocess.restype = C.c_int
    _lib.oracle_cls_topk.restype = C.c_int
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def cls_preprocess(img, variant, net_w, net_h):
    """batch_preprocess of the cls drivers for one u8 HWC BGR image [h, w, 3] (rows may be pitched): variant 0 (V8: yolov8,
    yolo11, yolo26) or 1 (V5) -> ([3, net_h, net_w] float32 planar RGB, (x, y, w, h) of the crop (V8) or of the pasted image
    (V5)), or None where the reference throws."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net_h, net_w), np.float32)
    rect = np.zeros(4, np.int32)
    rc = load().oracle_cls_preprocess(int(variant), C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]),
                                      C.c_size_t(a.strides[0]), int(net_w), int(net_h), _vp(out), _vp(rect))
    return None if rc else (out, tuple(int(v) for v in rect))


def softmax(logits):
    """softmax of the drivers, row by row: expf, a float sum in ascending index, divisions."""
    x = np.ascontiguousarray(logits, np.float32)
    out = np.empty_like(x)
    for r in range(x.shape[0]):
        load().oracle_cls_softmax(_vp(x[r]), int(x.shape[1]), _vp(out[r]))
    return out


def topk(res, k):
    """The first min(k, n) indices of each row in descending value, ties in ascending index, -0.0 == +0.0, +NaN above +inf and
    -NaN below -inf -> int32 [B, min(k, n)]."""
    r = np.ascontiguousarray(res, np.float32)
    kk = min(k, r.shape[1])
    out = np.empty((r.shape[0], kk), np.int32)
    for i in range(r.shape[0]):
        load().oracle_cls_topk(_vp(r[i]), int(r.shape[1]), int(k), _vp(out[i]))
    return out
