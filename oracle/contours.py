"""ctypes/numpy wrapper around oracle/libcontours_oracle.so: the CPU oracle of
cv::findContours(img, RETR_EXTERNAL, CHAIN_APPROX_NONE), the outlines the Mask R-CNN driver takes of each pasted canvas
(rcnn/rcnn.cpp:551-552).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "libcontours_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is None:
        _lib = _base.build_and_open(LIB)
    return _lib


def find_contours_external(img, max_contours=None, max_points=None):
    """cv2.findContours(img, RETR_EXTERNAL, CHAIN_APPROX_NONE) of a 2-D u8 array (nonzero = foreground), restated in C.
    Returns (n_contours, n_points, lengths [min(n, max_contours)] int32, points [min(total, max_points), 2] int32 (x, y)),
    contours in cv2's order; without capacities everything is returned."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 2 and a.strides[1] == 1
    h, w = a.shape
    if h == 0 or w == 0:
        return 0, 0, np.zeros(0, np.int32), np.zeros((0, 2), np.int32)
    lib = load()
    nc, npt = C.c_int(0), C.c_long(0)
    if max_contours is None or max_points is None:  # first call for the totals
        rc = lib.oracle_find_contours_external(a.ctypes.data_as(C.c_void_p), w, h, a.strides[0], 0, 0, C.byref(nc),
                                               C.byref(npt), None, None)
        assert rc == 0
        max_contours = nc.value if max_contours is None else max_contours
        max_points = npt.value if max_points is None else max_points
    lengths = np.zeros(max(int(max_contours), 1), np.int32)
    points = np.zeros((max(int(max_points), 1), 2), np.int32)
    rc = lib.oracle_find_contours_external(a.ctypes.data_as(C.c_void_p), w, h, a.strides[0], int(max_contours),
                                           int(max_points), C.byref(nc), C.byref(npt), lengths.ctypes.data_as(C.c_void_p),
                                           points.ctypes.data_as(C.c_void_p))
    assert rc == 0
    n, total = nc.value, npt.value
    return n, total, lengths[:min(n, int(max_contours))], points[:min(total, int(max_points))]


def cv2_contours(contours):
    """cv2's contour list -> (lengths int32, points [total, 2] int32), the oracle's layout."""
    lengths = np.array([len(c) for c in contours], np.int32)
    points = (np.concatenate([c.reshape(-1, 2) for c in contours]).astype(np.int32) if contours
              else np.zeros((0, 2), np.int32))
    return lengths, points
