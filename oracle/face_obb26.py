"""ctypes/numpy wrappers around two reference builds of oracle/Makefile (present where the reference tree was at build
time): yolo26's own draw_bbox_obb (oracle/_ref/libref_obb26_host.so) and retina_r50.cpp:373-388's host loop
(oracle/_ref/libref_retina_rows_host.so).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from .golden import RefOutputs


@functools.cache
def load_obb26():
    """yolo26's compiled draw_bbox_obb (None where oracle/_ref was not built)."""
    return RefOutputs.lib("libref_obb26_host.so")


@functools.cache
def load_retina_rows():
    """retina_r50.cpp:373-388's compiled loop, ref_retina_rows (None where oracle/_ref was not built)."""
    lib = RefOutputs.lib("libref_retina_rows_host.so")
    if lib is not None:
        lib.ref_retina_rows.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double,
                                        C.c_void_p, C.c_void_p]
    return lib


def ref_draw_bbox_obb_v26(img_w, img_h, boxes5):
    """boxes5 [n, 5] (cx, cy, w, h, angle) of one frame through yolo26's draw_bbox_obb (net 1024) -> (corners [n, 8] int32
    as get_corner hands them to cv::polylines, the text it printed)."""
    b = np.ascontiguousarray(boxes5, np.float32).reshape(-1, 5)
    n = b.shape[0]
    corners = np.zeros((n, 8), np.int32)
    cap = 128 * n + 64
    log = C.create_string_buffer(cap)
    length = load_obb26().ref_v26_draw_bbox_obb(int(img_w), int(img_h), n, b.ctypes.data_as(C.c_void_p),
                                                corners.ctypes.data_as(C.c_void_p), log, cap)
    assert length >= 0, "draw_bbox_obb did not draw one polygon per box"
    return corners, log.value.decode()
