"""ctypes/numpy wrapper around oracle/_ref/libref_pose_obb_host.so: the reference's own draw_bbox_obb (get_corner) and
draw_bbox_keypoints_line (get_rect_adapt_landmark) of yolov8 (net 640) and yolo11 (get_rect_obb, net 1024), compiled
against a header shim whose drawing calls record their points (present where the reference tree was at build time).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from .golden import RefOutputs

NUM_KPTS = 17   # kNumberOfPoints of both reference trees


@functools.cache
def load_ref():
    """The reference's compiled drawing functions (None where oracle/_ref was not built)."""
    ref = RefOutputs.lib("libref_pose_obb_host.so")
    if ref is not None:
        for fn in ("ref_v8_draw_bbox_obb", "ref_v11_draw_bbox_obb", "ref_v8_draw_bbox_keypoints_line",
                   "ref_v11_draw_bbox_keypoints_line"):
            getattr(ref, fn).restype = C.c_int
    return ref


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_draw_bbox_obb(tree, img_w, img_h, boxes5):
    """boxes5 [n, 5] (cx, cy, w, h, angle) of one frame through draw_bbox_obb of `tree` ("v8": net 640, "v11": net 1024)
    -> (corners [n, 8] int32 as get_corner hands them to cv::polylines, the text it printed)."""
    b = np.ascontiguousarray(boxes5, np.float32).reshape(-1, 5)
    n = b.shape[0]
    corners = np.zeros((n, 8), np.int32)
    cap = 128 * n + 64
    log = C.create_string_buffer(cap)
    fn = getattr(load_ref(), f"ref_{tree}_draw_bbox_obb")
    length = fn(int(img_w), int(img_h), n, _p(b), _p(corners), log, cap)
    assert length >= 0, "draw_bbox_obb did not draw one polygon per box"
    return corners, log.value.decode()


def ref_draw_bbox_keypoints_line(tree, img_w, img_h, boxes4, kpts):
    """boxes4 [n, 4] (l, t, r, b) and kpts [n, 51] of one frame through draw_bbox_keypoints_line -> (rects [n, 4] int32 as
    drawn, keypoints [n, 51] float32 as get_rect_adapt_landmark mapped them in place)."""
    b = np.ascontiguousarray(boxes4, np.float32).reshape(-1, 4)
    k = np.ascontiguousarray(kpts, np.float32).reshape(-1, 3 * NUM_KPTS)
    n = b.shape[0]
    rects = np.zeros((n, 4), np.int32)
    out = np.zeros_like(k)
    fn = getattr(load_ref(), f"ref_{tree}_draw_bbox_keypoints_line")
    assert fn(int(img_w), int(img_h), n, _p(b), _p(k), _p(rects), _p(out)) == 0
    return rects, out
