"""ctypes/numpy wrapper around oracle/librcnn_post_oracle.so: the CPU oracle of the Mask R-CNN post-process
(rcnn/rcnn.cpp:516-550) and of preprocessImg's pads (rcnn/common.hpp:79-102).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "librcnn_post_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _base.load()   # libtrtx_oracle.so, whose bilinear resize this library uses
    _lib = _base.build_and_open(LIB)
    _lib.oracle_rcnn_postprocess.restype = C.c_int
    return _lib

def rcnn_letterbox_pads(img_w, img_h, net_w, net_h):
    """preprocessImg's pads (rcnn/common.hpp:79-102) -> (left, right, top, bottom)."""
    p = np.zeros(4, np.int32)
    load().oracle_rcnn_letterbox_pads(int(img_w), int(img_h), int(net_w), int(net_h), p.ctypes.data_as(C.c_void_p))
    return tuple(int(v) for v in p)


def rcnn_mask_rect(box, img_w, img_h):
    """The paste rectangle (x, y, w, h) of rcnn/rcnn.cpp:543-546 for a box in original-image pixels, or None where the
    reference throws."""
    b = np.ascontiguousarray(box, np.float32)
    r = np.zeros(4, np.int32)
    ok = load().oracle_rcnn_mask_rect(b.ctypes.data_as(C.c_void_p), int(img_w), int(img_h), r.ctypes.data_as(C.c_void_p))
    return tuple(int(v) for v in r) if ok else None


def rcnn_postprocess(scores, boxes, classes, masks, img_w, img_h, net_w, net_h, score_thresh=0.6, max_masks=None,
                     canvases=None):
    """One image of rcnn/rcnn.cpp:516-550: scores [D], boxes [D,4], classes [D], masks [D,S,S] or None ->
    (rows [1 + D*7], canvases [max_masks, img_h, img_w] u8 or None).  `canvases` (u8, written in place) keeps its slots at or
    past the count."""
    lib = load()
    sc = np.ascontiguousarray(scores, np.float32)
    bx = np.ascontiguousarray(boxes, np.float32)
    cl = np.ascontiguousarray(classes, np.float32)
    D = sc.shape[0]
    max_masks = D if max_masks is None else int(max_masks)
    rows = np.zeros(1 + D * 7, np.float32)
    S, mp, cp = 1, None, None
    if masks is not None:
        m = np.ascontiguousarray(masks, np.float32)
        S = m.shape[-1]
        if canvases is None:
            canvases = np.zeros((max_masks, img_h, img_w), np.uint8)
        assert canvases.dtype == np.uint8 and canvases.flags["C_CONTIGUOUS"] and canvases.shape == (max_masks, img_h, img_w)
        mp, cp = m.ctypes.data_as(C.c_void_p), canvases.ctypes.data_as(C.c_void_p)
    else:
        canvases = None
    lib.oracle_rcnn_postprocess(sc.ctypes.data_as(C.c_void_p), bx.ctypes.data_as(C.c_void_p), cl.ctypes.data_as(C.c_void_p),
                                mp, D, S, int(net_w), int(net_h), int(img_w), int(img_h), C.c_float(score_thresh), max_masks,
                                rows.ctypes.data_as(C.c_void_p), cp)
    return rows, canvases
