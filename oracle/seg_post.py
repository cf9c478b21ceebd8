"""ctypes/numpy wrapper around oracle/libseg_post_oracle.so: the CPU oracle of the YOLO segmentation post-process
(process_mask + scale_mask + draw_mask_bbox's mask selection), and around oracle/_ref/libref_seg_host.so, the reference's own
draw_mask_bbox compiled against a header shim (present where the reference tree was at build time).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
import functools
from pathlib import Path

import numpy as np

from . import oracle as _base
from .golden import RefOutputs

HERE = Path(__file__).resolve().parent
LIB = HERE / "libseg_post_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _base.load()   # libtrtx_oracle.so: process_mask, the bilinear resize, get_rect
    _lib = _base.build_and_open(LIB)
    _lib.oracle_seg_postprocess.restype = C.c_int
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def scale_mask_rect(img_w, img_h, net_w=640, net_h=640):
    r = np.zeros(4, np.int32)
    load().oracle_scale_mask_rect(int(net_w), int(net_h), int(img_w), int(img_h), _p(r))
    return tuple(int(v) for v in r)


def seg_postprocess(variant, proto, dets, img_w, img_h, *, max_rows, row_floats=39, coeff_offset=7, max_masks,
                    net_w=640, net_h=640, canvases=None, scaled=False):
    """One image: proto [nm, mh, mw], dets [1 + max_rows*row_floats] -> (rows [1 + max_rows*6], canvases [max_masks, img_h,
    img_w] u8 (written in place when given; slots past the count keep their bytes), S [max_masks, img_h, img_w] fp32 or None)."""
    lib = load()
    pr = np.ascontiguousarray(proto, np.float32)
    d = np.ascontiguousarray(dets, np.float32)
    nm, mh, mw = pr.shape
    rows = np.zeros(1 + max_rows * 6, np.float32)
    if canvases is None:
        canvases = np.zeros((max_masks, img_h, img_w), np.uint8)
    assert canvases.dtype == np.uint8 and canvases.flags["C_CONTIGUOUS"] and canvases.shape == (max_masks, img_h, img_w)
    S = np.zeros((max_masks, img_h, img_w), np.float32) if scaled else None
    rc = lib.oracle_seg_postprocess(int(variant), _p(pr), nm, mh, mw, int(net_w), int(net_h), _p(d), int(max_rows),
                                    int(row_floats), int(coeff_offset), int(max_masks), int(img_w), int(img_h), _p(rows),
                                    _p(canvases), _p(S))
    if rc != 0:
        raise ValueError(f"empty scale_mask crop for {img_w} x {img_h}")
    return rows, canvases, S


@functools.cache
def load_ref():
    """The reference's compiled draw_mask_bbox (None where oracle/_ref was not built)."""
    _base.load()   # libref_seg_host.so links libtrtx_oracle.so through $ORIGIN/..
    return RefOutputs.lib("libref_seg_host.so")


def ref_draw_mask_select(variant, mask, bbox, img_w, img_h):
    """The pixels the reference's draw_mask_bbox colours for ONE detection (bbox in the variant's format) whose 640 x 640
    process_mask output is `mask`, drawn onto an all-zero img_w x img_h image: bool [img_h, img_w]."""
    ref = load_ref()
    m = np.ascontiguousarray(mask, np.float32)
    b = np.ascontiguousarray(bbox, np.float32)
    sel = np.zeros((img_h, img_w), np.uint8)
    fn = ref.ref_v8_draw_mask_select if variant == 0 else ref.ref_v5_draw_mask_select
    fn(int(img_w), int(img_h), _p(m), _p(b), _p(sel))
    return sel != 0
