"""ctypes/numpy wrapper around oracle/libv3family_oracle.so: the CPU oracle of the yolov3 family's decode, each driver's box
arithmetic and sigmoid (oracle/v3family_oracle.c; recipe oracle/Makefile).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base

HERE = Path(__file__).resolve().parent
LIB = HERE / "libv3family_oracle.so"
SPP, NET, V4, CSP = 2, 4, 5, 6  # box modes = the library's TRTX_YOLO_V3 / V3_NET / V4 / V4_CSP
_lib = None


def load():
    global _lib
    if _lib is None:
        _lib = _base.build_and_open(LIB)
    return _lib


def decode(heads, anchors, box_mode, net=(0, 0), strides=None, nc=80, max_out=1000, ignore_thresh=0.1):
    """heads: per level [B, 3*(5+nc), gh, gw] in the plugin's level order; anchors: 6 per level; net = (INPUT_W, INPUT_H)
    for modes NET / V4 / CSP, strides for SPP.  -> (out [B, 1+max_out*7], anchor_idx [B, max_out])."""
    lib = load()
    B = heads[0].shape[0]
    flat = [np.ascontiguousarray(h.reshape(B, h.shape[1], -1), np.float32) for h in heads]
    ptrs = (C.c_void_p * len(flat))(*[f.ctypes.data for f in flat])
    ia = lambda v: (C.c_int * len(v))(*[int(x) for x in v])  # noqa: E731
    gh, gw = [h.shape[2] for h in heads], [h.shape[3] for h in heads]
    st = list(strides) if strides is not None else [0] * len(flat)
    anc = np.ascontiguousarray(np.asarray(anchors, np.float32).reshape(-1))
    out = np.zeros((B, 1 + max_out * 7), np.float32)
    idx = np.full((B, max_out), -1, np.int32)
    lib.oracle_v3family_decode(ptrs, B, len(flat), ia(gh), ia(gw), ia(st), anc.ctypes.data_as(C.c_void_p), nc, max_out,
                               C.c_float(ignore_thresh), int(box_mode), int(net[0]), int(net[1]),
                               out.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p))
    return out, idx
