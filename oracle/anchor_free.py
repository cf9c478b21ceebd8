"""ctypes/numpy wrapper around oracle/libanchor_free_oracle.so: the CPU oracle of yolov9's converting nms() and yolov10's
get_topk + get_rect (oracle/anchor_free_oracle.c; recipe oracle/anchor_free.mk).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / "libanchor_free_oracle.so"
_lib = None


def load():
    global _lib
    if _lib is None:
        src = HERE / "anchor_free_oracle.c"
        if not LIB.exists() or LIB.stat().st_mtime < src.stat().st_mtime:
            subprocess.run(["make", "-C", str(HERE), "-f", "anchor_free.mk", str(LIB)], check=True, stdout=subprocess.DEVNULL)
        _lib = C.CDLL(str(LIB))
        _lib.oracle_v9_nms.restype = C.c_int
        _lib.oracle_topk.restype = C.c_int
    return _lib


def v9_nms(plugin_out_img, max_rows, det_floats, conf_thresh, nms_thresh):
    """One image's plugin buffer [1 + rows*det_floats] -> (kept rows [n, det_floats] with converted boxes, source row [n])."""
    lib = load()
    p = np.ascontiguousarray(plugin_out_img, np.float32)
    res = np.zeros((max(max_rows, 1), det_floats), np.float32)
    src = np.zeros(max(max_rows, 1), np.int32)
    n = lib.oracle_v9_nms(p.ctypes.data_as(C.c_void_p), int(max_rows), int(det_floats), C.c_float(conf_thresh),
                          C.c_float(nms_thresh), res.ctypes.data_as(C.c_void_p), src.ctypes.data_as(C.c_void_p))
    return res[:n].copy(), src[:n].copy()


def topk(plugin_out_img, max_rows, row_floats, conf_thresh, img_w, img_h, variant=0, net=(640, 640)):
    """One image -> its (x, y, w, h, conf, class) rows [n, 6]."""
    lib = load()
    p = np.ascontiguousarray(plugin_out_img, np.float32)
    rows = np.zeros((max(max_rows, 1), 6), np.float32)
    n = lib.oracle_topk(p.ctypes.data_as(C.c_void_p), int(max_rows), int(row_floats), C.c_float(conf_thresh), int(variant),
                        int(net[0]), int(net[1]), int(img_w), int(img_h), rows.ctypes.data_as(C.c_void_p))
    return rows[:n].copy()
