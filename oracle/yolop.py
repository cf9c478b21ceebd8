"""ctypes/numpy wrapper around oracle/libyolop_oracle.so: the CPU oracle of the YOLOP pre- and post-process (preprocess_img with
the driver's plane loop, get_rect, and the drivable-area / lane labels).  The NMS is oracle.oracle.nms(1, ...).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base


HERE = Path(__file__).resolve().parent
LIB = HERE / "libyolop_oracle.so"
NET_W, NET_H = 640, 384  # Yolo::INPUT_W, INPUT_H
MAP_W, MAP_H = 640, 360  # Yolo::IMG_W, IMG_H
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_yolop_preprocess.restype = C.c_int
    _lib.oracle_yolop_input_value.restype = C.c_float
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def input_value(c: int, u: int) -> np.float32:
    """The engine input value of byte u in plane c (0 = B, 1 = G, 2 = R)."""
    return np.float32(load().oracle_yolop_input_value(int(c), int(u)))


def preprocess(img, net_w: int = NET_W, net_h: int = NET_H):
    """preprocess_img + the plane loop for one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> ([3, net_h, net_w] float32
    planes B, G, R, (x, y, w, h) of the pasted image), or None where the reference throws."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net_h, net_w), np.float32)
    rect = np.zeros(4, np.int32)
    rc = load().oracle_yolop_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                        int(net_w), int(net_h), _vp(out), _vp(rect))
    return None if rc else (out, tuple(int(v) for v in rect))


def get_rect(img_w: int, img_h: int, bbox, net_w: int = NET_W, net_h: int = NET_H):
    """YOLOP's get_rect -> (x, y, w, h)."""
    b = np.ascontiguousarray(bbox, np.float32)
    r = np.zeros(4, np.int32)
    load().oracle_yolop_get_rect(int(net_w), int(net_h), int(img_w), int(img_h), _vp(b), _vp(r))
    return tuple(int(v) for v in r)


def nearest(dn: int, sn: int) -> np.ndarray:
    """INTER_NEAREST source index of each of dn destination indices over sn source samples -> int32 [dn]."""
    out = np.empty(dn, np.int32)
    load().oracle_yolop_nearest(int(dn), int(sn), _vp(out))
    return out


def labels(seg, lane, img_w: int, img_h: int) -> np.ndarray:
    """The driver's label of every frame pixel from one frame's [map_h, map_w] int32 maps -> u8 [img_h, img_w]: 2 lane,
    1 drivable area, 0 none."""
    s = np.ascontiguousarray(seg, np.int32)
    l_ = np.ascontiguousarray(lane, np.int32)
    out = np.empty((img_h, img_w), np.uint8)
    load().oracle_yolop_labels(_vp(s), _vp(l_), int(s.shape[1]), int(s.shape[0]), int(img_w), int(img_h), _vp(out),
                               C.c_size_t(img_w))
    return out


def rows(nms_rows: np.ndarray, img_w: int, img_h: int, max_rows: int) -> np.ndarray:
    """The post-process rows of one frame from its NMS result [n, >= 6] (cx, cy, w, h, conf, class, ...) -> [1 + max_rows*6]:
    n, then (x, y, w, h, conf, class) with YOLOP's get_rect, zeros past n."""
    out = np.zeros(1 + max_rows * 6, np.float32)
    n = min(len(nms_rows), max_rows)
    out[0] = n
    for i in range(n):
        r = nms_rows[i]
        out[1 + 6 * i:1 + 6 * i + 4] = get_rect(img_w, img_h, r[:4])
        out[1 + 6 * i + 4:1 + 6 * i + 6] = r[4:6]
    return out
