"""ctypes/numpy wrapper around oracle/libufld_oracle.so: the CPU oracle of the UFLD lane-detection pre- and post-process
(prepareImage, the driver's argmax and softmax_mul, and its loop from the flip to the points).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import oracle as _base


HERE = Path(__file__).resolve().parent
LIB = HERE / "libufld_oracle.so"
NET_W, NET_H = 800, 288  # INPUT_W, INPUT_H
SHAPE = (101, 56, 4)     # OUTPUT_C, OUTPUT_H, OUTPUT_W
COL_SAMPLE_W = 8
TUSIMPLE_ROW_ANCHOR = tuple(range(64, 288, 4))
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_ufld_input_value.restype = C.c_float
    _lib.oracle_ufld_postprocess.restype = C.c_int
    _lib.oracle_ufld_exp_disagreements.restype = C.c_long
    _lib.oracle_ufld_exp_disagreements.argtypes = [C.c_float, C.c_float, C.c_uint]
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def input_value(c: int, u: int) -> np.float32:
    """The engine input value of byte u in plane c (0 = R, 1 = G, 2 = B)."""
    return np.float32(load().oracle_ufld_input_value(int(c), int(u)))


def preprocess(img, net_w: int = NET_W, net_h: int = NET_H) -> np.ndarray:
    """prepareImage for one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> [3, net_h, net_w] float32 planes R, G, B."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net_h, net_w), np.float32)
    load().oracle_ufld_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                  int(net_w), int(net_h), _vp(out))
    return out


def argmax(x) -> np.ndarray:
    """The driver's argmax over axis 0 of x [C, H, W] float32 -> [H, W] float32 indices."""
    x = np.ascontiguousarray(x, np.float32)
    Cn, H, W = x.shape
    y = np.empty((H, W), np.float32)
    load().oracle_ufld_argmax(_vp(x), _vp(y), H, W, Cn)
    return y


def softmax_mul(x) -> np.ndarray:
    """The driver's softmax_mul over axis 0 of x [C, H, W] float32 (the first C - 1 entries) -> [H, W] float32 expectations."""
    x = np.array(x, np.float32, order="C", copy=True)
    Cn, H, W = x.shape
    y = np.empty((H, W), np.float32)
    load().oracle_ufld_softmax_mul(_vp(x), _vp(y), H, W, Cn)
    return y


def postprocess(prob, vis_w: int = 1280, vis_h: int = 720, row_anchor=TUSIMPLE_ROW_ANCHOR, net_w: int = NET_W,
                net_h: int = NET_H, col_sample_w: int = COL_SAMPLE_W) -> np.ndarray:
    """The driver loop of lane_det.cpp:358-410 over one frame: prob [C, H, W] float32 -> rows [1 + H*W*3]: the point count,
    then (x, y, lane) per point in draw order, zeros past the count."""
    p = np.ascontiguousarray(prob, np.float32)
    Cn, H, W = p.shape
    anchors = np.ascontiguousarray(row_anchor, np.int32)
    assert anchors.shape == (H,)
    out = np.empty(1 + H * W * 3, np.float32)
    load().oracle_ufld_postprocess(_vp(p), Cn, H, W, _vp(anchors), int(net_w), int(net_h), int(col_sample_w), int(vis_w),
                                   int(vis_h), _vp(out))
    return out


def exp_disagreements(lo: float, hi: float, stride: int = 1) -> int:
    """How many floats in [lo, hi] (every `stride`-th bit pattern from zero outwards) have glibc's expf(x) !=
    (float)exp((double)x)."""
    return int(load().oracle_ufld_exp_disagreements(lo, hi, stride))


# ------------------------------------------------------------------ test inputs ----------------------------------------
def edge_cells(C_=101, seed=5):
    """prob [C, 16, 4] whose cells cover the argmax and softmax_mul edges: ties, the truncation quirk, NaN, +-inf, logits
    above 88.7 (exp overflows), all-underflow cells, cells where max_ind stays -1, and plain random logits."""
    rng = np.random.default_rng(seed)
    H, W = 16, 4
    p = rng.normal(0, 3, (C_, H, W)).astype(np.float32)
    cell = lambda k: (slice(None), k // W, k % W)     # cell k: row k // W, lane k % W
    p[cell(0)] = 1.0                                    # all equal: the first wins
    p[[3, 9], 0, 1] = 20.0                              # two equal maxima: the first wins
    p[cell(2)] = -5.0
    p[3, 0, 2], p[7, 0, 2] = 3.7, 3.2                   # 3.2 > (float)(int)3.7: index 7 wins
    p[cell(3)] = -20000000.0                            # every value below -1e7: max_ind stays -1
    p[cell(4)] = np.nan                                 # all NaN: max_ind -1, expect NaN
    p[cell(5)] = np.linspace(-3, 3, C_)
    p[10, 1, 1] = np.inf                                # +inf: max = INT_MIN, so every later value above it wins
    p[5, 1, 2] = np.nan                                 # one NaN among finite logits
    p[20, 1, 2] = -np.inf
    p[11, 1, 3], p[12, 1, 3] = 100.0, 95.0              # exp overflows: inf / inf
    p[cell(8)] = 89.0                                   # every exp overflows
    p[cell(9)] = -200.0                                 # every exp underflows: 0 / 0
    p[cell(10)] = -100.0                                # subnormal exps
    p[C_ - 1, 2, 3] = 50.0                              # the "no lane" cell wins
    p[cell(12)] = 3e9                                   # above the int range: INT_MIN, then every later value
    p[0, 3, 0] = -1e7                                   # equal to the start: not taken
    p[0, 3, 1] = 2147483520.0                           # the largest float below 2^31 truncates exactly
    return p


def lane_prob(C_=101, H=56, W=4, seed=0, nan_cell=True):
    """Logits where lane 0 has points in most rows, lane 1 exactly 3 non-zero rows, lane 2 exactly 2, lane 3 none (its
    "no lane" cell wins everywhere), plus a NaN expectation in lane 0."""
    rng = np.random.default_rng(seed)
    p = rng.normal(0, 1, (C_, H, W)).astype(np.float32)
    p[C_ - 1] = 8.0                                     # "no lane" everywhere ...
    for j in range(H):
        if j % 5:
            p[C_ - 1, j, 0] = -8.0                      # ... but lane 0, 4 rows in 5
            p[rng.integers(0, C_ - 1), j, 0] = 9.0
    for j in (3, 17, 40 % H):
        p[C_ - 1, j, 1] = -8.0
    for j in (5, 30 % H):
        p[C_ - 1, j, 2] = -8.0
    if nan_cell:
        p[C_ - 1, 1, 0] = -8.0
        p[0, 1, 0] = np.nan                             # argmax skips it, the expectation is NaN: counted, not drawn
    return p
