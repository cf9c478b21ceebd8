"""Mask R-CNN pre-process (preprocessImg, rcnn/common.hpp:79-110, + the float widening of rcnn/rcnn.cpp:504-505) on the CPU:
the geometry the library derives from trtx_rcnn_letterbox_pads against the resize size and paste rectangle of the reference's
compiled preprocessImg (oracle/_ref/libref_rcnn_pre_host.so, or tests/golden/ref_rcnn_pre_host.npz where it was not built), the
oracle's canvases against a cv2 restatement of preprocessImg bit for bit (OpenCV's IPP on and off), and the argument checks
of trtx_rcnn_preprocess_enqueue."""
import ctypes as C

import numpy as np
import pytest

from oracle import rcnn_pre as RP
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

G = RefOutputs("ref_rcnn_pre_host")
F = np.float32


def calculate_size(img_w, img_h, min_size=800.0, max_size=1333.0):
    """calculateSize, rcnn/rcnn.cpp:349-366 -> (INPUT_W, INPUT_H)."""
    ratio = F(min_size) / F(min(img_h, img_w))
    if img_h < img_w:
        newh, neww = F(min_size), F(ratio * F(img_w))
    else:
        newh, neww = F(ratio * F(img_h)), F(min_size)
    if max(newh, neww) > max_size:
        ratio = F(max_size) / F(max(newh, neww))
        newh, neww = F(newh * ratio), F(neww * ratio)
    return int(float(neww) + 0.5), int(float(newh) + 0.5)


def _geometry_cases():
    cases = []
    for w, h in ((640, 480), (480, 640), (1920, 1080), (1080, 1920), (640, 640), (1, 1), (3, 2), (3, 1001), (1001, 3),
                 (641, 479), (1067, 800), (2134, 1600), (533, 400), (4000, 3000), (3000, 4000), (1279, 721), (17, 13)):
        cases.append((w, h) + calculate_size(w, h))
        cases.append((w, h, 1067, 800))
        cases.append((w, h, 800, 1067))
    rng = np.random.default_rng(21)
    for _ in range(150):   # landscape and portrait engines
        w, h = (int(v) for v in rng.integers(64, 3000, 2))
        cases.append((w, h) + calculate_size(w, h))
        cases.append((w, h) + calculate_size(h, w))
    for w in range(600, 640, 3):   # odd and even gaps on both axes
        cases.append((w, 480, 1067, 800))
        cases.append((480, w, 1067, 800))
    return cases


def _rect(lib, w, h, nw, nh):
    """(w, h, x, y) of the resized image as the library derives it: net - (pad_a + pad_b), at (pad_left, pad_top)."""
    p = (C.c_int * 4)()
    assert lib.trtx_rcnn_letterbox_pads(w, h, nw, nh, p) == 0
    return (nw - (p[0] + p[1]), nh - (p[2] + p[3]), p[0], p[2])


def test_geometry_equals_reference():
    """The resize size and paste rectangle of the reference's preprocessImg = trtx_rcnn_letterbox_pads + net - pads."""
    ref = G.lib("libref_rcnn_pre_host.so")
    lib = L.load()
    cases = _geometry_cases()
    assert len(cases) >= 200
    mine, refs = [], []
    gaps = set()
    for (w, h, nw, nh) in cases:
        rw, rh, x, y = _rect(lib, w, h, nw, nh)
        gaps.add(((nw - rw) % 2, (nh - rh) % 2))
        mine.append([rw, rh, x, y, rw, rh, w, h, nw, nh])     # resize (w, h), paste (x, y, w, h), then the case
        if ref is not None:
            g = np.zeros(6, np.int32)
            ref.ref_rcnn_preprocess_geometry(w, h, nw, nh, g.ctypes.data_as(C.c_void_p))
            refs.append(list(g) + [w, h, nw, nh])
    assert {(1, 0), (0, 1), (0, 0)} <= gaps                  # odd and even gaps
    G.equal("rcnn_pre_geometry", np.array(mine, np.int32), np.array(refs, np.int32) if ref is not None else None)


# ------------------------------------------------------------------ oracle vs cv2 ------------------------------
def _cv2_preprocess(cv2, img, net_w, net_h):
    """preprocessImg in cv2, line by line (float / int conversions as in common.hpp:80-102), then astype(float32)."""
    rows, cols = img.shape[:2]
    r_w = F(net_w / (cols * 1.0))
    r_h = F(net_h / (rows * 1.0))
    if r_h > r_w:
        w, h = net_w, int(F(r_w * F(rows)))
        x, y = F(0), F(F(net_h - h) / F(2))
    else:
        w, h = int(F(r_h * F(cols))), net_h
        x, y = F(F(net_w - w) / F(2)), F(0)
    left, top = int(np.round(np.float64(x) - 0.1)), int(np.round(np.float64(y) - 0.1))
    re = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
    out = np.full((net_h, net_w, 3), 128, np.uint8)
    out[top:top + h, left:left + w] = re
    return out.astype(np.float32), (left, top, w, h)


ORACLE_SIZES = [(640, 480, 1067, 800), (1066, 800, 1067, 800), (2134, 1600, 1067, 800), (533, 400, 1067, 800),
                (4000, 3000, 1067, 800), (1920, 1080, 1067, 600), (1920, 1080, 1333, 750), (480, 640, 800, 1067),
                (1080, 1920, 750, 1333), (1, 1, 1067, 800), (3, 2, 1067, 800), (641, 479, 1067, 800), (1067, 800, 1067, 800)]


def _oracle_sweep_sizes():
    rng = np.random.default_rng(22)
    out = []
    while len(out) < 110:
        w, h = (int(v) for v in rng.integers(1, 1400, 2))
        if rng.random() < 0.7 and min(w, h) * 8 > max(w, h):
            nw, nh = calculate_size(w, h)
        else:
            nw, nh = (int(v) for v in rng.integers(16, 400, 2))
        if min(_rect(L.load(), w, h, nw, nh)[:2]) > 0:      # empty rectangles: test_empty_rectangle
            out.append((w, h, nw, nh))
    return out


@pytest.mark.parametrize("ipp", [True, False])
def test_oracle_equals_cv2(ipp):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(23 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for (w, h, nw, nh) in ORACLE_SIZES + _oracle_sweep_sizes():
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            buf = np.zeros((h, w * 3 + 7), np.uint8)                        # an odd pitch and an unaligned base
            buf[:, 1:w * 3 + 1] = img.reshape(h, w * 3)
            pitched = np.lib.stride_tricks.as_strided(buf[:, 1:], (h, w, 3), (w * 3 + 7, 3, 1))
            ref, rect = _cv2_preprocess(cv2, img, nw, nh)
            got = RP.rcnn_preprocess(pitched, nw, nh)
            assert got is not None, (w, h, nw, nh)
            assert got[1] == rect, (w, h, nw, nh)
            assert np.array_equal(got[0], ref), (w, h, nw, nh, int((got[0] != ref).sum()))
    finally:
        cv2.ipp.setUseIPP(old)


def test_empty_rectangle():
    """1 x 5000 into 1067 x 800 resizes to width 0: cv::resize throws, the oracle refuses, the library returns UNSUPPORTED."""
    cv2 = pytest.importorskip("cv2")
    img = np.zeros((5000, 1, 3), np.uint8)
    with pytest.raises(cv2.error):
        _cv2_preprocess(cv2, img, 1067, 800)
    assert RP.rcnn_preprocess(img, 1067, 800) is None
    assert _rect(L.load(), 1, 5000, 1067, 800)[0] == 0


# ------------------------------------------------------------------ argument validation ------------------------
def test_rcnn_preprocess_argument_validation():
    """Every descriptor is checked before anything is launched (the pointers here are never dereferenced: a call that got as
    far as a launch would fail with TRTX_ERR_CUDA on a machine without a GPU, or fault on one with)."""
    lib = L.load()

    def descs(*sizes, ptr=4096, pitch=None):
        d = (L.ImageDesc * len(sizes))()
        for i, (w, h) in enumerate(sizes):
            d[i].data_dev, d[i].width, d[i].height = ptr, w, h
            d[i].pitch = 3 * w if pitch is None else pitch
        return d

    inv, uns = L.ERR_INVALID, L.ERR_UNSUPPORTED
    ok = descs((640, 480), (480, 640))
    assert lib.trtx_rcnn_preprocess_enqueue(None, 2, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, 0, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, -1, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, 2, 0, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, 2, 1067, -800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, 2, 1067, 800, None, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(ok, 2, 1067, 800, 4098, None) == inv         # not a float address
    assert lib.trtx_rcnn_preprocess_enqueue(descs((640, 480), (640, 480), ptr=None), 2, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(descs((640, 480), (0, 480)), 2, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(descs((640, 480), (640, -1)), 2, 1067, 800, 4096, None) == inv
    assert lib.trtx_rcnn_preprocess_enqueue(descs((640, 480), pitch=1919), 1, 1067, 800, 4096, None) == inv
    # the last descriptor is bad: the call is refused as a whole
    assert lib.trtx_rcnn_preprocess_enqueue(descs(*([(640, 480)] * 70 + [(640, 0)])), 71, 1067, 800, 4096, None) == inv
    # an empty resized rectangle (cv::resize throws), also behind valid images
    assert lib.trtx_rcnn_preprocess_enqueue(descs((1, 5000)), 1, 1067, 800, 4096, None) == uns
    assert lib.trtx_rcnn_preprocess_enqueue(descs((640, 480), (5000, 1)), 2, 1067, 800, 4096, None) == uns
    # rows wider than the kernel's shared-memory stage
    assert lib.trtx_rcnn_preprocess_enqueue(descs((6000, 100)), 1, 6000, 100, 4096, None) == uns
