"""The bicubic letterbox pre-process of yolov3-tiny and retinafaceAntiCov on the CPU: the oracle (oracle/cubic_oracle.c) against
cv2's 8-bit INTER_CUBIC with IPP off (bit for bit) and on (within 1), a numpy restatement of the resize that shows which
vertical pass OpenCV runs where, the whole preprocess_img + plane loop restated in Python around cv2, the 256 values of each
variant, and the argument checks of trtx_cubic_preprocess_enqueue that reject before any launch."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from oracle import cubic as CO
from tensorrtx_b200 import _lib as L

cv2 = pytest.importorskip("cv2")
F = np.float32
VARIANTS = (CO.YOLOV3_TINY, CO.ANTICOV)


@contextlib.contextmanager
def _ipp(on: bool):
    old_ipp, old_ocl = cv2.ipp.useIPP(), cv2.ocl.useOpenCL()
    cv2.ipp.setUseIPP(on)
    cv2.ocl.setUseOpenCL(False)
    try:
        yield
    finally:
        cv2.ipp.setUseIPP(old_ipp)
        cv2.ocl.setUseOpenCL(old_ocl)


def _cv_cubic(img, dw, dh, ipp=False):
    with _ipp(ipp):
        return cv2.resize(np.ascontiguousarray(img), (dw, dh), interpolation=cv2.INTER_CUBIC)


def _frame(rng, w, h, pad=0):
    """A random u8 BGR frame [h, w, 3], as a view into rows of 3 * w + pad bytes."""
    buf = rng.integers(0, 256, (h, 3 * w + pad), dtype=np.uint8)
    return buf[:, :3 * w].reshape(h, w, 3) if pad == 0 else np.lib.stride_tricks.as_strided(
        buf, (h, w, 3), (buf.strides[0], 3, 1))


# ------------------------------------------------------------------ a numpy restatement of the resize -----------------
def _cubic_axis(dn, sn):
    """resizeGeneric_'s tables of one axis: the 4 clamped taps and saturate_cast<short>(interpolateCubic(fx) * 2048)."""
    f = ((np.arange(dn) + 0.5) * (1.0 / (dn / sn)) - 0.5).astype(F)
    s = np.floor(f).astype(np.int64)
    x = f - s.astype(F)
    A, one = F(-0.75), F(1)
    x1, mx = x + one, one - x
    c0 = ((A * x1 - F(5) * A) * x1 + F(8) * A) * x1 - F(4) * A
    c1 = ((A + F(2)) * x - (A + F(3))) * x * x + one
    c2 = ((A + F(2)) * mx - (A + F(3))) * mx * mx + one
    c3 = one - c0 - c1 - c2
    w = np.rint(np.stack([c0, c1, c2, c3], 1) * F(2048)).astype(np.int64)
    return np.clip(s[:, None] - 1 + np.arange(4)[None, :], 0, sn - 1), w


def _np_cubic(img, dw, dh, vector_bytes):
    """cv::resize INTER_CUBIC restated: int horizontal pass; vertical pass in float (h0 b0' + (h1 b1' + (h2 b2' + h3 b3')),
    rounded half to even) for the first vector_bytes(3 * dw) bytes of a row and in fixed point ((sum + 2^21) >> 22) after."""
    sh, sw, _ = img.shape
    if (sw, sh) == (dw, dh):
        return np.array(img)
    xt, xw = _cubic_axis(dw, sw)
    yt, yw = _cubic_axis(dh, sh)
    H = (np.asarray(img).astype(np.int64)[:, xt, :] * xw[None, :, :, None]).sum(2).reshape(sh, 3 * dw)
    R = H[yt]
    fix = ((R * yw[:, :, None]).sum(1) + (1 << 21)) >> 22
    Rf, b = R.astype(F), yw.astype(F) * F(1.0 / (2048 * 2048))
    t = Rf[:, 3] * b[:, 3:4]
    for k in (2, 1, 0):
        t = Rf[:, k] * b[:, k:k + 1] + t
    nv = vector_bytes(3 * dw)
    out = fix
    out[:, :nv] = np.rint(t[:, :nv])
    return np.clip(out, 0, 255).astype(np.uint8).reshape(dh, dw, 3)


OPENCV = lambda W: W & ~7  # the 8-lane SSE loop of VResizeCubicVec_32s8u, then the scalar tail
ALTERNATIVES = {"16 lanes": lambda W: W & ~15, "all fixed point": lambda W: 0, "all float": lambda W: W}


def _letterbox_rect(w, h, net_w, net_h):
    r = (C.c_int * 4)()
    assert L.load().trtx_calib_letterbox_rect(w, h, net_w, net_h, r) == 0
    return tuple(r)


# (src w, h) -> (dst w, h): up- and downscales, integer ratios, the identity, 1-pixel-wide and -tall frames, odd sizes, and
# the letterbox rectangles of 608 and 640 nets
RESIZES = [((640, 480), (608, 456)), ((300, 200), (608, 405)), ((1920, 1080), (608, 342)), ((1920, 1080), (640, 360)),
           ((2, 2), (608, 608)), ((640, 640), (640, 640)), ((1, 37), (16, 608)), ((37, 1), (608, 16)), ((1, 1), (5, 3)),
           ((33, 17), (607, 313)), ((5, 7), (9, 11)), ((999, 555), (607, 337)), ((100, 100), (33, 33)),
           ((1280, 720), (640, 360)), ((320, 240), (640, 480)), ((53, 77), (67, 79)), ((1, 92), (47, 46)),
           ((24, 39), (24, 78)), ((19, 61), (30, 49)), ((4000, 3), (608, 1)), ((7, 1001), (5, 601))]
NET_RECTS = [((w, h), _letterbox_rect(w, h, n, n)[2:]) for n in (608, 640)
             for w, h in ((1920, 1080), (1280, 720), (640, 480), (480, 640), (300, 200), (1, 2), (3001, 17), (608, 608))]


@pytest.mark.parametrize("src,dst", RESIZES + NET_RECTS, ids=lambda v: "x".join(map(str, v)))
def test_oracle_and_numpy_equal_cv2_without_ipp(src, dst):
    """Bit for bit, on a pitched random frame and on a frame of the extreme bytes 0 and 255 (which saturates)."""
    rng = np.random.default_rng(hash((src, dst)) & 0xFFFF)
    for img in (_frame(rng, *src, pad=5), (_frame(rng, *src) >> 7) * 255):
        exp = _cv_cubic(img, *dst)
        assert np.array_equal(CO.resize(img, *dst), exp)
        assert np.array_equal(_np_cubic(img, *dst, OPENCV), exp)


def test_the_vertical_pass_split_is_what_opencv_runs():
    """Over random small sizes the 8-lane float prefix + fixed-point tail matches cv2 on every byte, and each alternative form
    (a 16-lane prefix, fixed point throughout, float throughout) misses somewhere: so the tests above discriminate them."""
    rng = np.random.default_rng(7)
    misses = dict.fromkeys(ALTERNATIVES, 0)
    for _ in range(1000):
        sw, sh, dw, dh = (int(v) for v in rng.integers(1, 130, 4))
        img = _frame(rng, sw, sh)
        exp = _cv_cubic(img, dw, dh)
        assert np.array_equal(CO.resize(img, dw, dh), exp), (sw, sh, dw, dh)
        for name, split in ALTERNATIVES.items():
            misses[name] += int((_np_cubic(img, dw, dh, split) != exp).sum())
    assert all(m > 0 for m in misses.values()), misses


@pytest.mark.parametrize("src,dst", [((640, 480), (608, 456)), ((300, 200), (608, 405)), ((1920, 1080), (608, 342)),
                                     ((1920, 1080), (640, 360)), ((2, 2), (608, 608)), ((1280, 720), (640, 360))])
def test_oracle_within_one_of_cv2_with_ipp(src, dst):
    """cv2 with IPP (x86 wheels' default) rounds differently: |delta| <= 1; integer ratios agree exactly."""
    rng = np.random.default_rng(3)
    img = _frame(rng, *src)
    d = CO.resize(img, *dst).astype(np.int16) - _cv_cubic(img, *dst, ipp=True)
    assert np.abs(d).max() <= 1
    if src[0] % dst[0] == 0 and src[1] % dst[1] == 0 or src == (2, 2):
        assert not d.any()


# ------------------------------------------------------------------ the whole chain, restated ---------------------------
def _py_value(variant, u):
    u = int(u)
    return F(u / 255.0) if variant == CO.YOLOV3_TINY else F((float(F(u)) - 127.5) * 0.0078125)


def _py_preprocess(img, variant, net_w, net_h):
    """preprocess_img statement by statement (float r_w, r_h from double divisions, products truncated to int), cv2 for the
    resize (IPP off), the 128 canvas, then the driver's plane loop data[i + c * H * W] = value(pixel i, byte 2 - c)."""
    rows, cols = img.shape[:2]
    r_w, r_h = F(net_w / (cols * 1.0)), F(net_h / (rows * 1.0))
    if r_h > r_w:
        w, h = net_w, int(r_w * F(rows))
        x, y = 0, int((net_h - h) / 2)
    else:
        w, h = int(r_h * F(cols)), net_h
        x, y = int((net_w - w) / 2), 0
    out = np.full((net_h, net_w, 3), 128, np.uint8)
    out[y:y + h, x:x + w] = _cv_cubic(img, w, h)
    lut = np.array([_py_value(variant, u) for u in range(256)], F)
    return np.stack([lut[out[:, :, 2 - c]] for c in range(3)]), (x, y, w, h)


@pytest.mark.parametrize("variant", VARIANTS)
def test_chain_equals_preprocess_img_and_the_plane_loop(variant):
    rng = np.random.default_rng(11 + variant)
    for (w, h), net in (((1920, 1080), 608), ((640, 480), 640), ((480, 640), 608), ((300, 200), 640), ((97, 301), 608),
                        ((608, 608), 608), ((1, 3), 640), ((5, 1), 608)):
        img = _frame(rng, w, h, pad=(w % 3) + 1)
        got, rect = CO.preprocess(img, variant, net, net)
        exp, exp_rect = _py_preprocess(img, variant, net, net)
        assert rect == exp_rect == _letterbox_rect(w, h, net, net), (w, h, net)
        assert np.array_equal(got, exp), (w, h, net)
    for (w, h), (net_w, net_h) in (((640, 480), (320, 608)), ((1280, 720), (608, 416))):  # rectangular nets
        img = _frame(rng, w, h)
        assert np.array_equal(CO.preprocess(img, variant, net_w, net_h)[0], _py_preprocess(img, variant, net_w, net_h)[0])


def test_values_of_all_256_bytes():
    """yolov3-tiny: u / 255.0 rounded once from double; retinafaceAntiCov: (u - 127.5) / 128, exact in float."""
    for variant in VARIANTS:
        got = np.array([CO.input_value(variant, u) for u in range(256)], F)
        assert np.array_equal(got, np.array([_py_value(variant, u) for u in range(256)], F)), variant
    anti = np.array([CO.input_value(CO.ANTICOV, u) for u in range(256)], np.float64)
    assert np.array_equal(anti, (np.arange(256) - 127.5) / 128)
    tiny = np.array([CO.input_value(CO.YOLOV3_TINY, u) for u in range(256)], F)
    assert np.array_equal(tiny, (np.arange(256) / 255.0).astype(F))
    assert tiny[0] == 0 and tiny[255] == 1 and np.all(np.diff(tiny) > 0)


def test_oracle_rejects_what_cv_resize_rejects():
    assert CO.preprocess(np.zeros((5000, 1, 3), np.uint8), CO.YOLOV3_TINY, 608, 608) is None  # w = (int)(0.1216 * 1) = 0
    assert CO.preprocess(np.zeros((1, 5000, 3), np.uint8), CO.ANTICOV, 640, 640) is None


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_rejected_arguments():
    lib = L.load()
    descs = (L.ImageDesc * 2)()
    for d in descs:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    pre = lambda v=CO.YOLOV3_TINY, d=descs, b=2, w=608, h=608, dst=16: lib.trtx_cubic_preprocess_enqueue(v, d, b, w, h, dst,
                                                                                                          None)
    assert pre(d=None) == L.ERR_INVALID
    assert pre(b=0) == L.ERR_INVALID
    assert pre(b=-1) == L.ERR_INVALID
    assert pre(w=0) == L.ERR_INVALID
    assert pre(h=-1) == L.ERR_INVALID
    assert pre(dst=None) == L.ERR_INVALID
    assert pre(dst=18) == L.ERR_INVALID  # not 4-byte aligned
    for v in (-1, 2, L.YOLO_V3):
        assert pre(v=v) == L.ERR_INVALID, v
    descs[1].pitch = 11  # < 3 * width
    assert pre() == L.ERR_INVALID
    descs[1].pitch, descs[1].data_dev = 12, None
    assert pre() == L.ERR_INVALID
    descs[1].data_dev, descs[1].height = 16, 0
    assert pre() == L.ERR_INVALID
    descs[1].height, descs[1].width = 4, -1
    assert pre() == L.ERR_INVALID
    # an empty rectangle, where cv::resize throws: 1 x 5000 at 608 gives w = (int)(0.1216f * 1) = 0
    descs[1].width, descs[1].height, descs[1].pitch = 1, 5000, 3
    assert pre() == L.ERR_UNSUPPORTED
    assert pre(v=CO.ANTICOV, w=640, h=640) == L.ERR_UNSUPPORTED
    # staged rows beyond shared memory: a 1200-wide rectangle shrunk 4x vertically needs 16 rows of 3 * 1200 ints
    descs[1].width, descs[1].height, descs[1].pitch = 4800, 100, 14400
    assert pre(w=1200, h=1200) == L.ERR_UNSUPPORTED
    # an invalid descriptor after an unsupported one is still TRTX_ERR_INVALID: every descriptor is checked first
    big = (L.ImageDesc * 70)()
    for d in big:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    big[0].width, big[0].height, big[0].pitch = 1, 5000, 3
    big[69].pitch = 0
    assert lib.trtx_cubic_preprocess_enqueue(0, big, 70, 608, 608, 16, None) == L.ERR_INVALID
