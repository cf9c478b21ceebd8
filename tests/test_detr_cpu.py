"""DETR on the CPU: the oracle (oracle/detr_oracle.c) against cv2 4.13 -- preprocessImg's cvtColor / resize / convertTo /
`/= 255` / `-= Scalar` / `/= Scalar` chain -- and against the driver's per-query loop restated in Python, the library's host
trtx_detr_get_rect against the oracle, and the argument checks of the DETR calls that reject before any launch."""
import ctypes as C

import numpy as np
import pytest

from oracle import detr as DO
from tensorrtx_b200 import _lib as L

F = np.float32
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)  # R, G, B: cvtColor runs first
NET_W, NET_H = 1066, 800
INT_MIN = np.iinfo(np.int32).min


def _cv2_chain(rgb):
    """preprocessImg after the resize, in cv2: convertTo(CV_32FC3) then `img /= 255`, a float product by (float)(1. / 255);
    `img -= Scalar(mean)` (cv::subtract); `img /= Scalar(std)` (cv::divide by a Scalar, a 4 x 1 double Mat)."""
    cv2 = pytest.importorskip("cv2")
    t = rgb.astype(np.float32) * F(1 / 255.0)
    t = cv2.subtract(t, MEAN + (0.0,))
    return cv2.divide(t, STD + (0.0,))


def _all_bytes_image():
    return np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(16, 16, 3)


# ------------------------------------------------------------------ pre-process: values -------------------------------
def test_values_equal_cv2_chain_on_all_768_bytes():
    """For every byte in every plane, cv2 4.13's chain equals the oracle's s = (float)u * (1.f / 255.f) - (float)mean_c in
    float, then (float)((double)s / std_c), with plane 0 = R meeting mean 0.485; a float division differs."""
    got = _cv2_chain(_all_bytes_image()).reshape(256, 3)
    u = np.arange(256)
    for c in range(3):
        assert np.array_equal(got[:, c], np.array([DO.input_value(c, v) for v in u], np.float32)), c
    fdiv = np.array([(F(v) * F(1 / 255.0) - F(MEAN[0])) / F(STD[0]) for v in u], np.float32)
    assert (fdiv != got[:, 0]).any()


def test_cpp_operators_are_the_cv2_calls_of_the_chain():
    """The C++ operators of preprocessImg, as OpenCV 4.x's core/operations.hpp defines them, give the chain's bytes:
    `Mat /= double` is convertTo(-1, 1. / s), here through cv2.normalize(NORM_MINMAX, 0, 1) of a float image holding 0 and 255
    (scale 1 / 255., shift 0); `-= Scalar` is cv::subtract(a, s, a), the same bytes as t - (float)mean; `/= Scalar` is
    cv::divide(a, Mat(s), a) with Mat(s) a 4 x 1 CV_64F matrix, the same bytes as the tuple form."""
    cv2 = pytest.importorskip("cv2")
    t = _all_bytes_image().astype(np.float32)
    conv = cv2.normalize(t, None, 0, 1, cv2.NORM_MINMAX, cv2.CV_32F)
    assert np.array_equal(conv, t * F(1 / 255.0))
    sub = cv2.subtract(conv, MEAN + (0.0,))
    assert np.array_equal(sub, conv - np.array(MEAN, np.float32))
    div_mat = cv2.divide(sub, np.array(STD + (0.0,), np.float64).reshape(4, 1))
    assert np.array_equal(div_mat, cv2.divide(sub, STD + (0.0,)))
    assert np.array_equal(div_mat, (sub.astype(np.float64) / np.array(STD)).astype(np.float32))


# ------------------------------------------------------------------ pre-process: the oracle -----------------------------
PRE_SIZES = [(1920, 1080), (1280, 720), (640, 480), (1066, 800), (2132, 1600), (533, 400), (4000, 3000), (1, 1), (1, 500),
             (500, 1)]


def _pre_sizes():
    rng = np.random.default_rng(17)
    return PRE_SIZES + [tuple(int(v) for v in s) for s in rng.integers(1, 2500, (8, 2))]


@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_cv2(ipp):
    """preprocessImg in cv2 (cvtColor BGR2RGB, resize of the whole frame to 1066 x 800 INTER_LINEAR, the chain above) split
    into R, G, B planes equals the oracle bit for bit: up- and down-scaling, the identity, the exact 2x downscale (where
    OpenCV takes INTER_AREA), 1 x N, N x 1 and seeded sizes; a pitched image reads the same."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for i, (w, h) in enumerate(_pre_sizes()):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            rgb = cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), (NET_W, NET_H), interpolation=cv2.INTER_LINEAR)
            want = _cv2_chain(rgb).transpose(2, 0, 1)
            got = DO.preprocess(img)
            assert np.array_equal(got, want), (w, h, ipp)
            if i % 4 == 0:
                buf = np.zeros((h, 3 * w + 5), np.uint8)
                buf[:, :3 * w] = img.reshape(h, 3 * w)
                pitched = np.lib.stride_tricks.as_strided(buf, (h, w, 3), (3 * w + 5, 3, 1))
                assert np.array_equal(DO.preprocess(pitched), got), (w, h)
    finally:
        cv2.ipp.setUseIPP(old)


# ------------------------------------------------------------------ post-process: the per-query loop --------------------
def _loop(scores, boxes, img_w, img_h, thresh=F(0.5)):
    """detr.cpp:779-799 in Python over one frame's queries, with float32 compares, for the oracle to be pinned to."""
    Q, Cn = scores.shape
    rows = []
    for q in range(Q):
        label, score = -1, F(-1)
        for j in range(Cn):
            if score < scores[q, j]:
                label, score = j, scores[q, j]
        if score > thresh and label != Cn - 1:
            rows.append([*DO.get_rect(img_w, img_h, boxes[q]), score, label])
    out = np.zeros(1 + Q * 6, np.float32)
    out[0] = len(rows)
    if rows:
        out[1:1 + 6 * len(rows)] = np.array(rows, np.float32).ravel()
    return out


def test_oracle_postprocess_is_the_loop():
    """The oracle's post loop equals the loop restated in Python on planted objects, equal maxima (the first wins), NaN scores
    (never taken) and an all-NaN query, a score of exactly 0.5f (not kept), no-object winners, a query with every score
    below -1 (label -1, not kept) and NaN / inf boxes."""
    rng = np.random.default_rng(3)
    Q, Cn = 100, 92
    s = rng.random((Q, Cn)).astype(np.float32) ** 8
    s /= s.sum(1, keepdims=True)
    b = rng.random((Q, 4)).astype(np.float32)
    s[0, 5] = s[0, 9] = 0.7                       # equal maxima: class 5
    s[1, :3] = np.nan
    s[1, 40] = 0.9                                # NaN first, then the maximum
    s[2] = np.nan                                 # all NaN
    s[3, 7] = 0.5                                 # exactly the threshold
    s[4, Cn - 1] = 0.95                           # no-object winner
    s[5] = -2.0                                   # nothing above the start score
    s[6, 3] = 0.8
    b[6] = (np.nan, 0.5, 0.2, 0.2)
    s[7, 4] = 0.8
    b[7] = (0.5, np.inf, 0.2, 0.2)
    s[8:40:3, 11] = 0.6
    for w, h in ((1920, 1080), (640, 480), (1, 1)):
        got = DO.postprocess(s, b, w, h)
        assert np.array_equal(got, _loop(s, b, w, h), equal_nan=True), (w, h)
        labels = got[1:1 + 6 * int(got[0])].reshape(-1, 6)[:, 5]
        assert 5 in labels and 40 in labels and 91 not in labels and 7 not in labels
    low = DO.postprocess(s, b, 640, 480, F(-1.0))  # the lowest threshold accepted: label -1 still never passes
    assert np.array_equal(low, _loop(s, b, 640, 480, F(-1.0)))
    assert 0 < low[0] <= Q - 3


# ------------------------------------------------------------------ get_rect ----------------------------------------------
RECT_SIZES = [(1920, 1080), (1280, 720), (1066, 800), (640, 480), (1, 1), (3000, 17), (17, 3000), (60000, 60000)]


def _boxes(n=3000, seed=7):
    rng = np.random.default_rng(seed)
    b = np.concatenate([rng.uniform(-0.2, 1.2, (n, 2)), rng.uniform(0, 1.5, (n, 2))], 1).astype(np.float32)
    special = np.array([[np.nan, 0.5, 0.1, 0.1], [0.5, np.inf, 0.1, 0.1], [-np.inf, 0.5, 0.1, 0.1], [0.5, 0.5, np.nan, 0.1],
                        [0.5, 0.5, np.inf, np.inf], [3e5, 0.5, 0.1, 0.1], [0.5, -3e5, 0.1, 0.1], [0.5, 0.5, 5e5, 0.1],
                        [1e30, 1e30, 1e30, 1e30], [0, 0, 0, 0], [0.5, 0.5, 1, 1], [0.0001, 0.0001, 0.0004, 0.0004],
                        [-0.0001, -0.0002, 0.0001, 0.0001], [1.5, 1.5, 0.2, 0.2], [-0.5, -0.5, 0.2, 0.2],
                        [0.5, 0.5, 1e-30, 1e-30], [0.5, 0.5, -0.3, -0.3]], np.float32)
    return np.concatenate([b, special])


def test_get_rect_equals_oracle():
    """trtx_detr_get_rect equals the oracle's restatement of detr.cpp:795-803 on 3 000 random boxes and on edge boxes x
    8 frame sizes: negative corners that truncate toward 0, boxes outside the frame, NaN / +-inf and values >= 2^31 (INT_MIN,
    as x86-64 converts them)."""
    lib = L.load()
    boxes = _boxes()
    seen_min = seen_neg_zero = False
    for w, h in RECT_SIZES:
        r = (C.c_int * 4)()
        for bx in boxes:
            bb = (C.c_float * 4)(*bx.tolist())
            assert lib.trtx_detr_get_rect(w, h, bb, r) == 0
            want = DO.get_rect(w, h, bx)
            assert tuple(r) == want, (w, h, bx, tuple(r), want)
            seen_min |= INT_MIN in want
            x1 = F((float(bx[0]) - float(bx[2]) / 2.0) * w)
            seen_neg_zero |= -1 < x1 < 0 and want[0] == 0
    assert seen_min and seen_neg_zero


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_abi_and_rejected_arguments():
    lib = L.load()
    assert lib.trtx_abi_sizeof(11) == C.sizeof(L.DetrPostParams) == 12
    descs = (L.ImageDesc * 2)()
    for d in descs:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    pre = lambda d=descs, b=2, w=NET_W, h=NET_H, dst=16: lib.trtx_detr_preprocess_enqueue(d, b, w, h, dst, None)
    assert pre(d=None) == L.ERR_INVALID
    assert pre(b=0) == L.ERR_INVALID
    assert pre(w=0) == L.ERR_INVALID
    assert pre(h=-1) == L.ERR_INVALID
    assert pre(dst=None) == L.ERR_INVALID
    assert pre(dst=18) == L.ERR_INVALID  # not 4-byte aligned
    assert pre(w=4758) == L.ERR_UNSUPPORTED  # the band's staged rows exceed shared memory
    descs[1].pitch = 11  # < 3 * width
    assert pre() == L.ERR_INVALID
    descs[1].pitch, descs[1].data_dev = 12, None
    assert pre() == L.ERR_INVALID
    descs[1].data_dev, descs[1].height = 16, 0
    assert pre() == L.ERR_INVALID
    assert lib.trtx_detr_get_rect(0, 10, (C.c_float * 4)(), (C.c_int * 4)()) == L.ERR_INVALID
    assert lib.trtx_detr_get_rect(10, 10, None, (C.c_int * 4)()) == L.ERR_INVALID

    q = L.DetrPostParams(100, 92, 0.5)
    wh = (C.c_int32 * 4)(1920, 1080, 1280, 720)
    post = lambda p=C.byref(q), f=wh, b=2, s=16, x=16, r=16: lib.trtx_detr_postprocess_enqueue(p, f, b, s, x, r, None)
    assert post(p=None) == L.ERR_INVALID
    assert post(f=None) == L.ERR_INVALID
    assert post(b=0) == L.ERR_INVALID
    assert post(s=None) == L.ERR_INVALID
    assert post(x=None) == L.ERR_INVALID
    assert post(r=None) == L.ERR_INVALID
    for field, bad in (("num_queries", 0), ("num_classes", 1), ("score_thresh", float("nan")), ("score_thresh", -1.0001)):
        q2 = L.DetrPostParams(100, 92, 0.5)
        setattr(q2, field, bad)
        assert post(p=C.byref(q2)) == L.ERR_INVALID, (field, bad)
    wh[3] = 0
    assert post() == L.ERR_INVALID
    wh[3] = 720
    for field, big in (("num_queries", (1 << 24) + 1), ("num_classes", (1 << 24) + 1)):
        q2 = L.DetrPostParams(100, 92, 0.5)
        setattr(q2, field, big)
        assert post(p=C.byref(q2)) == L.ERR_UNSUPPORTED, field
