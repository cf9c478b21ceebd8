"""RefineDet on the CPU: the oracle (oracle/refinedet_oracle.c) against cv2 4.13 -- base_transform's resize and planes --
and against the line-by-line transcription of the reference's libtorch post-process (oracle/refinedet.py) run in torch on
the CPU; the prior table; the driver's rectangles and RoiCorrect; and every argument the library rejects."""

import ctypes as C

import numpy as np
import pytest

from oracle import refinedet as RO
from tensorrtx_b200 import _lib as L

NET = RO.NET
ACCEPTED_NETS = range(64, 1025, 64)  # S multiple of 64 with P <= 2^16
SQRT_SENSITIVE = {192, 384, 448, 704, 768, 832, 896, 960}  # sides where sqrt(2.0) and sqrtf(2.f) give different priors


# ------------------------------------------------------------------ base_transform ---------------------------------------
def test_values_are_exact():
    for c, mean in enumerate((123, 117, 104)):
        for u in range(256):
            assert RO.input_value(c, u) == np.float32(u - mean)


PRE_SIZES = [(1920, 1080), (1280, 720), (320, 320), (640, 640), (160, 160), (640, 480), (3840, 2160), (1, 1), (1, 300),
             (300, 1), (17, 4000), (4000, 17)]


@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_cv2(ipp):
    """cv::resize of the whole frame to 320 x 320 (INTER_LINEAR) in cv2, then R - 123, G - 117, B - 104, equals the oracle
    bit for bit: up- and downscales, the identity, the exact 2x downscale (where OpenCV takes INTER_AREA), 1 x 1, 1 x N,
    N x 1 and seeded sizes; a pitched image reads the same."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(41 + ipp)
    sizes = PRE_SIZES + [tuple(int(v) for v in s) for s in rng.integers(1, 2500, (8, 2))]
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for i, (w, h) in enumerate(sizes):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            re = cv2.resize(img, (NET, NET), interpolation=cv2.INTER_LINEAR).astype(np.float64)
            want = np.stack([re[:, :, 2] - 123.0, re[:, :, 1] - 117.0, re[:, :, 0] - 104.0]).astype(np.float32)
            got = RO.preprocess(img)
            assert np.array_equal(got, want), (w, h, ipp)
            if i % 4 == 0:
                buf = np.zeros((h, 3 * w + 5), np.uint8)
                buf[:, :3 * w] = img.reshape(h, 3 * w)
                pitched = np.lib.stride_tricks.as_strided(buf, (h, w, 3), (3 * w + 5, 3, 1))
                assert np.array_equal(RO.preprocess(pitched), got), (w, h)
    finally:
        cv2.ipp.setUseIPP(old)


# ------------------------------------------------------------------ priors -----------------------------------------------
@pytest.mark.parametrize("net", ACCEPTED_NETS)
def test_prior_table(net):
    """The oracle's table equals PriorBox restated in Python (float statements, torch clamp) bit for bit.  The library takes
    sqrt(ar)'s float overload; the double overload gives the same table at S = 320 and at every accepted side but the
    listed ones, where some anchors differ in their last bit."""
    p = RO.priors(net)
    assert p.shape == (RO.num_priors(net), 4)
    assert np.array_equal(p, RO.prior_box(net).numpy())
    assert np.array_equal(p, RO.priors(net, double_sqrt=True)) == (net not in SQRT_SENSITIVE)
    assert (p >= 0).all() and (p <= 1).all()


def test_prior_table_at_320():
    p = RO.priors(NET)
    assert p.shape == (6375, 4)
    assert p[0].tolist() == [float(np.float32(0.5 / np.float32(40.0)))] * 2 + [float(np.float32(0.1))] * 2
    # level offsets 4800, 6000, 6300: the first prior of each level sits at its first cell
    for off, f in ((4800, 20), (6000, 10), (6300, 5)):
        assert p[off, 0] == float(np.float32(0.5 / np.float32(f)))


# ------------------------------------------------------------------ the post-process vs the transcription ----------------
def _compare(h, b, **kw):
    want = RO.reference_postprocess(*[x[b] for x in h], **kw)
    got = RO.postprocess(*[x[b] for x in h], **kw)
    n = int(got[0])
    assert n == len(want)
    g = got[1:1 + 6 * n].reshape(-1, 6)
    assert np.array_equal(g[:, 4:], want[:, 4:])  # the same kept set, in the same order
    # the boxes: glibc's exp here, torch's CPU exp there; a few ulps at most
    ulps = np.abs(g[:, :4].view(np.int32).astype(np.int64) - want[:, :4].view(np.int32).astype(np.int64))
    finite = np.isfinite(want[:, :4])
    assert np.array_equal(np.isnan(g[:, :4]), np.isnan(want[:, :4]))
    assert (ulps[finite] <= 4).all()
    return n


@pytest.mark.parametrize("seed,dense", [(0, 0), (1, 0), (2, 2500)])
def test_oracle_equals_transcription(seed, dense):
    """Seeded tie-free heads with planted objects, and classes with more than top_k candidates."""
    h = RO.heads(1, seed=seed, objects=40, dense=dense)
    assert _compare(h, 0) > 500


def test_oracle_equals_transcription_on_nan_and_inf():
    """NaN and +-inf in every head at candidates of three classes, including each class's highest score."""
    h = [x.copy() for x in RO.heads(1, seed=7, objects=30)]
    rng = np.random.default_rng(3)
    for c in (1, 7, 24):
        cand = np.flatnonzero(h[3][0, :, c] > 0.3)
        top = cand[np.argmax(h[3][0, cand, c])]
        h[0][0, top, 2] = np.inf
        ps = rng.choice(cand[cand != top], 8, replace=False)
        h[0][0, ps[0], 0] = np.nan
        h[2][0, ps[1], 3] = -np.inf
        h[2][0, ps[2], 1] = np.nan
        h[1][0, ps[3], 1] = np.nan
        h[1][0, ps[4], 1] = np.inf
        h[3][0, ps[5], c] = np.nan
        h[3][0, ps[6], c] = -np.inf
        h[2][0, ps[7], 2] = 300.0
    _compare(h, 0)


def test_oracle_keeps_the_tie_rule():
    """Equal scores: the lower prior index ranks first, and the top_k cut keeps the lowest indices of a tie."""
    P = RO.num_priors()
    z = np.zeros((P, 4), np.float32)
    arm = np.full((P, 2), 0.5, np.float32)
    conf = np.zeros((P, RO.NUM_CLASSES), np.float32)
    far = [0, 1500, 3000, 4500, 6000]  # non-overlapping priors
    conf[far, 3] = 0.5
    d = RO.postprocess(z, arm, z, conf, top_k=3, max_det=10)
    assert d[0] == 3
    got = d[1:1 + 18].reshape(3, 6)
    boxes = RO.priors()[far[:3]]
    want = np.concatenate([boxes[:, :2] - boxes[:, 2:] / 2, boxes[:, :2] - boxes[:, 2:] / 2 + boxes[:, 2:]], 1)
    assert np.array_equal(got[:, :4], want.astype(np.float32))


# ------------------------------------------------------------------ rectangles ------------------------------------------
def _rect_rows(rows_, cols, rws, th=0.2):
    dets = np.zeros(1 + 6 * len(rows_), np.float32)
    dets[0] = len(rows_)
    dets[1:] = np.asarray(rows_, np.float32).ravel()
    r = RO.rows(dets, cols, rws, th)
    return [tuple(int(v) for v in r[1 + 6 * i:5 + 6 * i]) for i in range(int(r[0]))]


def test_rectangles_and_roi_correct():
    """The driver's float products and conversions and every branch of RoiCorrect."""
    W, H = 640, 480
    cases = [
        ((0.1, 0.2, 0.5, 0.6), (64, 96, 256, 192)),          # plain: (int)(0.1f * 640) = 64, w = (int)(320 - 64)
        ((-0.2, -0.1, 0.3, 0.4), (0, 0, 320, 240)),          # x = -128, w = (int)(192.00001f + 128); then x -> 0
        ((0.999, 0.999, 1.5, 1.5), (0, 0, 321, 241)),        # x = 639 >= cols - 1 resets to 0 and keeps w = 960 - 639
        ((0.5, 0.5, 0.4, 0.4), (320, 240, 1, 1)),            # w <= 0 becomes 1
        ((0.9, 0.9, 2.0, 2.0), (576, 432, 63, 47)),          # x + w > cols - 1: w = cols - 1 - x
        ((np.nan, 0.5, 0.6, np.inf), (0, 240, 1, 1)),        # NaN and inf convert to INT_MIN, so do x2 * cols - INT_MIN
        ((0.25, 0.25, 3.4e6, 0.5), (160, 120, 1, 120)),      # a width beyond the int range: INT_MIN, then 1
        ((0.0, 0.0, 3.3e6, 1.0), (0, 0, 639, 479)),          # a width just inside it, cut at the edge
    ]
    for (box, want) in cases:
        got = _rect_rows([(*box, 0.5, 1.0)], W, H)
        assert got == [want], (box, got, want)
    # on a 200000-wide frame x + w passes INT_MAX and wraps below cols - 1 as on x86-64, so w is not cut
    x2 = np.float32(10737.418)  # x2 * 200000 rounds to 2^31: x = 100000, w = (int)(2^31 - 100000 in float) = 2147383680
    assert _rect_rows([(0.5, 0.1, x2, 0.5, 0.5, 1.0)], 200000, 100) == [(100000, 10, 2147383680, 40)]
    # the score filter: `score < TH` drops, equality keeps
    assert len(_rect_rows([(0.1, 0.1, 0.2, 0.2, np.float32(0.2), 1.0), (0.1, 0.1, 0.2, 0.2, 0.19999, 1.0)], W, H)) == 1
    # 1 x 1 and 2 x 2 frames: on 1 x 1, w = 0 - x leaves an empty rectangle
    assert _rect_rows([(0.1, 0.2, 0.5, 0.6, 0.5, 1.0)], 1, 1) == [(0, 0, 0, 0)]
    assert _rect_rows([(0.1, 0.2, 0.5, 0.6, 0.5, 1.0)], 2, 2) == [(0, 0, 1, 1)]


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_abi_and_rejected_arguments():
    lib = L.load()
    assert lib.trtx_abi_sizeof(14) == C.sizeof(L.RefinedetParams) == 32
    descs = (L.ImageDesc * 2)()
    for d in descs:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    pre = lambda d=descs, b=2, n=NET, dst=16: lib.trtx_refinedet_preprocess_enqueue(d, b, n, dst, None)  # noqa: E731
    assert pre(d=None) == L.ERR_INVALID
    assert pre(b=0) == L.ERR_INVALID
    assert pre(n=0) == L.ERR_INVALID
    assert pre(dst=None) == L.ERR_INVALID
    assert pre(dst=18) == L.ERR_INVALID  # not 4-byte aligned
    assert pre(n=4758) == L.ERR_UNSUPPORTED  # the band's staged rows exceed shared memory
    descs[1].pitch = 11  # < 3 * width
    assert pre() == L.ERR_INVALID
    descs[1].pitch, descs[1].data_dev = 12, None
    assert pre() == L.ERR_INVALID
    descs[1].data_dev, descs[1].height = 16, 0
    assert pre() == L.ERR_INVALID

    fields = (("net", 320), ("num_classes", 25), ("obj_thresh", 0.01), ("conf_thresh", 0.01), ("nms_thresh", 0.45),
              ("top_k", 1000), ("max_det", 24000), ("score_thresh", 0.2))
    mk = lambda **kw: L.RefinedetParams(*[kw.get(n, v) for n, v in fields])  # noqa: E731
    q = mk()
    ws = lib.trtx_refinedet_workspace_size(C.byref(q), 2)
    assert ws == 256 + 2 * 24 * 1000 * 2 + (-(2 * 24 * 1000 * 2) % 256)
    wh = (C.c_int32 * 4)(1280, 720, 1920, 1080)
    post = lambda p=C.byref(q), b=2, x=16, w=256, nb=ws, d=16, f=wh, r=16: lib.trtx_refinedet_postprocess_enqueue(  # noqa
        p, b, x, x, x, x, w, nb, d, f, r, None)
    assert post(p=None) == L.ERR_INVALID
    assert post(b=0) == L.ERR_INVALID
    assert post(x=None) == L.ERR_INVALID
    assert post(d=None) == L.ERR_INVALID
    assert post(w=None) == L.ERR_INVALID
    assert post(f=None) == L.ERR_INVALID  # rows without frames
    assert post(r=None) == L.ERR_INVALID  # frames without rows
    assert post(nb=ws - 1) == L.ERR_WORKSPACE
    assert post(w=128) == L.ERR_INVALID  # not 256-byte aligned
    for field, bad in (("net", 0), ("net", -64), ("num_classes", 1), ("top_k", 0), ("max_det", 0),
                       ("obj_thresh", float("nan")), ("conf_thresh", float("nan")), ("nms_thresh", float("nan")),
                       ("score_thresh", float("nan"))):
        assert post(p=C.byref(mk(**{field: bad}))) == L.ERR_INVALID, (field, bad)
        assert lib.trtx_refinedet_workspace_size(C.byref(mk(**{field: bad})), 2) == 0
    for field, bad in (("net", 300), ("net", 1088), ("top_k", 1025), ("num_classes", 1025), ("max_det", (1 << 24) + 1)):
        assert post(p=C.byref(mk(**{field: bad}))) == L.ERR_UNSUPPORTED, (field, bad)
    assert lib.trtx_refinedet_workspace_size(C.byref(mk(net=1024)), 2) > 0  # P = 65280
    for k, v in ((0, 0), (3, -1)):
        old, wh[k] = wh[k], v
        assert post() == L.ERR_INVALID, k
        wh[k] = old
    wh[2] = (1 << 24) + 1
    assert post() == L.ERR_UNSUPPORTED
