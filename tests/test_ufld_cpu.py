"""UFLD on the CPU: the oracle (oracle/ufld_oracle.c) against cv2 4.13 -- prepareImage's cvtColor / resize / convertTo and the
`(c - mean) / std` MatExpr -- against the driver's own argmax and softmax_mul (oracle/_ref/libref_ufld_host.so, or
tests/golden/ref_ufld_host.npz where it was not built), against the driver loop of lane_det.cpp:358-410 restated in Python,
the exp the device uses against glibc's expf, and the argument checks of the UFLD calls that reject before any launch."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from oracle import ufld as UO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

F = np.float32
MEAN, STD = (F(0.485), F(0.456), F(0.406)), (F(0.229), F(0.224), F(0.225))  # the driver's `static float`, R, G, B
NET_W, NET_H = UO.NET_W, UO.NET_H
G = RefOutputs("ref_ufld_host")


def _coeffs(c):
    """MatOp_AddEx's convertTo coefficients of `(ch - mean[c]) / std[c]`: alpha = 1 / std, beta = -mean / std in double."""
    return 1.0 / float(STD[c]), -float(MEAN[c]) / float(STD[c])


def _round_f32(x: Fraction) -> np.float32:
    """x rounded once to the nearest float32, ties to even."""
    f = F(float(x))
    cands = [np.nextafter(f, F(-np.inf)), f, np.nextafter(f, F(np.inf))]
    best = min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.array(v).view(np.uint32)) & 1))
    return F(best)


def _fma_f32(s, a, b) -> np.float32:
    return _round_f32(Fraction(float(s)) * Fraction(float(a)) + Fraction(float(b)))


def _s_values():
    return np.arange(256).astype(np.float32) * F(1.0 / 255.0)  # convertTo(CV_32FC3, 1. / 255.): (float)u * (float)(1. / 255.)


# ------------------------------------------------------------------ pre-process: values -------------------------------
def test_values_equal_cv2_convert_on_all_768_bytes():
    """For every byte in every plane the oracle's fmaf(s, (float)(1 / std), (float)(-mean / std)) equals cv2 4.13's
    convertTo kernel, reached through normalize(NORM_MINMAX) with the same alpha and beta (s holds both 0 and 1), and a
    restatement with one exact rounding.  The unfused form, subtract-then-divide in float and the chain in double miss
    most values, so the fused form is what the driver computes on an FMA build of OpenCV."""
    cv2 = pytest.importorskip("cv2")
    s = _s_values()
    for c in range(3):
        a, b = _coeffs(c)
        got = np.array([UO.input_value(c, u) for u in range(256)], np.float32)
        cv = cv2.normalize(s.reshape(16, 16), None, alpha=b, beta=b + a, norm_type=cv2.NORM_MINMAX, dtype=cv2.CV_32F).ravel()
        assert np.array_equal(got, cv), c
        assert np.array_equal(got, np.array([_fma_f32(v, F(a), F(b)) for v in s], np.float32)), c
        unfused = s * F(a) + F(b)
        sub_div = (s - MEAN[c]) / STD[c]
        dbl = ((s.astype(np.float64) - float(MEAN[c])) / float(STD[c])).astype(np.float32)
        for other in (unfused, sub_div, dbl):
            assert (other != got).sum() > 100, c


def _bytes_lut():
    return np.array([[UO.input_value(c, u) for u in range(256)] for c in range(3)], np.float32)


PRE_SIZES = [(1920, 1080), (1280, 720), (800, 288), (1600, 576), (400, 144), (640, 480), (3840, 2160), (1, 1), (1, 300),
             (300, 1), (17, 4000), (4000, 17)]


def _pre_sizes():
    rng = np.random.default_rng(23)
    return PRE_SIZES + [tuple(int(v) for v in s) for s in rng.integers(1, 2500, (8, 2))]


@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_cv2(ipp):
    """prepareImage's resize in cv2 (cvtColor BGR2RGB, then resize of the whole frame to 800 x 288, INTER_LINEAR) through
    the value table above, split into R, G, B planes, equals the oracle bit for bit: up- and downscales, the identity, the
    exact 2x downscale (where OpenCV takes INTER_AREA), 1 x 1, 1 x N, N x 1, tall, wide and seeded sizes; a pitched image
    reads the same."""
    cv2 = pytest.importorskip("cv2")
    lut = _bytes_lut()
    rng = np.random.default_rng(31 + ipp)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        for i, (w, h) in enumerate(_pre_sizes()):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            rgb = cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), (NET_W, NET_H), interpolation=cv2.INTER_LINEAR)
            want = np.stack([lut[c][rgb[:, :, c]] for c in range(3)])
            got = UO.preprocess(img)
            assert np.array_equal(got, want), (w, h, ipp)
            if i % 4 == 0:
                buf = np.zeros((h, 3 * w + 5), np.uint8)
                buf[:, :3 * w] = img.reshape(h, 3 * w)
                pitched = np.lib.stride_tricks.as_strided(buf, (h, w, 3), (3 * w + 5, 3, 1))
                assert np.array_equal(UO.preprocess(pitched), got), (w, h)
    finally:
        cv2.ipp.setUseIPP(old)


# ------------------------------------------------------------------ the driver's argmax and softmax_mul ----------------
def test_argmax_and_softmax_mul_equal_the_drivers():
    """The oracle's argmax and softmax_mul equal the driver's own functions, compiled where they lie with -ffp-contract=off
    (or their stored outputs), on the edge cells of oracle.ufld.edge_cells, on CULane's shape and on random logits."""
    ref = G.lib("libref_ufld_host.so")
    cases = {"edge": UO.edge_cells(), "culane": UO.edge_cells(201, seed=6),
             "random": np.random.default_rng(9).normal(0, 4, (101, 56, 4)).astype(np.float32)}
    for name, p in cases.items():
        Cn, H, W = p.shape
        got_a, got_s = UO.argmax(p), UO.softmax_mul(p)
        live_a = live_s = None
        if ref is not None:
            live_a, live_s = np.empty((H, W), np.float32), np.empty((H, W), np.float32)
            x = p.copy()
            ref.ref_ufld_argmax(C.c_void_p(x.ctypes.data), C.c_void_p(live_a.ctypes.data), H, W, Cn)
            x = p.copy()
            ref.ref_ufld_softmax_mul(C.c_void_p(x.ctypes.data), C.c_void_p(live_s.ctypes.data), H, W, Cn)
        G.equal(f"argmax_{name}", got_a, live_a, nan_ok=True)
        G.equal(f"softmax_mul_{name}", got_s, live_s, nan_ok=True)
    a, s = UO.argmax(cases["edge"]), UO.softmax_mul(cases["edge"])
    assert a[0, 0] == 0 and a[0, 1] == 3 and a[0, 2] == 7 and a[0, 3] == -1 and a[1, 0] == -1  # first / tie / quirk / -1
    assert a[1, 1] == 100 and a[3, 0] == 100 and a[3, 1] == 0 and a[2, 3] == 100            # after +inf / 3e9; 2^31 - 128
    assert np.isnan(s[1, 0]) and np.isnan(s[2, 0]) and np.isnan(s[2, 1]) and s[2, 2] > 0       # NaN, inf / inf, 0 / 0


def test_driver_exp_is_the_double_exp():
    """The driver's unqualified exp(float), compiled against the shim's includes, resolves to the C library's double exp,
    which (float)exp((double)x) restates; and on a sample of every 1024th float in [-104, 89], glibc's expf differs from it
    in a small fraction of the values (DESIGN §4.8 records the full count)."""
    ref = G.lib("libref_ufld_host.so")
    if ref is not None:
        assert ref.ref_ufld_exp_is_float() == 0
    n = UO.exp_disagreements(-104.0, 89.0, 1024)
    total = (int(np.float32(104).view(np.uint32)) + int(np.float32(89).view(np.uint32))) // 1024
    assert 0 < n < total * 1e-3, (n, total)


# ------------------------------------------------------------------ the driver loop ------------------------------------
def _loop(prob, vis_w, vis_h, anchors, net_w=NET_W, net_h=NET_H, col_sample_w=8):
    """lane_det.cpp:358-410 in Python over one frame, float32 arithmetic, for the oracle to be pinned to."""
    Cn, H, W = prob.shape
    rev = prob[:, ::-1, :]
    max_ind = UO.argmax(rev)
    expect = UO.softmax_mul(rev)
    expect[max_ind == F(Cn - 1)] = 0
    lanes = [k for k in range(W) if sum(1 for g in range(H) if expect[g, k] != 0) > 2]
    rows = []
    for k in range(H):
        for ll in lanes:
            e = expect[k, ll]
            if e > 0:
                fx = F(F(F(e * F(col_sample_w)) * F(vis_w)) / F(net_w))
                x = int(fx) if -2.0 ** 31 <= fx < 2.0 ** 31 else -2 ** 31
                x = (x - 1 + 2 ** 31) % 2 ** 32 - 2 ** 31
                prod = vis_h * int(anchors[H - 1 - k])
                y = (abs(prod) // net_h if prod >= 0 else -(abs(prod) // net_h)) - 1  # C's truncating division
                rows.append((x, y, ll))
    out = np.zeros(1 + H * W * 3, np.float32)
    out[0] = len(rows)
    if rows:
        out[1:1 + 3 * len(rows)] = np.array(rows, np.float32).ravel()
    return out


@pytest.mark.parametrize("shape", [(101, 56, 4), (201, 18, 4)])
def test_oracle_postprocess_is_the_loop(shape):
    """The oracle's loop equals the loop restated in Python: lanes with many, 3, 2 and no non-zero rows, a NaN expectation,
    the edge cells, the 1280 x 720 `vis` and other picture sizes; TuSimple's shape and CULane's C = 201, H = 18."""
    Cn, H, W = shape
    anchors = np.array(UO.TUSIMPLE_ROW_ANCHOR if H == 56 else np.linspace(121, 287, H).astype(int), np.int32)
    rest = np.random.default_rng(1).normal(0, 2, (Cn, H - 16, W)).astype(np.float32)
    for p in (UO.lane_prob(Cn, H, W), np.concatenate([UO.edge_cells(Cn), rest], 1)):
        for vw, vh in ((1280, 720), (1920, 1080), (640, 480), (1, 1), (100000, 70000)):
            got = UO.postprocess(p, vw, vh, anchors)
            assert np.array_equal(got, _loop(p, vw, vh, anchors)), (shape, vw, vh)
    got = UO.postprocess(UO.lane_prob(Cn, H, W), 1280, 720, anchors)
    lanes = set(got[1:1 + 3 * int(got[0])].reshape(-1, 3)[:, 2].tolist())
    assert lanes == {0.0, 1.0}, lanes


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_abi_and_rejected_arguments():
    lib = L.load()
    assert lib.trtx_abi_sizeof(13) == C.sizeof(L.UfldPostParams) == 24
    descs = (L.ImageDesc * 2)()
    for d in descs:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    pre = lambda d=descs, b=2, w=NET_W, h=NET_H, dst=16: lib.trtx_ufld_preprocess_enqueue(d, b, w, h, dst, None)
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
    descs[1].height, descs[1].width = 4, -1
    assert pre() == L.ERR_INVALID

    mk = lambda **kw: L.UfldPostParams(*[kw.get(n, v) for n, v in (("num_cells", 101), ("num_rows", 56), ("num_lanes", 4),
                                                                   ("net_w", 800), ("net_h", 288), ("col_sample_w", 8))])
    q = mk()
    anchors = (C.c_int32 * 56)(*UO.TUSIMPLE_ROW_ANCHOR)
    wh = (C.c_int32 * 4)(1280, 720, 1920, 1080)
    post = lambda p=C.byref(q), a=anchors, f=wh, b=2, x=16, r=16: lib.trtx_ufld_postprocess_enqueue(p, a, f, b, x, r, None)
    assert post(p=None) == L.ERR_INVALID
    assert post(a=None) == L.ERR_INVALID
    assert post(f=None) == L.ERR_INVALID
    assert post(b=0) == L.ERR_INVALID
    assert post(b=-3) == L.ERR_INVALID
    assert post(x=None) == L.ERR_INVALID
    assert post(r=None) == L.ERR_INVALID
    for field, bad in (("num_cells", 1), ("num_rows", 0), ("num_lanes", -1), ("net_w", 0), ("net_h", -288),
                       ("col_sample_w", 0)):
        assert post(p=C.byref(mk(**{field: bad}))) == L.ERR_INVALID, (field, bad)
    for k in (0, 3):
        old, wh[k] = wh[k], 0
        assert post() == L.ERR_INVALID, k
        wh[k] = old
    # one CTA per frame: H * W threads, (C - 1) * H * W exponentials in shared memory
    assert post(p=C.byref(mk(num_rows=56, num_lanes=19))) == L.ERR_UNSUPPORTED  # H * W = 1064
    assert post(p=C.byref(mk(num_cells=239, num_rows=56, num_lanes=4))) == L.ERR_UNSUPPORTED  # 238 * 224 > 53 248
    # frames: a side above 2^24; h * anchor overflowing int32; |y| above 2^24
    for w, h in (((1 << 24) + 1, 720), (1280, (1 << 24) + 1), (1280, 8_000_000), (1280, 1 << 24)):
        wh[2], wh[3] = w, h
        assert post() == L.ERR_UNSUPPORTED, (w, h)
    wh[2], wh[3] = 1920, 1080
    big = (C.c_int32 * 56)(*UO.TUSIMPLE_ROW_ANCHOR)
    big[10] = 3_000_000  # 1080 * 3e6 overflows int32
    assert post(a=big) == L.ERR_UNSUPPORTED
    big[10] = 1_800_000  # 1080 * 1.8e6 fits, but 1080 * 1.8e6 / 100 - 1 > 2^24
    assert post(p=C.byref(mk(net_h=100)), a=big) == L.ERR_UNSUPPORTED
