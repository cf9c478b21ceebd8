"""CenterNet on the CPU: the oracle (oracle/centernet_oracle.c) against the sample's own pre_process and ctdet_decode
(oracle/_ref/ref_centernet.pyc where it was built, tests/golden/ref_centernet_host.npz elsewhere) and against cv2 4.13, the
decode's order on ties, NaN, empty and saturated maps against its definition, the rows against the driver loop run in
torch, and the argument checks of the CenterNet calls that reject before any launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import centernet as CO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

GOLD = RefOutputs("ref_centernet_host")

# landscape and square frames (the sample's pre_process runs on these): L < 512, 512, 1024, 1920, odd sizes, 1 x 1
PRE_SIZES = [(1, 1), (3, 3), (7, 5), (100, 60), (255, 255), (301, 300), (511, 400), (512, 512), (513, 200), (640, 480),
             (700, 699), (1023, 767), (1024, 768), (1024, 1024), (1280, 720), (1333, 1000), (1536, 1000), (1920, 1080),
             (2001, 1999), (3000, 3000), (1, 5)]  # (w, h); the last one is 5 x 1, one pixel wide


def _frame(rng, w, h):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _sample_pre(img):
    ref = CO.reference()
    return None if ref is None else ref.pre_process(img)[0]


@pytest.mark.parametrize("ipp", [True, False])
def test_preprocess_oracle_equals_sample(ipp):
    """The oracle equals the sample's pre_process (float64 canvas, cv.resize, normalisation, transpose) bit for bit on 21
    landscape and square frames (the identity at 512, up- and downscales, odd sizes, 1 x 1) and a 5 x 1 frame that numpy
    broadcasts over its rows; a pitched frame reads the same."""
    cv2 = pytest.importorskip("cv2")
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        rng = np.random.default_rng(5)
        for w, h in PRE_SIZES:
            img = _frame(rng, w, h)
            got = CO.preprocess(img)
            GOLD.equal(f"pre_{w}x{h}", got, _sample_pre(img), msg=(w, h, ipp))
            pitched = np.zeros((h, w + 3, 3), np.uint8)[:, 1:w + 1]
            pitched[...] = img
            assert np.array_equal(CO.preprocess(pitched), got)
    finally:
        cv2.ipp.setUseIPP(old)


def test_preprocess_all_256_bytes():
    """At 512 x 512 the resize is the identity, so every byte u reads (float)(((u / 255.) - 0.5) / 0.5) in its own plane."""
    u = np.arange(512 * 512 * 3, dtype=np.int64) % 256
    img = u.reshape(512, 512, 3).astype(np.uint8)
    want = ((img.astype(np.float64) / 255. - 0.5) / 0.5).astype(np.float32).transpose(2, 0, 1)
    got = CO.preprocess(img)
    assert np.array_equal(got, want)
    GOLD.equal("pre_bytes", got, _sample_pre(img))


@pytest.mark.parametrize("w,h", [(2, 2), (2, 1), (300, 400), (480, 640), (720, 1280), (999, 1000), (5, 700)])
def test_preprocess_frames_the_sample_rejects(w, h):
    """For 1 < w < L the sample's `img[:h, :L] = image` raises; the library defines the canvas as the frame at the top-left
    and zeros elsewhere.  The oracle equals cv2.resize of that canvas, built explicitly, then the normalisation."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(w * 7 + h)
    img = _frame(rng, w, h)
    ref = CO.reference()
    if ref is not None:
        with pytest.raises(ValueError):
            ref.pre_process(img)
    L_ = max(h, w, 3)
    canvas = np.zeros((L_, L_, 3))
    canvas[:h, :w] = img
    want = ((cv2.resize(canvas, (512, 512)) / 255. - 0.5) / 0.5).astype(np.float32).transpose(2, 0, 1)
    assert np.array_equal(CO.preprocess(img), want)


# ------------------------------------------------------------------ decode ---------------------------------------------
def tie_free_heads(seed, B, Cn, H, W):
    """Logits whose sigmoids are all distinct within an image: a shuffled grid over [-15, 3] per image, where neighbouring
    logits are many float ulps apart after the sigmoid, so the reference's topk order is fully determined.  wh in [0, 60), reg in [0, 1)."""
    rng = np.random.default_rng(seed)
    grid = np.linspace(-15.0, 3.0, Cn * H * W)
    heat = np.stack([rng.permutation(grid) for _ in range(B)]).astype(np.float32).reshape(B, Cn, H, W)
    wh = rng.uniform(0, 60, (B, 2, H, W)).astype(np.float32)
    reg = rng.uniform(0, 1, (B, 2, H, W)).astype(np.float32)
    return heat, wh, reg


def _sample_decode(heat, wh, reg, k):
    ref = CO.reference()
    if ref is None:
        return None
    return ref.ctdet_decode(torch.from_numpy(heat), torch.from_numpy(wh), torch.from_numpy(reg), K=k).numpy()


def assert_dets(got, want, msg=""):
    """classes, cells and boxes exact; scores within rtol 2e-6 (torch's sigmoid and expf may differ by a few ulps)"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, msg
    keep = [0, 1, 2, 3, 5]
    assert np.array_equal(got[..., keep], want[..., keep], equal_nan=True), msg
    np.testing.assert_allclose(got[..., 4], want[..., 4], rtol=2e-6, atol=0, equal_nan=True, err_msg=str(msg))


DECODE_SHAPES = [(80, 128, 128, 100), (3, 16, 20, 1), (2, 8, 8, 64), (5, 33, 17, 40), (1, 7, 300, 50), (12, 64, 48, 200)]


@pytest.mark.parametrize("shape", DECODE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_decode_oracle_equals_sample(shape):
    """On tie-free logits the oracle equals the sample's ctdet_decode: classes, cells and boxes exactly, scores within
    rtol 2e-6; K = 1 and K = H * W included.  Where K reaches past the peaks (K = H * W), the zero-valued rest ties and
    torch's order among ties is its own: those rows are checked against the definition instead."""
    Cn, H, W, k = shape
    heat, wh, reg = tie_free_heads(sum(shape), 1, Cn, H, W)
    got = CO.decode(heat[0], wh[0], reg[0], k)
    assert_dets(got, definition_decode(heat[0], wh[0], reg[0], k), shape)
    npos = int((got[:, 4] > 0).sum())
    key = "dec_" + "x".join(map(str, shape))
    ref = _sample_decode(heat, wh, reg, k)
    if ref is not None:
        assert_dets(got[:npos], ref[0][:npos], shape)
        assert (ref[0][npos:, 4] == 0).all()
    GOLD.close(key, got[:npos, 4], None if ref is None else ref[0][:npos, 4], rtol=2e-6)
    GOLD.equal(key + "_boxes", got[:npos, [0, 1, 2, 3, 5]], None if ref is None else ref[0][:npos, [0, 1, 2, 3, 5]])


def definition_decode(heat, wh, reg, k):
    """The decode as the library defines it, in numpy: sigmoid, the 3 x 3 peak test (NaN-propagating max), the k best
    suppressed values NaN first, then descending, ties to the smaller flat index."""
    Cn, H, W = heat.shape
    with np.errstate(over="ignore", invalid="ignore"):
        s = (np.float32(1) / (np.float32(1) + np.exp(-heat.astype(np.float32)))).astype(np.float32)
    p = np.full((Cn, H + 2, W + 2), -np.inf, np.float32)
    p[:, 1:-1, 1:-1] = s
    m = np.full_like(s, -np.inf)
    for dy in range(3):
        for dx in range(3):
            win = p[:, dy:dy + H, dx:dx + W]
            m = np.where(np.isnan(m) | np.isnan(win), np.nan, np.maximum(m, win))
    with np.errstate(invalid="ignore"):
        v = (s * (m == s).astype(np.float32)).reshape(-1)
    flat = np.arange(v.size)
    order = np.lexsort((flat, -np.nan_to_num(v, nan=0.0), ~np.isnan(v)))[:k]
    cell = order % (H * W)
    ys, xs = cell // W, cell % W
    x = xs.astype(np.float32) + reg[0].reshape(-1)[cell]
    y = ys.astype(np.float32) + reg[1].reshape(-1)[cell]
    hw, hh = wh[0].reshape(-1)[cell] / np.float32(2), wh[1].reshape(-1)[cell] / np.float32(2)
    return np.stack([x - hw, y - hh, x + hw, y + hh, v[order], (order // (H * W)).astype(np.float32)], 1)


def special_heads(case, seed=0, Cn=4, H=12, W=10):
    """Logits for the order's edge cases: ties, all -inf (every value 0), NaN cells, saturated plateaus."""
    rng = np.random.default_rng(seed)
    heat = rng.uniform(-6, 6, (Cn, H, W)).astype(np.float32)
    if case == "ties":
        heat = rng.integers(-3, 3, (Cn, H, W)).astype(np.float32)
    elif case == "empty":
        heat[...] = -np.inf
    elif case == "nan":
        heat.reshape(-1)[rng.choice(heat.size, 9, replace=False)] = np.nan
    elif case == "plateau":
        heat[1, 2:7, 3:9] = 20.0
        heat[3] = rng.uniform(17, 40, (H, W))
    elif case == "sparse":  # fewer than K positive cells: the rest are zero cells in flat order
        heat[...] = -np.inf
        heat[2, 5, 5], heat[0, 1, 1], heat[3, 11, 9] = 1.0, 2.0, -1.0
    wh = rng.uniform(0, 30, (2, H, W)).astype(np.float32)
    reg = rng.uniform(0, 1, (2, H, W)).astype(np.float32)
    return heat, wh, reg


SPECIAL = ["ties", "empty", "nan", "plateau", "sparse"]


@pytest.mark.parametrize("case", SPECIAL)
@pytest.mark.parametrize("k", [1, 37, 120])
def test_decode_edge_cases_follow_the_definition(case, k):
    """Ties, an all -inf map, NaN cells, saturated plateaus and maps with fewer than K positive cells: the oracle equals the
    definition, NaNs by position."""
    heat, wh, reg = special_heads(case)
    assert_dets(CO.decode(heat, wh, reg, k), definition_decode(heat, wh, reg, k), case)


def test_reference_tie_order_is_not_index_order():
    """On an all -inf map every suppressed value is 0; the definition takes class 0's first K cells in index order, while
    torch's topk returns an implementation-defined order (recorded for 80 x 128 x 128 on torch 2.11's CPU topk: class 0,
    row 0, columns 41, 0, 51, 37, 59, 88, ...).  Both return K zeros."""
    ref = CO.reference()
    Cn, H, W, k = 80, 128, 128, 100
    heat = np.full((1, Cn, H, W), -np.inf, np.float32)
    wh = np.zeros((1, 2, H, W), np.float32)
    reg = np.zeros((1, 2, H, W), np.float32)
    got = CO.decode(heat[0], wh[0], reg[0], k)
    assert (got[:, 4] == 0).all() and (got[:, 5] == 0).all()
    assert np.array_equal(got[:, 0], np.arange(k, dtype=np.float32) % W)
    if ref is None:
        pytest.skip("oracle/_ref/ref_centernet.pyc not built")
    r = _sample_decode(heat, wh, reg, k)[0]
    assert (r[:, 4] == 0).all()
    assert not np.array_equal(r[:, :4], got[:, :4])


@pytest.mark.parametrize("w,h", [(1920, 1080), (640, 480), (100, 3000), (1, 1), (2, 1)])
def test_rows_equal_the_driver_loop(w, h):
    """The oracle's rows equal the sample's `if i[-2] > 0.5: i[:4] *= 4*s` loop run in torch on the same dets (s =
    max(image.shape) / 512), bit for bit, with NaN and boundary scores among them."""
    heat, wh, reg = tie_free_heads(w + h, 1, 6, 32, 32)
    heat[0, 0, 3, 3] = np.nan
    dets = CO.decode(heat[0], wh[0], reg[0], 100)
    dets[7, 4] = np.float32(0.5)
    dets[8, 4] = np.nextafter(np.float32(0.5), np.float32(1))
    got = CO.rows(dets, w, h)
    s = max((h, w, 3)) / 512
    kept = []
    for i in torch.from_numpy(dets.copy()):
        if i[-2] > 0.5:
            i[:4] *= 4 * s
            kept.append(i.numpy().copy())
    want = np.zeros(1 + 100 * 6, np.float32)
    want[0] = len(kept)
    if kept:
        want[1:1 + 6 * len(kept)] = np.concatenate(kept)
    assert np.array_equal(got, want)


# ------------------------------------------------------------------ rejected calls -------------------------------------
def _params(**kw):
    v = dict(num_classes=80, height=128, width=128, k=100, net=512, down=4, score_thresh=0.5)
    v.update(kw)
    return L.CenternetParams(*v.values())


FAKE = 1 << 20  # a non-null, 256-byte aligned address; no call below reaches a launch


def _decode_rc(p, batch=2, heat=FAKE, wh=FAKE, reg=FAKE, ws=FAKE, ws_bytes=1 << 30, dets=FAKE, frames=True, rows=FAKE):
    fw = (C.c_int32 * 4)(640, 480, 1920, 1080) if frames is True else frames
    return L.load().trtx_centernet_decode_enqueue(C.byref(p) if p is not None else None, batch, heat, wh, reg, ws, ws_bytes,
                                                  dets, fw, rows, None)


def test_decode_rejects_before_any_launch():
    lib = L.load()
    assert lib.trtx_centernet_workspace_size(C.byref(_params()), 32) == 2 * 32 * 80 * 100 * 4
    inv, uns, wsp = L.ERR_INVALID, L.ERR_UNSUPPORTED, L.ERR_WORKSPACE
    cases = [
        (dict(p=None), inv), (dict(batch=0), inv), (dict(p=_params(num_classes=0)), inv), (dict(p=_params(height=0)), inv),
        (dict(p=_params(width=-1)), inv), (dict(p=_params(k=0)), inv), (dict(p=_params(k=16385, height=128, width=128)), inv),
        (dict(p=_params(height=4, width=4, k=17)), inv), (dict(heat=None), inv), (dict(wh=None), inv), (dict(reg=None), inv),
        (dict(ws=None), inv), (dict(dets=None), inv), (dict(frames=None), inv), (dict(rows=None), inv),
        (dict(p=_params(net=0)), inv), (dict(p=_params(down=0)), inv), (dict(p=_params(score_thresh=float("nan"))), inv),
        (dict(frames=(C.c_int32 * 4)(640, 0, 1920, 1080)), inv), (dict(frames=(C.c_int32 * 4)(640, 480, -1, 1080)), inv),
        (dict(ws_bytes=2 * 2 * 80 * 100 * 4 - 1), wsp), (dict(ws=FAKE + 16), inv),
        (dict(p=_params(num_classes=1025)), uns), (dict(p=_params(height=1025, k=1)), uns),
        (dict(p=_params(width=1025, k=1)), uns), (dict(p=_params(height=1024, width=1024, k=1024)), L.OK),
        (dict(p=_params(k=1025)), uns),
    ]
    for kw, want in cases:
        p = kw.pop("p", _params())
        if want == L.OK:  # the largest accepted map: only its workspace size is asked, no launch
            assert lib.trtx_centernet_workspace_size(C.byref(p), 2) > 0
            continue
        assert _decode_rc(p, **kw) == want, (kw, want)
    # with no rows, net / down / score_thresh are not read
    assert _decode_rc(_params(net=0), ws=None, frames=None, rows=None) == inv  # the null workspace, not the net


def test_preprocess_rejects_before_any_launch():
    lib = L.load()

    def rc(descs, batch=None, net=512, dst=FAKE):
        arr = (L.ImageDesc * len(descs))(*descs) if descs is not None else None
        return lib.trtx_centernet_preprocess_enqueue(arr, len(descs) if batch is None else batch, net, dst, None)

    good = L.ImageDesc(FAKE, 640, 480, 1920, 0)
    assert rc(None, batch=1) == L.ERR_INVALID
    assert rc([good], batch=0) == L.ERR_INVALID
    assert rc([good], net=0) == L.ERR_INVALID
    assert rc([good], dst=None) == L.ERR_INVALID
    assert rc([good], dst=FAKE + 2) == L.ERR_INVALID
    assert rc([good, L.ImageDesc(None, 640, 480, 1920, 0)]) == L.ERR_INVALID
    assert rc([good, L.ImageDesc(FAKE, 0, 480, 1920, 0)]) == L.ERR_INVALID
    assert rc([good, L.ImageDesc(FAKE, 640, -1, 1920, 0)]) == L.ERR_INVALID
    assert rc([good, L.ImageDesc(FAKE, 640, 480, 1919, 0)]) == L.ERR_INVALID
    assert rc([good], net=8193) == L.ERR_UNSUPPORTED
