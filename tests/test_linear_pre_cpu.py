"""The bilinear letterbox pre-process of yolov3, yolov4, scaled-yolov4, yolov3-spp and RetinaFace, and the truncating get_rect of
yolov3, yolov4, scaled-yolov4, yolov3-tiny and yolov3-spp, on the CPU: the oracle (oracle/linear_oracle.c) against cv2 4.x's
8-bit INTER_LINEAR with IPP on and off and the drivers' plane loops restated around it (cv2.dnn.blobFromImage for yolov3-spp),
bit for bit; the 256 values of each chain; yolov3-spp's letterbox; trtx_get_rect's two new variants against the oracle and a
numpy restatement of the drivers' statements; trtx_get_rect, trtx_yolov3spp_letterbox and the oracle against the five drivers'
own compiled get_rect and yolov3-spp's compiled letterbox (oracle/_ref/libref_v3_*_host.so, or tests/golden/ref_v3_host.npz where
they were not built); and the argument checks that reject before any launch."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from oracle import linear as LO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

cv2 = pytest.importorskip("cv2")
F = np.float32
VARIANTS = (LO.YOLOV3, LO.RETINA, LO.YOLOV3_SPP)
# the drivers' own get_rect and yolov3-spp's letterbox, compiled where they lie (oracle/Makefile), or their stored outputs
G = RefOutputs("ref_v3_host")
REF_DRIVERS = ("yolov3", "yolov4", "csp", "tiny", "spp")
REF_NETS = {"yolov3": (608, 608), "yolov4": (608, 608), "csp": (512, 512), "tiny": (608, 608), "spp": (608, 608)}
MEANS = (104.0, 117.0, 123.0)


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


def _frame(rng, w, h, pad=0):
    """A random u8 BGR frame [h, w, 3] whose rows are `pad` bytes longer than 3 * w."""
    buf = rng.integers(0, 256, (h, 3 * w + pad), dtype=np.uint8)
    return np.lib.stride_tricks.as_strided(buf, (h, w, 3), (3 * w + pad, 3, 1))


def _preprocess_img_rect(w, h, net_w, net_h):
    """preprocess_img's rectangle: float r_w, r_h from double divisions, products truncated to int."""
    r_w, r_h = F(net_w / (w * 1.0)), F(net_h / (h * 1.0))
    if r_h > r_w:
        rw, rh = net_w, int(r_w * F(h))
        return 0, int((net_h - rh) / 2), rw, rh
    rw, rh = int(r_h * F(w)), net_h
    return int((net_w - rw) / 2), 0, rw, rh


def _spp_letterbox(w, h, mx):
    """yolov3-spp's letterbox -> (canvas_w, canvas_h, x, y, w, h)."""
    r = min(F(min(mx / (w * 1.0), mx / (h * 1.0))), F(1.0))
    uw, uh = int(r * F(w)), int(r * F(h))
    dw, dh = (mx - uw) % 32, (mx - uh) % 32
    return uw + dw, uh + dh, dw // 2, dh // 2, uw, uh


def _py_value(variant, c, u):
    if variant == LO.YOLOV3:
        return F(u / 255.0)
    if variant == LO.RETINA:
        return F(u - MEANS[c])
    return F(u) * F(1 / 255.0)


def _cv_preprocess(img, variant, net_w, net_h, mx=608, ipp=False):
    """The drivers' chain around cv2: the resize pasted on a 128 canvas, then the plane loop (R, G, B planes of u / 255.0 for
    yolov3, B, G, R planes of u - mean for RetinaFace) or cv::dnn::blobFromImage(pr, 1 / 255.0, size, 0, swapRB, false)."""
    img = np.ascontiguousarray(img)
    rows, cols = img.shape[:2]
    if variant == LO.YOLOV3_SPP:
        cw, ch, x, y, w, h = _spp_letterbox(cols, rows, mx)
        assert (cw, ch) == (net_w, net_h)
    else:
        x, y, w, h = _preprocess_img_rect(cols, rows, net_w, net_h)
    out = np.full((net_h, net_w, 3), 128, np.uint8)
    with _ipp(ipp):
        out[y:y + h, x:x + w] = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
        if variant == LO.YOLOV3_SPP:
            return cv2.dnn.blobFromImage(out, 1.0 / 255.0, (net_w, net_h), (0, 0, 0), True, False)[0], (x, y, w, h)
    lut = np.array([[_py_value(variant, c, u) for u in range(256)] for c in range(3)], F)
    chan = (0, 1, 2) if variant == LO.RETINA else (2, 1, 0)
    return np.stack([lut[c][out[:, :, chan[c]]] for c in range(3)]), (x, y, w, h)


# down- and upscales, the identity, tall and wide, and 1-pixel rectangle edges (2 x 1000 and 1000 x 2 at 608: a side of 1)
CASES = [((1920, 1080), (608, 608)), ((300, 200), (608, 608)), ((608, 608), (608, 608)), ((640, 480), (640, 480)),
         ((1920, 1080), (640, 480)), ((480, 1280), (608, 608)), ((2432, 600), (512, 512)), ((97, 301), (608, 608)),
         ((2, 1000), (608, 608)), ((1000, 2), (608, 608)), ((1, 3), (640, 480)), ((731, 1299), (512, 512))]
SPP_SIZES = [(1920, 1080), (300, 200), (608, 608), (607, 129), (128, 128), (1080, 1920), (600, 2432), (1000, 3), (333, 517),
             (609, 608), (2, 1000)]


@pytest.mark.parametrize("ipp", [False, True])
@pytest.mark.parametrize("variant", (LO.YOLOV3, LO.RETINA))
def test_oracle_equals_cv2_and_the_plane_loop(variant, ipp):
    rng = np.random.default_rng(21 + variant)
    for i, ((w, h), (net_w, net_h)) in enumerate(CASES):
        img = _frame(rng, w, h, pad=i % 4)
        got, rect = LO.preprocess(img, variant, net_w, net_h)
        exp, exp_rect = _cv_preprocess(img, variant, net_w, net_h, ipp=ipp)
        assert rect == exp_rect, (w, h, net_w, net_h)
        assert np.array_equal(got, exp), (w, h, net_w, net_h, ipp)
    assert any(min(_preprocess_img_rect(w, h, *net)[2:]) == 1 for (w, h), net in CASES)


@pytest.mark.parametrize("ipp", [False, True])
def test_spp_oracle_equals_cv2_letterbox_and_blob(ipp):
    """yolov3-spp at and below MAX (a frame no larger than 608 is copied), above it, tall and wide: the letterbox's canvas and
    cv2.dnn.blobFromImage's planes, bit for bit."""
    rng = np.random.default_rng(5)
    for i, (w, h) in enumerate(SPP_SIZES):
        cw, ch, *rect = _spp_letterbox(w, h, 608)
        assert LO.spp_letterbox(w, h, 608) == (cw, ch, *rect)
        assert P.yolov3spp_letterbox(w, h, 608) == ((cw, ch), tuple(rect)), (w, h)
        img = _frame(rng, w, h, pad=i % 3)
        got, got_rect = LO.preprocess(img, LO.YOLOV3_SPP, cw, ch, 608)
        exp, exp_rect = _cv_preprocess(img, LO.YOLOV3_SPP, cw, ch, ipp=ipp)
        assert got_rect == exp_rect and np.array_equal(got, exp), (w, h, ipp)
        if w <= 608 and h <= 608:  # the frame itself, not resized
            x, y = rect[:2]
            assert rect[2:] == [w, h]
            assert np.array_equal(got[0, y:y + h, x:x + w], (np.ascontiguousarray(img)[:, :, 2] * F(1)) * F(1 / 255.0))
    # another MAX; a canvas that is not net_w x net_h
    assert LO.spp_letterbox(1920, 1080, 416) == _spp_letterbox(1920, 1080, 416)
    assert LO.preprocess(_frame(rng, 300, 200), LO.YOLOV3_SPP, 608, 608, 608) is None


def test_values_of_all_256_bytes():
    """yolov3: u / 255.0 rounded once from double; RetinaFace: u - mean, exact; yolov3-spp: blobFromImage's float product.
    The first and the last differ in the last bit for some bytes, so each is pinned to its own reference."""
    u = np.arange(256)
    v3 = np.array([[LO.input_value(LO.YOLOV3, c, k) for k in u] for c in range(3)], F)
    assert np.array_equal(v3, np.broadcast_to((u / 255.0).astype(F), (3, 256)))
    retina = np.array([[LO.input_value(LO.RETINA, c, k) for k in u] for c in range(3)], np.float64)
    assert np.array_equal(retina, u[None, :] - np.array(MEANS)[:, None])
    spp = np.array([[LO.input_value(LO.YOLOV3_SPP, c, k) for k in u] for c in range(3)], F)
    img = np.stack([u.astype(np.uint8)] * 3, axis=1)[None]  # one row of 256 grey pixels
    for ipp in (False, True):
        with _ipp(ipp):
            blob = cv2.dnn.blobFromImage(img, 1.0 / 255.0, (256, 1), (0, 0, 0), True, False)[0, :, 0, :]
        assert np.array_equal(spp, blob)
    assert np.array_equal(spp[0], u.astype(F) * F(1 / 255.0))
    differ = int((spp[0] != v3[0]).sum())
    assert 0 < differ < 256, differ
    for variant in VARIANTS:
        exp = np.array([[_py_value(variant, c, k) for k in u] for c in range(3)], F)
        got = np.array([[LO.input_value(variant, c, k) for k in u] for c in range(3)], F)
        assert np.array_equal(got, exp), variant


# ------------------------------------------------------------------ get_rect -------------------------------------------
def _np_get_rect(variant, net_w, net_h, img_w, img_h, boxes):
    """The drivers' get_rect in numpy float32 (each operation rounded once), vectorised over boxes [n, 4] -> (rects [n, 4] int64,
    defined [n])."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _np_get_rect_body(variant, net_w, net_h, img_w, img_h, boxes.astype(F))


def _np_get_rect_body(variant, net_w, net_h, img_w, img_h, b):
    half_w, half_h = b[:, 2] / F(2), b[:, 3] / F(2)
    if variant == LO.YOLOV3_SPP:
        cw, ch, px, py, uw, uh = _spp_letterbox(img_w, img_h, net_w)
        ratio = min(F(min(net_w / (img_w * 1.0), net_w / (img_h * 1.0))), F(1.0))
        c = [b[:, 0] - half_w - F(px), b[:, 1] - half_h - F(py), b[:, 0] + half_w - F(px), b[:, 1] + half_h - F(py)]
    else:
        r_w, r_h = F(net_w / (img_w * 1.0)), F(net_h / (img_h * 1.0))
        c = [b[:, 0] - half_w, b[:, 1] - half_h, b[:, 0] + half_w, b[:, 1] + half_h]
        if r_h > r_w:
            ratio, pad, k = r_w, (F(net_h) - r_w * F(img_h)) / F(2), 1
        else:
            ratio, pad, k = r_h, (F(net_w) - r_h * F(img_w)) / F(2), 0
        c[k], c[k + 2] = c[k] - pad, c[k + 2] - pad
    ok = np.ones(len(b), bool)
    v = []
    for x in c:
        fine = (x >= F(-2 ** 31)) & (x < F(2 ** 31))
        t = np.where(fine, np.trunc(np.where(fine, x, 0)), 0).astype(np.int64)
        q = t.astype(F) / ratio
        fine2 = (q >= F(-2 ** 31)) & (q < F(2 ** 31))
        ok &= fine & fine2
        v.append(np.where(fine2, np.trunc(np.where(fine2, q, 0)), 0).astype(np.int64))
    w, h = v[2] - v[0], v[3] - v[1]
    ok &= (w >= -2 ** 31) & (w <= 2 ** 31 - 1) & (h >= -2 ** 31) & (h <= 2 ** 31 - 1)
    rect = np.stack([v[0], v[1], w, h], 1)
    return np.where(ok[:, None], rect, 0), ok


def _boxes(rng, n):
    """cx, cy, w, h in network pixels: inside, negative (truncation toward zero), past the frame, huge, non-finite."""
    b = np.concatenate([rng.uniform(-50, 700, (n, 2)), rng.uniform(0, 400, (n, 2))], 1).astype(F)
    b[: n // 8, :2] = rng.uniform(-40, 0, (n // 8, 2))
    b[n // 8: n // 4] *= F(4)
    b[n // 4: n // 4 + 64] = rng.choice(np.array([np.nan, np.inf, -np.inf, 1e30, -3e9, 2.2e9, 1e9], F), (64, 4))
    b[n // 4 + 64: n // 4 + 96] = rng.uniform(-1, 1, (32, 4)).astype(F) * F(2e9)
    return b


FRAMES = [(1920, 1080), (1080, 1920), (608, 608), (640, 480), (300, 200), (1, 7), (7, 1), (4000, 3000), (99, 331), (5, 70000),
          (70000, 5), (2047, 1151)]
NETS = {LO.YOLOV3: [(608, 608), (512, 512), (416, 416), (640, 480)], LO.YOLOV3_SPP: [(608, 608), (416, 416)]}
LIB_VARIANT = {LO.YOLOV3: L.YOLO_V3, LO.YOLOV3_SPP: L.RECT_YOLOV3_SPP}


@pytest.mark.parametrize("variant", (LO.YOLOV3, LO.YOLOV3_SPP))
def test_get_rect_library_oracle_and_numpy_agree(variant):
    """trtx_get_rect, the C oracle and the numpy restatement give the same rectangles and the same undefined boxes on 2 048
    boxes x 12 frames x every net; negative corners truncate toward zero (-0.9 -> 0), so rectangles straddling 0 shrink."""
    rng = np.random.default_rng(7 + variant)
    boxes = _boxes(rng, 2048)
    lib = L.load()
    r = (C.c_int * 4)()
    undefined = toward_zero = 0
    for net_w, net_h in NETS[variant]:
        for w, h in FRAMES:
            exp, ok = _np_get_rect(variant, net_w, net_h, w, h, boxes)
            undefined += int((~ok).sum())
            for i, bb in enumerate(boxes):
                got, defined = LO.get_rect(variant, net_w, net_h, w, h, bb)
                assert defined == ok[i] and got == tuple(exp[i]), (net_w, net_h, w, h, bb, got, exp[i])
                assert lib.trtx_get_rect(LIB_VARIANT[variant], net_w, net_h, w, h, (C.c_float * 4)(*bb), r) == 0
                assert tuple(r) == got, (net_w, net_h, w, h, bb, tuple(r), got)
            with np.errstate(invalid="ignore"):
                toward_zero += int(((boxes[:, 0] - boxes[:, 2] / 2) < 0).sum())
    assert undefined > 0 and toward_zero > 0


def test_get_rect_spelled_cases():
    """Hand-checked values: a 1920 x 1080 frame in 608 x 608 pads y by 133 (float) and scales by 608 / 1920."""
    r_w = F(608 / 1920.0)
    pad = (F(608) - r_w * F(1080)) / F(2)
    bb = [100.0, 200.0, 50.0, 60.0]
    l, r = int(F(100) - F(25)), int(F(100) + F(25))
    t, b = int(F(200) - F(30) - pad), int(F(200) + F(30) - pad)
    exp = tuple(int(F(v) / r_w) for v in (l, t)) + (int(F(r) / r_w) - int(F(l) / r_w), int(F(b) / r_w) - int(F(t) / r_w))
    assert P.get_rect(1920, 1080, bb, 608, 608, L.YOLO_V3) == exp
    # truncation toward zero: l = (int)(-0.5f) = 0, not -1
    assert P.get_rect(608, 608, [0.25, 10.0, 1.5, 2.0], 608, 608, L.YOLO_V3)[0] == 0
    # yolov3-spp: a 300 x 200 frame is not scaled (ra = 1), pads (308 % 32) / 2 = 10 and (408 % 32) / 2 = 12
    assert P.get_rect(300, 200, [110.0, 112.0, 20.0, 40.0], 608, 608, L.RECT_YOLOV3_SPP) == (90, 80, 20, 40)
    for bad in ([np.nan, 1, 1, 1], [1, np.inf, 1, 1], [3e9, 1, 1, 1], [-1.5e9, 0, 1.5e9, 0]):
        assert P.get_rect(1920, 1080, bad, 608, 608, L.YOLO_V3) == (0, 0, 0, 0), bad
        assert P.get_rect(1920, 1080, bad, 608, 608, L.RECT_YOLOV3_SPP) == (0, 0, 0, 0), bad


# ------------------------------------------------------------------ argument checks (no launch) ------------------------
def test_rejected_arguments():
    lib = L.load()
    descs = (L.ImageDesc * 2)()
    for d in descs:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12

    def pre(v=LO.YOLOV3, d=descs, b=2, w=608, h=608, mx=608, dst=16):
        return lib.trtx_linear_preprocess_enqueue(v, d, b, w, h, mx, dst, None)

    assert pre(d=None) == L.ERR_INVALID
    assert pre(b=0) == L.ERR_INVALID
    assert pre(w=0) == L.ERR_INVALID
    assert pre(h=-1) == L.ERR_INVALID
    assert pre(dst=None) == L.ERR_INVALID
    assert pre(dst=18) == L.ERR_INVALID  # not 4-byte aligned
    for v in (-1, 3, L.RECT_YOLOV3_SPP):
        assert pre(v=v) == L.ERR_INVALID, v
    assert pre(v=LO.YOLOV3_SPP, w=32, h=32, mx=0) == L.ERR_INVALID
    assert pre(v=LO.YOLOV3_SPP, w=608, h=608) == L.ERR_INVALID  # a 4 x 4 frame's canvas is 4 + 604 % 32 = 32 wide
    descs[1].pitch = 11  # < 3 * width
    assert pre() == L.ERR_INVALID
    descs[1].pitch, descs[1].data_dev = 12, None
    assert pre() == L.ERR_INVALID
    descs[1].data_dev, descs[1].width, descs[1].height, descs[1].pitch = 16, 1, 5000, 3  # an empty rectangle
    assert pre() == L.ERR_UNSUPPORTED
    assert pre(v=LO.RETINA, w=640, h=480) == L.ERR_UNSUPPORTED
    one = (L.ImageDesc * 1)()
    one[0].data_dev, one[0].width, one[0].height, one[0].pitch = 16, 1, 5000, 3
    assert pre(v=LO.YOLOV3_SPP, d=one, b=1) == L.ERR_UNSUPPORTED  # spp: its canvas side is 0 there, but empty comes first
    descs[1].width, descs[1].height, descs[1].pitch = 4800, 100, 14400  # a rectangle 4 800 wide: staged rows too large
    assert pre(w=4800, h=4800) == L.ERR_UNSUPPORTED
    # SPP frames with different canvases: 300 x 200 -> 320 x 224, 250 x 200 -> 256 x 224
    descs[0].width, descs[0].height, descs[0].pitch = 300, 200, 900
    descs[1].width, descs[1].height, descs[1].pitch = 250, 200, 750
    assert pre(v=LO.YOLOV3_SPP, w=320, h=224) == L.ERR_INVALID
    assert pre(v=LO.YOLOV3_SPP, w=256, h=224) == L.ERR_INVALID
    # an invalid descriptor after an unsupported one is still TRTX_ERR_INVALID: every descriptor is checked first
    big = (L.ImageDesc * 70)()
    for d in big:
        d.data_dev, d.width, d.height, d.pitch = 16, 4, 4, 12
    big[0].width, big[0].height, big[0].pitch = 1, 5000, 3
    big[69].pitch = 0
    assert lib.trtx_linear_preprocess_enqueue(0, big, 70, 608, 608, 608, 16, None) == L.ERR_INVALID
    # the letterbox helper
    g = (C.c_int * 6)()
    assert lib.trtx_yolov3spp_letterbox(0, 5, 608, g) == L.ERR_INVALID
    assert lib.trtx_yolov3spp_letterbox(5, 5, 0, g) == L.ERR_INVALID
    assert lib.trtx_yolov3spp_letterbox(5, 5, 608, None) == L.ERR_INVALID
    assert lib.trtx_yolov3spp_letterbox(1, 5000, 608, g) == L.ERR_UNSUPPORTED and g[4] == 0
    # get_rect
    bb, r = (C.c_float * 4)(1, 1, 1, 1), (C.c_int * 4)()
    assert lib.trtx_get_rect(L.RECT_YOLOV3_SPP, 608, 416, 100, 100, bb, r) == L.ERR_INVALID  # MAX is one side
    for v in (L.YOLO_V26, 4, 15, 17):
        assert lib.trtx_get_rect(v, 608, 608, 100, 100, bb, r) == L.ERR_INVALID, v
    assert lib.trtx_get_rect(L.YOLO_V3, 608, 608, 0, 100, bb, r) == L.ERR_INVALID


def test_seg_rows_entry_checks():
    """The rows-only mode of trtx_yolo_seg_postprocess_enqueue takes the two rectangle variants; with canvases they are
    TRTX_ERR_INVALID, and SPP needs a square net.  Rejected before any launch (the device pointers are never read)."""
    lib = L.load()

    q = L.MaskParams(L.YOLO_V3, 608, 608, 152, 152, 32, 7, 0, 1)
    arr = (L.Frame * 1)()
    arr[0].img_w, arr[0].img_h, arr[0].masks_dev, arr[0].pitch = 64, 48, 32, 64
    assert lib.trtx_yolo_seg_postprocess_enqueue(C.byref(q), arr, 1, C.c_void_p(16), C.c_void_p(16), 10, C.c_void_p(16),
                                                 None) == L.ERR_INVALID  # canvases with a rectangle-only variant
    q.variant, q.net_h = L.RECT_YOLOV3_SPP, 416
    arr[0].masks_dev = None
    assert lib.trtx_yolo_seg_postprocess_enqueue(C.byref(q), arr, 1, None, C.c_void_p(16), 10, C.c_void_p(16),
                                                 None) == L.ERR_INVALID  # net_w != net_h


# ------------------------------------------------------------------ against the drivers' compiled code ------------------
@pytest.mark.parametrize("driver", REF_DRIVERS)
def test_get_rect_equals_the_drivers_compiled_get_rect(driver):
    """trtx_get_rect and the oracle equal each driver's own compiled get_rect -- yolov3, yolov4, scaled-yolov4 (its common.hpp),
    yolov3-tiny (TRTX_YOLO_V3, at the driver's INPUT_W x INPUT_H) and yolov3-spp (TRTX_RECT_YOLOV3_SPP, MAX_INPUT_SIZE) -- on
    1 024 boxes x 12 frames, negative, past-the-frame and huge boxes included.  Boxes the oracle finds undefined in the
    reference (non-finite, out of the int range) are left out of the comparison: the compiled code's result there is
    whatever x86-64 gives, and the library's is {0, 0, 0, 0}."""
    ref = G.lib(f"libref_v3_{driver}_host.so")
    net_w, net_h = REF_NETS[driver]
    if ref is not None:
        wh = (C.c_int * 2)()
        ref.ref_v3_net(wh)
        assert (wh[0], wh[1]) == (net_w, net_h)
    spp = driver == "spp"
    variant, lib_variant = (LO.YOLOV3_SPP, L.RECT_YOLOV3_SPP) if spp else (LO.YOLOV3, L.YOLO_V3)
    boxes = _boxes(np.random.default_rng(31), 1024)
    lib = L.load()
    r = (C.c_int * 4)()
    got, live, defined = [], [], []
    for w, h in FRAMES:
        for bb in boxes:
            cb = (C.c_float * 4)(*bb)
            assert lib.trtx_get_rect(lib_variant, net_w, net_h, w, h, cb, r) == 0
            orc, ok = LO.get_rect(variant, net_w, net_h, w, h, bb)
            assert tuple(r) == orc
            got.append(orc)
            defined.append(ok)
            if ref is not None:
                ref.ref_v3_get_rect(w, h, cb, r)
                live.append(tuple(r) if ok else (0, 0, 0, 0))
    assert sum(defined) > len(defined) // 2 and not all(defined)
    G.equal(f"{driver}.get_rect", np.array(got, np.int64), None if ref is None else np.array(live, np.int64))


def test_spp_letterbox_equals_the_drivers_compiled_letterbox():
    """trtx_yolov3spp_letterbox and the oracle equal yolov3-spp's own compiled letterbox (its canvas and the rectangle it pastes
    the resized frame into) on frame sizes at, below and above MAX_INPUT_SIZE, tall and wide."""
    ref = G.lib("libref_v3_spp_host.so")
    sizes = [(w, h) for w in (1, 2, 31, 127, 128, 300, 607, 608, 609, 1000, 1920, 4000) for h in (1, 3, 129, 200, 608, 1080,
                                                                                                   2432, 70000)]
    lib = L.load()
    g = (C.c_int * 6)()
    got, live = [], []
    for w, h in sizes:
        rc = lib.trtx_yolov3spp_letterbox(w, h, 608, g)
        assert rc in (L.OK, L.ERR_UNSUPPORTED) and (rc == L.OK) == (g[4] > 0 and g[5] > 0)
        assert tuple(g) == LO.spp_letterbox(w, h, 608), (w, h)
        got.append(tuple(g))
        if ref is not None:
            ref.ref_v3_letterbox(w, h, g)
            live.append(tuple(g))
    G.equal("spp.letterbox", np.array(got, np.int64), None if ref is None else np.array(live, np.int64))
