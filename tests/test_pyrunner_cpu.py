"""The Python runners' pre- and post-process without a GPU: the library's preprocess_image rectangle against the runners'
arithmetic, the numpy oracle (oracle/pyrunner.py) against the runners' own methods -- run from the reference tree where it
is present, else against their digests in tests/golden/ref_pyrunner_host.npz --, the oracle's tie and termination rules, and
the C ABI's rejections."""

import ctypes as C
import math

import numpy as np
import pytest

from oracle import golden as G
from oracle import pyrunner as PR
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

R = G.RefOutputs("ref_pyrunner_host")
NETS = [(640, 640), (608, 608), (1024, 1024), (640, 384)]
COMMON_SIDES = [333, 360, 480, 540, 576, 600, 720, 768, 800, 1024, 1080, 1200, 1440, 2160]


def _runner_rect(w, h, net_w, net_h):
    """preprocess_image's statements (yolov8_det_trt.py:223-236) as the runner writes them."""
    r_w, r_h = net_w / w, net_h / h
    if r_h > r_w:
        tw, th, tx1 = net_w, int(r_w * h), 0
        ty1 = int((net_h - th) / 2)
    else:
        tw, th, ty1 = int(r_h * w), net_h, 0
        tx1 = int((net_w - tw) / 2)
    return tx1, ty1, tw, th


@pytest.mark.parametrize("net_w,net_h", NETS)
def test_rect_equals_runner_arithmetic(net_w, net_h):
    """Every width 1..2100 against the common heights and every height against the common widths."""
    lib = L.load()
    r = (C.c_int * 4)()
    sizes = [(w, h) for h in COMMON_SIDES for w in range(1, 2101)] + [(w, h) for w in COMMON_SIDES for h in range(1, 2101)]
    for w, h in sizes:
        assert lib.trtx_pyrunner_letterbox_rect(w, h, net_w, net_h, r) == 0
        exp = _runner_rect(w, h, net_w, net_h)
        assert tuple(r) == exp == PR.letterbox_rect(w, h, net_w, net_h), (w, h, tuple(r), exp)


def test_rect_differs_from_preprocess_img():
    """592 x 333 into 640 x 640: the runner's double ratio gives 360 rows, preprocess_img's float ratio 359."""
    assert P.pyrunner_letterbox_rect(592, 333) == (0, 140, 640, 360)
    r = (C.c_int * 4)()
    L.load().trtx_calib_letterbox_rect(592, 333, 640, 640, r)
    assert tuple(r) == (0, 140, 640, 359)


def test_data_rule_is_linear_yolov3s():
    """The runner's float32 u / 255.0 is (float)(u / 255.0) for every byte, TRTX_LINEAR_YOLOV3's value."""
    u = np.arange(256)
    assert np.array_equal(u.astype(np.float32) / 255.0, (u / 255.0).astype(np.float32))


@pytest.mark.parametrize("net", PR.PRE_NETS)
def test_preprocess_oracle_equals_runner(net):
    """The oracle's letterbox equals the runner's preprocess_image bit for bit on the GPU test's frames."""
    pytest.importorskip("cv2")
    ref = PR.reference_runner("yolov8_det_trt", *net)
    for i, f in enumerate(PR.pre_frames(net)):
        got = PR.preprocess(f, *net)
        R.equal(f"pre-{net[0]}x{net[1]}-{i}", got, None if ref is None else ref.preprocess_image(f)[0][0])


@pytest.mark.parametrize("key,runner,dets,sizes", PR.post_cases(P.PYRUNNER_PRESETS), ids=lambda v: v if isinstance(v, str) else "")
def test_postprocess_oracle_equals_runner(key, runner, dets, sizes):
    """Every preset on 32 frames of mixed sizes: distinct and equal label columns, boxes past the frame's edge, NaN
    confidences, a count of 0, 1 and past max_rows."""
    preset = P.PYRUNNER_PRESETS[runner]
    got = PR.canonical([PR.postprocess(d, w, h, preset) for d, (w, h) in zip(dets, sizes)])
    ref = PR.reference_runner(runner)
    exp = None if ref is None else PR.canonical([PR.reference_rows(ref, d, w, h) for d, (w, h) in zip(dets, sizes)])
    R.equal(key, got, exp)


def _buf(rows, F=6, max_rows=8):
    b = np.zeros(1 + max_rows * F, np.float32)
    b[0] = len(rows)
    b[1:1 + len(rows) * F] = np.asarray(rows, np.float32).reshape(-1)
    return b


def test_label_column_groups_the_nms():
    """yolov8's 90-float rows: two overlapping rows of classes 1 and 2 with float 89 equal come back as one row; with
    float 89 distinct, as two.  The runner agrees where it is present."""
    rows = np.zeros((2, 90), np.float32)
    rows[0, :6] = [100, 100, 200, 200, 0.9, 1]
    rows[1, :6] = [105, 105, 205, 205, 0.8, 2]
    ref = PR.reference_runner("yolov8_det_trt")
    for label, n in ((0.0, 1), (None, 2)):
        rows[:, 89] = rows[:, 5] if label is None else label
        buf = _buf(rows, 90, 4)
        got = PR.postprocess(buf, 640, 640, P.PYRUNNER_PRESETS["yolov8_det_trt"])
        assert len(got) == n
        if ref is not None:
            assert np.array_equal(got, PR.reference_rows(ref, buf, 640, 640))


def test_termination_rule():
    """Front rows that do not remove themselves -- a NaN label, a NaN box corner, an inverted box -- are kept once and do
    not suppress; the runner's loop does not end on these rows, so only the rule is checked."""
    preset = P.PYRUNNER_PRESETS["yolov10_det_trt"]
    rows = [[10, 10, 50, 50, 0.9, np.nan], [12, 12, 52, 52, 0.8, np.nan],  # NaN labels: both kept
            [300, 300, 200, 200, 0.7, 3], [301, 301, 201, 201, 0.6, 3],    # inverted: IoU of each with itself <= 0.4
            [400, np.nan, 450, 450, 0.55, 4], [400, 400, 450, 450, 0.52, 4]]  # NaN corner: no pair with it matches
    got = PR.postprocess(_buf(rows), 640, 640, preset)
    assert np.array_equal(got[:, 4], np.float32([0.9, 0.8, 0.7, 0.6, 0.55, 0.52]))


def test_tie_rule():
    """Equal confidences are taken in ascending row order: the earlier row is kept and removes the later."""
    preset = P.PYRUNNER_PRESETS["yolov10_det_trt"]
    rows = [[0, 0, 10, 10, 0.5, 0], [20, 20, 40, 40, 0.7, 0], [21, 21, 41, 41, 0.7, 0], [1, 1, 11, 11, 0.5, 0]]
    got = PR.postprocess(_buf(rows), 640, 640, preset)
    assert np.array_equal(got[:, 0], np.float32([20, 0]))


def _params(**kw):
    d = dict(box_format=L.BOX_LTRB, net_w=640, net_h=640, row_floats=90, label_col=89, conf_col=-1, conf_thresh=0.5,
             nms_thresh=0.4)
    d.update(kw)
    return L.PyrunnerParams(*d.values())


def test_abi_rejections():
    """Every malformed call is refused before any launch, so these run without a device."""
    lib = L.load()
    assert lib.trtx_abi_sizeof(16) == C.sizeof(L.PyrunnerParams)
    wh = (C.c_int32 * 4)(640, 480, 1920, 1080)
    bad_wh = (C.c_int32 * 4)(640, 480, 0, 1080)
    D, O = C.c_void_p(1 << 20), C.c_void_p(1 << 21)  # never dereferenced: each call below fails its checks first
    post = lib.trtx_pyrunner_postprocess_enqueue
    cases = [
        (None, wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(), None, 2, D, 1000, O, L.ERR_INVALID),
        (_params(), wh, 0, D, 1000, O, L.ERR_INVALID),
        (_params(), wh, 2, None, 1000, O, L.ERR_INVALID),
        (_params(), wh, 2, D, 1000, None, L.ERR_INVALID),
        (_params(), wh, 2, D, 0, O, L.ERR_INVALID),
        (_params(box_format=L.BOX_RETINA), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(net_w=0), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(label_col=4), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(label_col=90), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(conf_col=89), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(conf_col=4), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(conf_col=90), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(conf_thresh=math.nan), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(nms_thresh=math.nan), wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(), wh, 2, C.c_void_p((1 << 20) + 2), 1000, O, L.ERR_INVALID),
        (_params(), bad_wh, 2, D, 1000, O, L.ERR_INVALID),
        (_params(), wh, 2, D, 2049, O, L.ERR_UNSUPPORTED),
    ]
    for i, (p, f, b, d, m, o, rc) in enumerate(cases):
        assert post(None if p is None else C.byref(p), f, b, d, m, o, None) == rc, i
    r = (C.c_int * 4)()
    assert lib.trtx_pyrunner_letterbox_rect(0, 10, 640, 640, r) == L.ERR_INVALID
    assert lib.trtx_pyrunner_letterbox_rect(10, 10, 640, 640, None) == L.ERR_INVALID
    descs = (L.ImageDesc * 1)()
    descs[0].data_dev, descs[0].width, descs[0].height, descs[0].pitch = 1 << 20, 1, 2000, 3
    assert lib.trtx_linear_preprocess_enqueue(L.LINEAR_PY, descs, 1, 640, 640, 0, O, None) == L.ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        P.PyRunnerPostprocess("yolov6")
