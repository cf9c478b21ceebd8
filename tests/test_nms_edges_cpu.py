"""Pins oracle.nms -- which the GPU NMS tests trust -- to the reference's own compiled host nms() / nms_obb() / RetinaFace
nms() on the inputs where the two could part, built by oracle/nms_cases.py exactly as tests/test_nms_paths_gpu.py builds
them: float class ids, IoUs at and a few ulps around the threshold, degenerate boxes, thresholds below 0 and above 4, and
NaN coordinates.  Confidences are distinct, so the reference's std::sort (not stable) has one answer.  Where oracle/_ref
was not built the reference's outputs come from tests/golden/ref_host_calls.npz."""
import ctypes as C

import numpy as np
import pytest

from oracle import nms_cases as NC
from oracle.golden import RefOutputs

G = RefOutputs("ref_host_calls")

# variant -> (reference library, function, floats per reference Detection row)
REF = {0: ("libref_yolov8_host.so", "ref_v8_nms", 90), 1: ("libref_yolov5_host.so", "ref_v5_nms", 38),
       2: ("libref_retina_host.so", "ref_retina_nms", 15), 3: ("libref_yolov8_host.so", "ref_v8_nms_obb", 90)}
CONF = 0.25  # RetinaFace's nms() has its own `<= 0.1`


def _compare(oracle, key, variant, rows, thr):
    """rows = (box, conf, cls) -> one reference buffer; the oracle's kept rows == the reference's, bit for bit."""
    box, conf_col, cls = rows
    lib_name, fn_name, F = REF[variant]
    n = len(conf_col)
    buf = np.zeros(1 + n * F, np.float32)
    buf[0] = n
    r = buf[1:].reshape(n, F)
    r[:, 5:] = np.random.default_rng(n).uniform(-5, 5, (n, F - 5))
    r[:, :4], r[:, 4] = box, conf_col
    if variant != 2:
        r[:, 5] = cls
    conf = 0.1 if variant == 2 else CONF
    mine, _ = oracle.nms(variant, buf, n, F, conf, thr)
    ref = None
    lib = G.lib(lib_name)
    if lib is not None:
        out = np.zeros((n + 1) * F, np.float32)
        args = (thr,) if variant == 2 else (conf, thr)
        k = getattr(lib, fn_name)(buf.ctypes.data_as(C.c_void_p), *[C.c_float(t) for t in args], out.ctypes.data_as(C.c_void_p))
        ref = out[:k * F].reshape(k, F)
    G.equal(key, mine, ref, nan_ok=True)
    return mine


@pytest.mark.parametrize("variant", [0, 1, 3])
def test_float_class_ids_group_like_the_reference(oracle, variant):
    """std::map<float, ...> keys: -3 < -1 < -0.0 == +0.0 < 2.0 < 2.5 < 1e9 < 3e9 < 5e9, 2.5 rows lying on 2.0 rows, every
    row emitted with its own class float."""
    rng = np.random.default_rng(2100 + variant)
    mine = _compare(oracle, f"edges.class_ids.{variant}", variant, NC.float_id_rows(rng, variant, 180), 0.45)
    assert mine[0, 5] == -3.0 and np.signbit(mine[:, 5]).sum() > (mine[:, 5] < 0).sum()


@pytest.mark.parametrize("variant,thr", [(v, t) for v in (0, 1, 2) for t in (0.45, 0.5, 0.4)])
def test_iou_at_and_around_the_threshold(oracle, variant, thr):
    """Float IoU exactly fl(thr) (kept; for thr 0.45 and 0.4 with the exact quotient above fl(thr), where the division-free
    sign test of the kernel would suppress) and 1..3 ulps either side; RetinaFace also on small boxes whose `+ 1e-6` decides."""
    rows, kept, sign_test_wrong = NC.threshold_rows(variant, thr)
    assert sign_test_wrong == (thr != 0.5)
    assert len(_compare(oracle, f"edges.threshold.{variant}.{thr}", variant, rows, thr)) == kept


@pytest.mark.parametrize("variant,thr", [(v, t) for v in (0, 1, 2) for t in (0.45, -0.25, 4.5)])
def test_degenerate_boxes(oracle, variant, thr):
    """Zero-area (some on one point: IoU 0/0), inverted, 1e30 (the intersection overflows), +-inf and NaN coordinates, with
    thr < 0 (disjoint boxes overlap) and thr > 4."""
    rng = np.random.default_rng(2200 + variant + int(10 * thr))
    _compare(oracle, f"edges.degenerate.{variant}.{thr}", variant, NC.degenerate_rows(rng, variant), thr)


@pytest.mark.parametrize("variant,thr", [(v, t) for v in (0, 1, 2) for t in (0.45, -0.25)])
def test_nan_coordinates(oracle, variant, thr):
    """A NaN in one coordinate of a kept or a later row.  std::max(a, b) is `a < b ? b : a` and std::min(a, b) is
    `b < a ? b : a`: a NaN in the later row is ignored and one in the kept row propagates.  (CXCYWH areas hold no cx / cy,
    so a row with a NaN centre can be suppressed; LTRB rows with a NaN can be, when thr < 0, as disjoint.)"""
    rng = np.random.default_rng(2300 + variant + int(10 * thr))
    box, conf, cls = NC.random_rows(rng, variant, 120, rng.integers(0, 2, 120), NC.distinct_conf(rng, 120))
    nan_rows = np.flatnonzero(np.arange(120) % 3 == 1)
    box[nan_rows, rng.integers(0, 4, len(nan_rows))] = np.nan
    _compare(oracle, f"edges.nan_coords.{variant}.{thr}", variant, (box, conf, cls), thr)
