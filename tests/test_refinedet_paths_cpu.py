"""The cases of tests/test_refinedet_paths_gpu.py pinned on the CPU: the oracle (oracle/refinedet_oracle.c) equals the
transcription of the reference's libtorch post-process run in torch on the CPU on each tie-free case -- every accepted
side, C = 2 .. 1024 and every top_k there -- and the crafted geometry does what its case claims under nms()'s IoU in
NumPy float64.  A failure there then points at the kernel, not at a broken fixture."""

import numpy as np
import pytest

from oracle import refinedet as RO
from oracle import refinedet_cases as RC

F32 = np.float32


def _compare(case, b=0, exact=False):
    """The oracle against the CPU transcription on frame b: the same kept set in the same order, the boxes equal (zero
    offsets: exact) or within 4 ulps (glibc's exp here, torch's CPU exp there) -> the rows."""
    h = [x[b] for x in case.h]
    want = RO.reference_postprocess(*h, **case.kw)
    max_det = (case.h[3].shape[2] - 1) * case.kw["top_k"]
    got = RO.postprocess(*h, **case.kw, max_det=max_det)
    n = int(got[0])
    assert n == len(want)
    g = got[1:1 + 6 * n].reshape(-1, 6)
    assert np.array_equal(g[:, 4:].view(np.int32), want[:, 4:].view(np.int32))
    assert np.array_equal(np.isnan(g[:, :4]), np.isnan(want[:, :4]))
    fin = ~np.isnan(want[:, :4])
    ulps = np.abs(g[:, :4].view(np.int32).astype(np.int64) - want[:, :4].view(np.int32).astype(np.int64))
    assert (ulps[fin] <= (0 if exact else 4)).all()
    return want


def _kept(rows):
    labels = rows[:, 5].astype(int)
    return {c: int((labels == c).sum()) for c in np.unique(labels)}


# ------------------------------------------------------------------ the oracle against the transcription ---------------
@pytest.mark.parametrize("net", RC.SIDES)
def test_side_oracle_equals_transcription(net):
    """Every accepted side, with C cycling over 2, 21, 25, 81 and top_k over the whole list."""
    case = RC.side(net)
    assert _compare(case).shape[0] > 0


@pytest.mark.parametrize("net", [64, 128])
def test_many_classes_oracle_equals_transcription(net):
    case = RC.many_classes(net)
    for b in range(2):
        assert len(_compare(case, b)) > 1025


@pytest.mark.parametrize("K", RC.TOP_KS)
def test_cut_oracle_equals_transcription(K):
    """0, 1, K - 1, K, K + 1 and K + 8000 candidates: the K best are kept, the rest cut."""
    case = RC.cut(K)
    got = _kept(_compare(case, exact=True))
    assert {c: got.get(c, 0) for c in case.claims} == case.claims


# ------------------------------------------------------------------ the geometry the cases claim -----------------------
def test_disjoint_squares_are_all_kept():
    b = RC.boxes(1024)[RC.disjoint_squares(1024)]
    assert len(b) == 1024
    assert RC.nms_keep(b, 0.45) == list(range(1024))


def test_chain_alternates():
    """Along each row neighbours overlap above 0.45 and next-but-one neighbours below it, so every other box is kept; the
    three rows do not overlap one another."""
    b = RC.boxes(1024)[RC.chain(1024, (0, 64, 127))]
    for i in range(0, len(b) - 2):
        if i % 128 < 126:
            assert RC.iou(b[i], b[i + 1])[0] > 0.45 and RC.iou(b[i], b[i + 2])[0] < 0.45
    assert RC.nms_keep(b, 0.45) == list(range(0, 384, 2))


def _class_boxes(case, c):
    """Class c's candidates' boxes in score order (descending, distinct scores)."""
    ids = np.flatnonzero(case.h[3][0, :, c] > F32(0.01))
    ids = ids[np.argsort(-case.h[3][0, ids, c], kind="stable")]
    return RC.decode(RO.priors(case.kw["net"])[ids], case.h[0][0, ids], case.h[2][0, ids])


def test_edges_geometry():
    case = RC.edges(0.45)
    same = _class_boxes(case, 2)
    assert len(same) == 1500 and (same == same[0]).all() and np.isfinite(same).all()
    assert RC.iou(same[0], same[1])[0] == 1.0
    assert np.isnan(_class_boxes(case, 3)).any(axis=1).sum() == 64
    flat = _class_boxes(case, 4)
    zero = (flat[:, 2] == flat[:, 0]) | (flat[:, 3] == flat[:, 1])
    assert zero.sum() == len(flat) - len(range(4, len(flat), 5))  # all but every fifth anchor
    assert np.isnan(RC.iou(flat[zero][0], flat[zero][1:])).all()  # 0 / 0
    for c, n in case.claims.items():
        assert len(RC.nms_keep(_class_boxes(case, c), 0.45)) == n
    for t in (0.0, -0.5):
        assert all(len(RC.nms_keep(_class_boxes(case, c), t)) == 1 for c in (1, 2, 3, 4))


def test_pairs_straddle_and_rounding_flips():
    (i, j, v), (ri, rj, t) = RC.pair_search()
    b = RC.boxes(320)
    assert RC.iou(b[i], b[j])[0] == v and float(F32(v)) != v
    above, below = np.nextafter(F32(v), F32(1)), np.nextafter(F32(v), F32(0))
    assert below < v < above
    assert len(RC.nms_keep(b[[i, j]], float(above))) == 2 and len(RC.nms_keep(b[[i, j]], float(below))) == 1
    assert float(F32(t)) == t
    assert len(RC.nms_keep(b[[ri, rj]], t)) != len(RC.nms_keep(b[[ri, rj]], t, round_i=False))
    for case in (RC.pair(i, j, float(above)), RC.pair(ri, rj, t)):
        _compare(case, exact=True)


@pytest.mark.parametrize("B", [1, 3])
def test_frames_oracle_and_claims(B):
    """Scores at, below and above score_thresh and +inf reach the rows; NaN scores are never candidates; frame 1 of 3 is
    empty."""
    case = RC.frames(B)
    rows = [_compare(case, b) for b in range(B)]
    for b in range(B):
        if B >= 3 and b == 1:
            assert (case.h[1][1, :, 1] <= F32(0.5)).all() and len(rows[1]) == 0
            continue
        s = rows[b][:, 4]
        assert np.isinf(s[0]) and not np.isnan(s).any()
        assert (s == F32(0.2)).sum() <= 1


def test_negative_conf_ties():
    """Every prior is a candidate of both classes, and the cut at 1024 falls inside the +-0 tie; the oracle orders the
    tie by prior index."""
    case = RC.negative_conf()
    d = RO.postprocess(*[x[0] for x in case.h], **case.kw, max_det=2048)
    rows = d[1:1 + 6 * int(d[0])].reshape(-1, 6)
    s = case.h[3][0, :, 1] * np.where(case.h[1][0, :, 1] > F32(0.01), F32(1), F32(0))
    assert (s == 0).sum() > 1024 - (s > 0).sum() > 0
    assert _kept(rows).keys() == {1, 2}
