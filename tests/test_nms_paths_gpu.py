"""nms_kernel (tensorrtx_b200/csrc/nms.cu) on every path it can take, against the oracle's nms() bit for bit.

The kernel chooses its sort and suppression code from the data, and a release build cannot say which path ran.  So every
test here builds plugin-format rows directly and asserts the input property that routes them (`_route`):
  phase B  radix select of the top 2048 rows, ties at the cut by lower row: more than min(max_rows, 2048) rows pass
  phase C  (1) bucketed counting sort: integer class ids in [0, 1024), <= 256 rows per class
           (2) packed 64-bit bitonic sort in registers: integer ids in [0, 65535], M <= 1024
           (3) the same in shared memory: M in 1025..2048
           (4) generic 128-bit bitonic sort: two rows share (class, conf), or an id that is not an integer in [0, 65535]
  phase E  short (<= 32 rows), medium (33..96) and long (> 96) class segments; overlaps()'s division fallback
Every image is compared with oracle.nms of the same rows: count, keep_index == the oracle's source rows (order included),
rows as bits (NaN-aware), keep == 1, extras carried along, the tail zero and keep_index -1 past the count."""
import numpy as np
import pytest
import torch

from oracle import nms_cases as NC
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu

# variant (the oracle's): 0 v8 LTRB, 1 v5 CXCYWH, 2 RetinaFace (LTRB, +1e-6, one class), 3 v8 oriented boxes (ProbIoU)
FMT = {0: L.BOX_LTRB, 1: L.BOX_CXCYWH, 2: L.BOX_RETINA, 3: L.BOX_OBB}
ROW = {0: 8, 1: 8, 2: 15, 3: 90}                       # floats per plugin row
EXTRA = {0: (6, 2), 1: (6, 2), 2: (5, 10), 3: (89, 1)}  # (offset, count) of the floats carried into the output row
M_EDGES = (0, 1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _buf(images, variant, max_rows, seed=0, counts=None):
    """images[b] = (box [n, 4], conf [n], cls [n]) -> plugin buffer [B, 1 + max_rows*F] with seeded extras."""
    rng = np.random.default_rng(seed)
    F = ROW[variant]
    buf = np.zeros((len(images), 1 + max_rows * F), np.float32)
    for b, (box, conf, cls) in enumerate(images):
        n = len(conf)
        rows = buf[b, 1:1 + n * F].reshape(n, F)
        rows[:, 5:] = rng.uniform(-50, 700, (n, F - 5))
        if variant == 3:
            rows[:, 89] = rng.uniform(0, np.pi, n)
        rows[:, :4], rows[:, 4] = box, conf
        if variant != 2:
            rows[:, 5] = cls
        buf[b, 0] = n if counts is None else counts[b]
    return buf


def _run(dev, buf, variant, conf, thr, max_det=None, mode=L.NMS_GREEDY):
    t = torch.from_numpy(buf).to(dev)
    if variant == 3:
        comp, idx = P.batch_nms_obb(t, buf.shape[0], buf.shape[1], conf, thr, max_det=max_det, mode=mode, return_index=True)
    else:
        off, ne = EXTRA[variant]
        comp, idx = P.batch_nms(t, buf.shape[0], buf.shape[1], conf, thr, box_format=FMT[variant], det_floats=ROW[variant],
                                max_det=max_det, mode=mode, extra_floats=ne, extra_offset=off, return_index=True)
    torch.cuda.synchronize()
    return comp.cpu().numpy(), idx.cpu().numpy()


def _rows(img, variant, max_rows):
    F = ROW[variant]
    n = min(max(int(img[0]) if np.isfinite(img[0]) else 0, 0), max_rows)
    return img[1:1 + n * F].reshape(n, F)


def _expected(oracle, img, variant, conf, thr):
    """oracle.nms of one image.  NaN confidences: the library drops them (`!(conf > conf_thresh)`, as v8's nms() does);
    v5 / RetinaFace / nms_obb keep them and then sort with a comparator that is no strict weak order, so their result is
    undefined -- the oracle sees those rows with conf -inf, which no threshold keeps."""
    img = img.copy()
    F = ROW[variant]
    max_rows = (img.shape[0] - 1) // F
    if variant != 0:
        r = img[1:].reshape(max_rows, F)
        r[np.isnan(r[:, 4]), 4] = -np.inf
    return oracle.nms(variant, img, max_rows, F, conf, thr)


def _assert_image(comp_b, idx_b, res, src, variant, max_det, what=""):
    off, ne = EXTRA[variant]
    R = 7 + ne
    n = min(len(res), max_det)
    assert int(comp_b[0]) == n, (what, int(comp_b[0]), n)
    assert np.array_equal(idx_b[:n], src[:n]), what                    # same kept rows, same order
    rows = comp_b[1:1 + n * R].reshape(n, R)
    nc = 5 if variant == 2 else 6
    assert np.array_equal(_bits(rows[:, :nc]), _bits(res[:n, :nc])), what  # box, conf, class: copies of the source row
    if variant == 2:
        assert np.all(_bits(rows[:, 5]) == 0), what
    assert np.all(rows[:, 6] == 1), what
    assert np.array_equal(_bits(rows[:, 7:]), _bits(res[:n, off:off + ne])), what
    assert np.all(_bits(comp_b[1 + n * R:]) == 0) and np.all(idx_b[n:] == -1), what


def _check(oracle, buf, comp, idx, variant, conf, thr, max_det=None):
    max_det = max_det or (buf.shape[1] - 1) // ROW[variant]
    out = []
    for b in range(buf.shape[0]):
        res, src = _expected(oracle, buf[b], variant, conf, thr)
        _assert_image(comp[b], idx[b], res, src, variant, max_det, f"image {b}")
        out.append(len(res))
    return out


def _route(img, variant, conf, max_rows=None):
    """The paths nms_kernel takes for one image (<= 2048 rows above conf): (M, sort path, class segment lengths)."""
    F = ROW[variant]
    rows = _rows(img, variant, max_rows or (img.shape[0] - 1) // F)
    keep = rows[:, 4] > np.float32(conf)
    M = int(keep.sum())
    if M == 0:
        return 0, "empty", []
    cls = (rows[keep, 5] if variant != 2 else np.zeros(M, np.float32)).astype(np.float64) + 0.0   # -0.0 -> +0.0
    cf = rows[keep, 4].astype(np.float64) + 0.0
    _, seg = np.unique(cls, return_counts=True)
    packed = bool(np.all(np.isfinite(cls) & (cls >= 0) & (cls <= 65535) & (cls == np.floor(cls))))
    ties = len(set(zip(cls.tolist(), cf.tolist()))) < M
    if not packed or ties:
        path = "generic"
    elif cls.max() < 1024 and seg.max() <= 256:
        path = "bucketed"
    else:
        path = "packed-registers" if M <= 1024 else "packed-shared"
    return M, path, sorted(seg.tolist())


# ------------------------------------------------------------------ sort paths ----------------------------------------
SORT_CASES = [(v, r) for v in (0, 1, 2, 3) for r in ("bucketed", "wide", "ties") if not (v == 2 and r == "wide")]


@pytest.mark.parametrize("variant,route", SORT_CASES)
def test_sort_paths_at_their_edges(oracle, dev, variant, route):
    """One launch, one image per M in {0, 1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048}:
    bucketed: ids in [0, 80), distinct confidences -> path (1) (RetinaFace, one class: (1) up to 256 rows, then (2)/(3));
    wide: ids in [0, 1203] with id 1203 present -> path (2) for M <= 1024, (3) above;
    ties: fp16-quantised confidences and a forced (class, conf) tie -> path (4), where box[0] orders the tied rows of
    LTRB / OBB (yolov8's cmp) and the row index those of CXCYWH / RetinaFace."""
    rng = np.random.default_rng(1000 + 10 * variant + len(route))
    images = []
    for M in M_EDGES:
        if route == "ties":
            conf = np.float16(rng.uniform(0.3, 0.99, M)).astype(np.float32)
            if M >= 2:
                conf[1] = conf[0]
            cls = rng.integers(0, 80, M)
            if M >= 2:
                cls[1] = cls[0]
        else:
            conf = NC.distinct_conf(rng, M)
            cls = rng.integers(0, 80 if route == "bucketed" else 1204, M)
            if route == "wide" and M:
                cls[0] = 1203
        images.append(NC.random_rows(rng, variant, M, cls, conf))
    buf = _buf(images, variant, 2048, seed=variant)
    for b, M in enumerate(M_EDGES):
        m, path, _ = _route(buf[b], variant, 0.25)
        assert m == M
        if M == 0:
            want = "empty"
        elif route == "ties":
            want = "generic" if M >= 2 else "bucketed"
        elif route == "wide" or (variant == 2 and M > 256):
            want = "packed-registers" if M <= 1024 else "packed-shared"
        else:
            want = "bucketed"
        assert path == want, (M, path, want)
    comp, idx = _run(dev, buf, variant, 0.25, 0.45)
    kept = _check(oracle, buf, comp, idx, variant, 0.25, 0.45)
    assert kept[-1] > 50


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_class_of_256_and_257_rows(oracle, dev, variant):
    """A class of exactly 256 rows still takes the bucketed sort (1); one of 257 rows sends the image to the packed sort (2)
    (a long segment for phase E either way).  RetinaFace: the whole image is that class."""
    rng = np.random.default_rng(1100 + variant)
    images = []
    for big in (256, 257):
        n_other = 0 if variant == 2 else 400
        cls = np.concatenate([np.full(big, 7), rng.integers(8, 80, n_other)])
        images.append(NC.random_rows(rng, variant, big + n_other, cls, NC.distinct_conf(rng, big + n_other)))
    buf = _buf(images, variant, 1024, seed=variant)
    assert _route(buf[0], variant, 0.25)[1] == "bucketed" and max(_route(buf[0], variant, 0.25)[2]) == 256
    assert _route(buf[1], variant, 0.25)[1] == "packed-registers" and max(_route(buf[1], variant, 0.25)[2]) == 257
    comp, idx = _run(dev, buf, variant, 0.25, 0.45)
    _check(oracle, buf, comp, idx, variant, 0.25, 0.45)


@pytest.mark.parametrize("variant", [0, 1, 3])
def test_class_ids_at_the_sort_key_limits(oracle, dev, variant):
    """Integer ids around the packed keys' limits: 1023 (bucketed, 1), 1024 and 1203 (an LVIS-sized head; packed, 2),
    65535 (the largest id a packed key holds, 2) and 65536 (generic, 4)."""
    rng = np.random.default_rng(1200 + variant)
    ids = (1023, 1024, 1203, 65535, 65536)
    images = [NC.random_rows(rng, variant, 300, rng.choice([0, 3, 17, hi - 1, hi], 300), NC.distinct_conf(rng, 300)) for hi in ids]
    buf = _buf(images, variant, 300, seed=variant)
    paths = [_route(buf[b], variant, 0.25)[1] for b in range(len(ids))]
    assert paths == ["bucketed", "packed-registers", "packed-registers", "packed-registers", "generic"]
    comp, idx = _run(dev, buf, variant, 0.25, 0.45)
    _check(oracle, buf, comp, idx, variant, 0.25, 0.45)


# ------------------------------------------------------------------ class ids as floats --------------------------------
@pytest.mark.parametrize("variant", [0, 1, 3])
def test_class_ids_are_compared_as_floats(oracle, dev, variant):
    """Negative, signed-zero, fractional and huge class ids (path (4)): grouped and ordered as floats, and every row keeps
    its own class float -- a truncating int key sorts -1 last, merges 2.0 with 2.5 and 3e9 with 5e9, and emits -0.0 as 0.0."""
    rng = np.random.default_rng(1300 + variant)
    buf = _buf([NC.float_id_rows(rng, variant), NC.float_id_rows(rng, variant, 90)], variant, 240, seed=variant)
    assert all(_route(buf[b], variant, 0.25)[1] == "generic" for b in range(2))
    comp, idx = _run(dev, buf, variant, 0.25, 0.45)
    _check(oracle, buf, comp, idx, variant, 0.25, 0.45)
    n = int(comp[0, 0])
    cls = comp[0, 1:1 + n * 8 if variant == 3 else 1 + n * 9].reshape(n, -1)[:, 5]
    assert cls[0] == -3.0 and {2.0, 2.5} <= set(cls.tolist()) and np.signbit(cls).sum() > len(np.flatnonzero(cls < 0))


# ------------------------------------------------------------------ class segments ------------------------------------
def _chain_segment(m, cls, first_rank, rng, variant):
    """m rows of one class made of suppression chains on the integer grid: row k of a chain is [k, y, k + 4, y + 1], so it
    overlaps row k+1 with IoU 3/5 and row k+2 with IoU 1/3 -- greedy keeps every other row of a chain.  Chain lengths are
    random (1..40), so kept and suppressed rows fall on both sides of every 32-row chunk boundary; each chain has a y band of
    its own and the confidences fall strictly along the segment."""
    x1, y1, k, band = [], [], 0, 0
    while k < m:
        ln = min(int(rng.integers(1, 41)), m - k)
        x1 += list(range(ln))
        y1 += [2 * band] * ln
        k, band = k + ln, band + 1
    x1, y1 = np.asarray(x1, np.float64), np.asarray(y1, np.float64)
    conf = (0.99 - (first_rank + np.arange(m)) * 2.0 ** -14).astype(np.float32)
    return NC.boxes(variant, x1, y1, x1 + 4, y1 + 1), conf, np.full(m, cls, np.float32)


def _segments_image(rng, variant, lengths):
    parts, rank = [], 0
    for c, m in enumerate(lengths):
        parts.append(_chain_segment(m, 3 * c + 1, rank, rng, variant))
        rank += m
    box, conf, cls = (np.concatenate(p) for p in zip(*parts))
    perm = rng.permutation(len(conf))                # arrival order is arbitrary
    return box[perm], conf[perm], cls[perm]


SEGMENT_IMAGES = ([1, 2, 31, 32, 33, 64, 65, 95, 96, 97, 128, 1000], [2048], [97, 128, 200, 300, 500, 97, 33, 5])


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_class_segments_of_every_length(oracle, dev, variant):
    """Phase E: short (<= 32), medium (33..96, 2-3 chunks, scheduled first) and long (> 96, whole-CTA 32-row chunks against
    the kept list) class segments of 1, 2, 31, 32, 33, 64, 65, 95, 96, 97, 128, 1000 and 2048 rows, several long ones in one
    image.  RetinaFace has one class: one segment per image, of 33, 97, 1000 and 2048 rows."""
    rng = np.random.default_rng(1400 + variant)
    if variant == 2:
        images = [_segments_image(rng, variant, [m]) for m in (33, 97, 1000, 2048)]
        want = [[33], [97], [1000], [2048]]
    else:
        images = [_segments_image(rng, variant, s) for s in SEGMENT_IMAGES]
        want = [sorted(s) for s in SEGMENT_IMAGES]
    buf = _buf(images, variant, 2048, seed=variant)
    for b in range(len(images)):
        assert _route(buf[b], variant, 0.25)[2] == want[b]
    comp, idx = _run(dev, buf, variant, 0.25, 0.45 if variant != 2 else 0.4)
    kept = _check(oracle, buf, comp, idx, variant, 0.25, 0.45 if variant != 2 else 0.4)
    for b, k in enumerate(kept):
        assert sum(want[b]) // 2 <= k < sum(want[b])


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_max_det_below_the_kept_count(oracle, dev, variant):
    """max_det smaller than the kept count: the first max_det rows of the oracle's order, count = max_det."""
    rng = np.random.default_rng(1500 + variant)
    buf = _buf([_segments_image(rng, variant, [97, 128, 33] if variant != 2 else [300])], variant, 512, seed=variant)
    comp, idx = _run(dev, buf, variant, 0.25, 0.45, max_det=61)
    assert _check(oracle, buf, comp, idx, variant, 0.25, 0.45, max_det=61)[0] > 61


# ------------------------------------------------------------------ the threshold -------------------------------------
@pytest.mark.parametrize("variant,thr", [(v, t) for v in (0, 1, 2) for t in (0.45, 0.5, 0.4)])
def test_iou_exactly_at_and_ulps_around_the_threshold(oracle, dev, variant, thr):
    """Pairs whose float IoU is exactly fl(thr) (kept: `iou > thr` is false) and 1..3 ulps either side (nms_cases.
    threshold_rows), all inside |inter - thr*denom| <= 1e-5*denom, where overlaps() takes the IEEE division instead of its
    division-free sign test.  For thr 0.45 and 0.4 the pair at fl(thr) has its exact quotient above fl(thr): the sign of
    t = fma(-thr, denom, inter) says "overlaps" there and only the division keeps the row, so a kernel without the fallback
    fails here.  (For thr 0.5 no such pair exists: a float quotient that rounds to 0.5 is exactly 0.5.)  RetinaFace adds
    small boxes whose `+ 1e-6` in the denominator keeps a row that would be suppressed without it."""
    img, kept, sign_test_wrong = NC.threshold_rows(variant, thr)
    assert sign_test_wrong == (thr != 0.5)
    buf = _buf([img], variant, 64, seed=variant)
    comp, idx = _run(dev, buf, variant, 0.25, thr)
    assert _check(oracle, buf, comp, idx, variant, 0.25, thr)[0] == kept


@pytest.mark.parametrize("variant,thr", [(v, t) for v in (0, 1, 2) for t in (0.45, -0.25, 4.5)])
def test_degenerate_boxes_and_extreme_thresholds(oracle, dev, variant, thr):
    """Zero-area, inverted, 1e30, +-inf and NaN coordinates, with thr 0.45, thr < 0 (disjoint boxes overlap: zero_hit) and
    thr > 4 (no division-free test).  NaN coordinates: std::max / std::min ignore a NaN in the later row and propagate one
    in the kept row; overlaps() and the oracle take their operands in that order."""
    rng = np.random.default_rng(1600 + variant + int(10 * thr))
    buf = _buf([NC.degenerate_rows(rng, variant), NC.degenerate_rows(rng, variant, 64)], variant, 160, seed=variant)
    comp, idx = _run(dev, buf, variant, 0.25, thr)
    _check(oracle, buf, comp, idx, variant, 0.25, thr)


# ------------------------------------------------------------------ confidences ---------------------------------------
@pytest.mark.parametrize("variant,conf", [(v, c) for v in (0, 1, 2, 3) for c in (0.5, 0.0, -1.0)])
def test_confidence_edges(oracle, dev, variant, conf):
    """Confidences exactly at conf_thresh (dropped) and one ulp above (kept), +inf and -inf, subnormals and +-0.0 (kept
    only below a negative threshold, where they tie), and NaN (always dropped: see _expected)."""
    rng = np.random.default_rng(1700 + variant)
    n = 200
    t = np.float32(conf)
    special = np.array([t, np.nextafter(t, np.float32(np.inf)), np.inf, -np.inf, np.nan, 1e-45, 2e-40, 0.0, -0.0,
                        np.nextafter(t, np.float32(-np.inf))], np.float32)
    c = NC.distinct_conf(rng, n)
    c[:len(special) * 10] = np.repeat(special, 10)
    box, c, cls = NC.random_rows(rng, variant, n, rng.integers(0, 4, n), c)
    buf = _buf([(box, c, cls)], variant, n, seed=variant)
    comp, idx = _run(dev, buf, variant, float(t), 0.45)
    _check(oracle, buf, comp, idx, variant, float(t), 0.45)
    n_out = int(comp[0, 0])
    R = 7 + EXTRA[variant][1]
    assert not np.isnan(comp[0, 1:1 + n_out * R].reshape(n_out, R)[:, 4]).any()


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_radix_select_cut_inside_a_block_of_equal_confidences(oracle, dev, variant):
    """Phase B: 3000 rows pass conf_thresh (max_rows 3000 > 2048).  Ranks 1500..2499 all have confidence +0.0 or -0.0
    (one key), so the cut at rank 2048 falls inside that block and takes its 548 rows of lowest index.  Expected: the oracle
    on exactly the selected rows."""
    rng = np.random.default_rng(1800 + variant)
    n = 3000
    conf = np.empty(n, np.float32)
    perm = rng.permutation(n)
    hi, zero, lo = perm[:1500], perm[1500:2500], perm[2500:]
    conf[hi] = NC.distinct_conf(rng, 1500, 0.5, 0.99)
    conf[zero] = np.where(rng.integers(0, 2, 1000) == 1, np.float32(-0.0), np.float32(0.0))
    conf[lo] = -NC.distinct_conf(rng, 500, 0.1, 0.9)
    img = NC.random_rows(rng, variant, n, rng.integers(0, 80, n), conf)
    buf = _buf([img], variant, n, seed=variant)
    sel = np.sort(np.concatenate([hi, np.sort(zero)[:548]]))
    assert (conf > 0).sum() < 2048 < (conf >= 0).sum() and len(sel) == 2048
    assert np.signbit(conf[np.sort(zero)[:548]]).any() and not np.signbit(conf[np.sort(zero)[:548]]).all()
    F = ROW[variant]
    sub = np.zeros(1 + 2048 * F, np.float32)
    sub[0] = 2048
    sub[1:].reshape(2048, F)[:] = buf[0, 1:].reshape(n, F)[sel]
    res, src = _expected(oracle, sub, variant, -1.0, 0.45)
    comp, idx = _run(dev, buf, variant, -1.0, 0.45, max_det=2048)
    _assert_image(comp[0], idx[0], res, sel[src], variant, 2048)
    assert len(res) > 100


# ------------------------------------------------------------------ one launch, many paths ----------------------------
def test_mixed_batch_equals_single_images(oracle, dev):
    """One launch over images on different paths -- bucketed, packed in registers (id 1203), packed in shared memory,
    generic (ties), float class ids -- plus an empty image, a count above max_rows, a negative count and a NaN count.  Each
    image equals its own batch-1 call and the oracle."""
    rng = np.random.default_rng(1900)
    v = 0
    images, counts = [], []
    for n, hi, ties in ((300, 80, False), (600, 1204, False), (1500, 1204, False), (400, 80, True)):
        conf = np.float16(rng.uniform(0.3, 0.99, n)).astype(np.float32) if ties else NC.distinct_conf(rng, n)
        cls = rng.integers(0, hi, n)
        cls[:2] = hi - 1
        if ties:
            conf[1] = conf[0]
        images.append(NC.random_rows(rng, v, n, cls, conf))
        counts.append(n)
    images.append(NC.float_id_rows(rng, v))
    counts.append(240)
    for cnt in (0, 5000, -5, np.nan):
        images.append(NC.random_rows(rng, v, 2048, rng.integers(0, 80, 2048), NC.distinct_conf(rng, 2048)))
        counts.append(cnt)
    buf = _buf(images, v, 2048, seed=3, counts=counts)
    assert [_route(buf[b], v, 0.25)[1] for b in range(5)] == ["bucketed", "packed-registers", "packed-shared", "generic",
                                                            "generic"]
    comp, idx = _run(dev, buf, v, 0.25, 0.45)
    kept = _check(oracle, buf, comp, idx, v, 0.25, 0.45)
    assert kept[5] == kept[7] == kept[8] == 0 and kept[6] > 100
    for b in range(buf.shape[0]):
        c1, i1 = _run(dev, buf[b:b + 1].copy(), v, 0.25, 0.45)
        assert np.array_equal(_bits(c1[0]), _bits(comp[b])) and np.array_equal(i1[0], idx[b]), b


# ------------------------------------------------------------------ one-shot ------------------------------------------
def _oneshot_family(rng, variant, family):
    if family == "chains":
        return _segments_image(rng, variant, [1, 31, 33, 97, 200])
    if family == "ties":
        n = 500
        return NC.random_rows(rng, variant, n, rng.integers(0, 6, n), np.float16(rng.uniform(0.3, 0.99, n)).astype(np.float32))
    return NC.float_id_rows(rng, variant)


@pytest.mark.parametrize("variant,family", [(v, f) for v in (0, 1) for f in ("chains", "ties", "class_ids")])
def test_oneshot_mode_paths(oracle, dev, variant, family):
    """One-shot mode (the reference's decode_kernel + nms_kernel): a row is dropped when any same-class row before it
    overlaps it.  The reference orders equal confidences by its atomicAdd slot -- the HIGHER slot wins -- while the kernel
    puts them in (box[0], row) order (LTRB; row order for CXCYWH) and lets the EARLIER row win.  The rows permuted into
    descending (box[0], row) order therefore put them in the slots whose reference outcome the kernel's choice is, so the
    keep flags are compared with oracle.cuda_decode_nms of that permutation."""
    rng = np.random.default_rng(2000 + 10 * variant + len(family))
    box, conf, cls = _oneshot_family(rng, variant, family)
    buf = _buf([(box, conf, cls)], variant, len(conf), seed=variant)
    n_in = len(conf)
    F = ROW[variant]
    rows = buf[0, 1:].reshape(n_in, F)
    rid = np.arange(n_in)
    perm = np.lexsort((-rid, -(rows[:, 0] + 0.0))) if variant == 0 else rid[::-1]
    pbuf = np.zeros_like(buf[0])
    pbuf[0] = n_in
    pbuf[1:].reshape(n_in, F)[:] = rows[perm]
    exp = oracle.cuda_decode_nms(pbuf, n_in, F, 0.25, 0.45, n_in)[1:].reshape(n_in, 7)
    comp, idx = _run(dev, buf, variant, 0.25, 0.45, mode=L.NMS_ONESHOT)
    n = int(comp[0, 0])
    R = 7 + EXTRA[variant][1]
    got = comp[0, 1:1 + n * R].reshape(n, R)
    slot = np.empty(n_in, np.int64)
    slot[perm] = np.arange(n_in)
    assert n == int((conf >= np.float32(0.25)).sum()) and set(idx[0, :n].tolist()) == set(rid[conf >= np.float32(0.25)].tolist())
    assert np.array_equal(_bits(got[:, :7]), _bits(exp[slot[idx[0, :n]]]))      # rows and keep flags, bit for bit
    assert 0 < got[:, 6].sum() and (variant != 0 or got[:, 6].sum() < n)   # (one-shot reads CXCYWH rows as corners)
    # rows in the header's order: class asc (as floats), conf desc, then box[0] (LTRB) and row
    key = (rid, rows[:, 0] + 0.0 if variant == 0 else np.zeros(n_in), -(conf + 0.0), cls.astype(np.float64) + 0.0)
    order = np.lexsort(key)
    assert np.array_equal(idx[0, :n], order[np.isin(order, idx[0, :n])])


# ------------------------------------------------------------------ fused decode + NMS --------------------------------
def _fused_vs_two_stage_vs_oracle(oracle, dev, heads, nc, max_out, conf):
    B = heads[0].shape[0]
    hd = [torch.from_numpy(h).to(dev).contiguous() for h in heads]
    plug = P.YoloLayerPlugin(nc, 17, 0.0, 640, 640, max_out, False, False, False, (8, 16, 32))
    fused = P.FusedYoloDecodeNms(plug, B, conf, 0.45, device=dev)
    comp, idx = fused.enqueue(B, hd)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    two = P.batch_nms(out, B, plug.output_elems(), conf, 0.45, max_det=max_out).cpu().numpy()
    assert np.array_equal(_bits(two), _bits(comp))
    ref, ref_idx = oracle.yolov8_decode(heads, nc=nc, max_out=max_out)
    for b in range(B):
        one = ref[b].copy()
        one[0] = min(one[0], max_out)
        res, src = oracle.nms(0, one, max_out, 90, conf, 0.45)
        n = int(comp[b, 0])
        assert n == len(res) and n > 20
        assert np.array_equal(idx[b, :n], ref_idx[b][src])
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=1e-4, rtol=0)
    return ref


def test_fused_lvis_sized_head(oracle, dev):
    """nc = 1203 through FusedYoloDecodeNms: candidates with class ids >= 1024 send every image to the packed sort (2)."""
    heads = synth.yolov8_heads(2, seed=212, nc=1203)
    ref = _fused_vs_two_stage_vs_oracle(oracle, dev, heads, 1203, 1000, 0.5)
    for b in range(2):
        rows = ref[b, 1:1 + min(int(ref[b, 0]), 1000) * 90].reshape(-1, 90)
        assert (rows[rows[:, 4] > 0.5, 5] >= 1024).any()


def test_fused_more_than_1024_candidates(oracle, dev):
    """max_out = 2000 on dense heads: more than 1024 candidates enter the NMS, whose row capacity S is then 2048."""
    heads = synth.yolov8_heads(2, seed=211, n_obj=300)
    ref = _fused_vs_two_stage_vs_oracle(oracle, dev, heads, 80, 2000, 0.5)
    for b in range(2):
        rows = ref[b, 1:1 + 2000 * 90].reshape(2000, 90)
        assert ref[b, 0] > 2000 and (rows[:, 4] > 0.5).sum() > 1024
