"""Top-k selection and sort order of the Faster R-CNN plugins (RpnDecode, PredictorDecode, RpnNms, BatchedNms) where scores
tie, and the YOLO NMS's `bbox[0]` tie-break on signed zeros.

Each plugin must give the prefix of a STABLE descending sort in which -0.0 and +0.0 are one key, as cub's radix sort in the
reference and the CPU oracle's comparison sort do: equal scores keep ascending input index.  Continuous random scores
almost never tie, so every case here feeds score families in which ties decide the result, varied per image of a batch:
  fp16     an FP16 engine's scores widened to float: a few dozen distinct values, the cut inside a block of > 1024 ties;
  equal    every score the same: the output is indices 0 .. k-1 in order;
  zeros    a block of zeros straddling the cut, -0.0 and +0.0 interleaved by index;
  special  as `zeros`, plus +-inf, +-FLT_MAX and subnormals of both signs.
Deltas are zero (the decodes place each anchor / proposal as is), so every (cell, anchor) or (box, class) has its own,
bit-exact box and a wrong order shows up as a box mismatch; one case per decode keeps random deltas.  Scores are compared
by bit pattern.  Every output is checked against the CPU oracle bit for bit and, where oracle/_ref was built, against the
reference's own functions (elsewhere against tests/golden/ref_rcnn_sort_gpu.npz, oracle/golden.py).  The reference's
RpnNms and BatchedNms are called once per image (their batch > 1 bug, DESIGN.md) and only up to 1024 boxes: above that
their kernels race across blocks, and the larger cases are checked against the oracle alone.  Rows the reference leaves
untouched must keep what the caller put there."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_rcnn_sort_gpu")

FMAX = np.float32(np.finfo(np.float32).max)
SENT = -7.25                     # what an output the plugin must not write keeps
IMG_H, IMG_W, STRIDE = 800, 1067, 16.0
REF_MAX = 1024                   # the reference's RpnNms / BatchedNms are race-free up to one block of boxes
FAMILIES = ("fp16", "equal", "zeros", "special")
SPECIALS = (np.inf, -np.inf, FMAX, -FMAX, 1e-45, -1e-45, 3e-39, -3e-39)   # the last four are subnormal


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _same(what, got, exp):
    g, e = _bits(got), _bits(exp)
    assert g.shape == e.shape, (what, g.shape, e.shape)
    bad = np.argwhere(g != e)
    assert not len(bad), f"{what}: {len(bad)} elements differ, first at {bad[:4].tolist()}"


def _np(t):
    return None if t is None else t.cpu().numpy()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _sent(shape, dev):
    return torch.full(shape, SENT, dtype=torch.float32, device=dev)


def _ws(dev):
    return torch.empty(256, dtype=torch.uint8, device=dev)


def _fp16(x):
    return np.asarray(x, np.float16).astype(np.float32)


def _signed_zeros(s):
    """every zero of s gets the sign of its index's parity (odd: -0.0)"""
    odd = (np.arange(s.size) % 2 == 1).reshape(s.shape)
    return np.where(s == 0, np.where(odd, np.float32(-0.0), np.float32(0.0)), s).astype(np.float32)


def _with_specials(s, rng):
    s = s.copy()
    flat = s.reshape(-1)
    m = max(flat.size // 64, 1)
    pick = rng.permutation(flat.size)
    for j, v in enumerate(SPECIALS):
        flat[pick[j * m:(j + 1) * m]] = np.float32(v)
    return s


def rpn_scores(family, n, k, rng):
    """n RPN logits of one family, k = how many the plugin keeps"""
    if family == "equal":
        return np.full(n, 0.75, np.float32)
    s = _fp16(np.round(rng.standard_normal(n) * 4) / 2)          # N(0, 2) on a 0.5 grid
    if family == "fp16":
        return s
    s = _signed_zeros(s - np.sort(s)[::-1][k - 1])                # the k-th largest becomes 0: zeros at the cut
    return _with_specials(s, rng) if family == "special" else s


def class_probs(family, N, Cc, k, rng):
    """[N, Cc] class probabilities of one family (softmax over Cc + background, as the predictor head gives them)"""
    if family == "equal":
        return np.full((N, Cc), 0.25, np.float32)
    if family == "late":
        # the ties at the cut lie on both sides of index 65536 and the cut itself above it: the index select's
        # upper-byte pass has two buckets to choose from and must take the second
        s = np.full(N * Cc, 0.125, np.float32)
        s[:65536] = np.where(rng.random(65536) < 0.005, 0.125, 0.0625)
        return s.reshape(N, Cc)
    z = rng.standard_normal((N, Cc + 1)) * 3.0
    p = np.exp(z - z.max(-1, keepdims=True))
    p = (p / p.sum(-1, keepdims=True))[:, :Cc]
    s = _fp16(np.round(p * (4 if family == "fp16" else 2)) / (4 if family == "fp16" else 2))
    if family == "fp16":
        return s
    # zeros / special: probabilities that round to 0 (softmax underflow), fewer than k nonzero -> a zero block at the cut
    s = _signed_zeros(s)
    return _with_specials(s, rng) if family == "special" else s


def _tie_block_at_cut(s, k):
    """size of the block of equal scores the k-th largest belongs to, asserting that the cut falls strictly inside it"""
    f = s.reshape(-1).astype(np.float64) + 0.0                    # -0.0 == 0.0
    v = np.sort(f)[::-1][k - 1]
    above, tied = int((f > v).sum()), int((f == v).sum())
    assert above < k < above + tied, (above, tied, k)
    return tied, np.flatnonzero(f == v)


def anchors64():
    """64 anchors: 8 sizes x 8 aspect ratios, anchor a offset by (a / 4, a / 8) from its cell's corner, so that on a grid
    of up to 40 x 20 cells no box is clipped and no two (cell, anchor) pairs share a box"""
    res = []
    for size in (16, 24, 32, 48, 64, 96, 128, 192):
        for ar in (0.25, 0.4, 0.5, 0.75, 1.0, 1.5, 2.0, 3.0):
            w, h = np.float32(size / np.sqrt(ar)), np.float32(size * np.sqrt(ar))
            ox, oy = np.float32(len(res) / 16), np.float32(len(res) / 32)
            res += [ox, oy, ox + w, oy + h]
    return np.asarray(res, np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# RpnDecode
# ---------------------------------------------------------------------------------------------------------------------
def _rpn_decode(key, scores, deltas, H, W, top_n, dev, exact=True):
    B, A = scores.shape[:2]
    lib = G.lib("libref_rcnn.so")
    anchors = anchors64()[:4 * A]
    sd, dd = torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)
    os_, ob = _sent((B, top_n), dev), _sent((B, top_n, 4), dev)
    assert P.RpnDecodePlugin(top_n, anchors, STRIDE, IMG_H, IMG_W, H, W).enqueue(B, [sd, dd], [os_, ob], _ws(dev)) == 0
    rs = rb = None
    if lib is not None:
        rs, rb = _sent((B, top_n), dev), _sent((B, top_n, 4), dev)
        assert lib.ref_rpn_decode(B, _p(sd), _p(dd), _p(rs), _p(rb), H, W, IMG_H, IMG_W, C.c_float(STRIDE),
                                  anchors.ctypes.data_as(C.c_void_p), A, top_n) == 0
    from oracle import oracle as O
    es, eb = O.rpn_decode(scores, deltas, IMG_H, IMG_W, STRIDE, anchors, top_n)
    gs, gb = _np(os_), _np(ob)
    _same(f"{key}.scores vs oracle", gs, es)
    G.equal(f"{key}.scores", _bits(gs), None if rs is None else _bits(_np(rs)))
    if exact:
        _same(f"{key}.boxes vs oracle", gb, eb)
        G.equal(f"{key}.boxes", _bits(gb), None if rb is None else _bits(_np(rb)))
    else:   # glibc vs CUDA expf, and the reference build's FMA contraction
        np.testing.assert_allclose(gb, eb, rtol=2e-6, atol=1e-4)
        G.close(f"{key}.boxes", gb, _np(rb), rtol=3e-7, atol=1e-4)
    return gs, gb


@pytest.mark.parametrize("top_n", [1, 31, 6000, 8192])
def test_rpn_decode_ties(dev, top_n):
    """64 anchors x 20 x 40 cells = 51 200 scores, batch 3, the families rotating over the images"""
    A, H, W = 64, 20, 40
    n = A * H * W
    rng = np.random.default_rng(1000 + top_n)
    fams = [FAMILIES[(b + top_n) % 4] for b in range(3)]
    scores = np.stack([rpn_scores(f, n, top_n, rng) for f in fams]).reshape(3, A, H, W)
    for f, s in zip(fams, scores):
        if f == "equal" or (top_n >= 6000 and f in ("fp16", "zeros")):
            assert _tie_block_at_cut(s, top_n)[0] > 1024, f
    gs, gb = _rpn_decode(f"rpn_decode.{top_n}", scores, np.zeros((3, 4 * A, H, W), np.float32), H, W, top_n, dev)
    for b, f in enumerate(fams):
        assert len(np.unique(gb[b], axis=0)) == top_n        # every kept entry has its own box: the order is visible


@pytest.mark.parametrize("H,W,top_n", [(8, 16, 8192), (4, 8, 2047), (8, 16, 8191)])
def test_rpn_decode_at_and_past_top_n(dev, H, W, top_n):
    """n == top_n (no sort: every entry in index order) and n == top_n + 1 (a select that drops exactly one)"""
    A = 64
    n = A * H * W
    rng = np.random.default_rng(1100 + top_n)
    scores = np.stack([rpn_scores(f, n, min(top_n, n - 1), rng) for f in ("zeros", "special", "fp16")]).reshape(3, A, H, W)
    _rpn_decode(f"rpn_decode_n.{n}.{top_n}", scores, np.zeros((3, 4 * A, H, W), np.float32), H, W, top_n, dev)


def test_rpn_decode_random_deltas(dev):
    A, H, W, top_n = 64, 20, 40, 6000
    rng = np.random.default_rng(1200)
    scores = np.stack([rpn_scores(f, A * H * W, top_n, rng) for f in ("fp16", "zeros")]).reshape(2, A, H, W)
    deltas = (rng.standard_normal((2, 4 * A, H, W)) * 0.3).astype(np.float32)
    _rpn_decode("rpn_decode_deltas", scores, deltas, H, W, top_n, dev, exact=False)


# ---------------------------------------------------------------------------------------------------------------------
# PredictorDecode
# ---------------------------------------------------------------------------------------------------------------------
def _proposals(B, N, rng):
    x1 = rng.integers(0, 900, (B, N)); y1 = rng.integers(0, 650, (B, N))
    w = rng.integers(8, 300, (B, N)); h = rng.integers(8, 300, (B, N))
    return np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)


def _predictor_decode(key, scores, deltas, props, dev, exact=True):
    B, N, Cc = scores.shape
    lib = G.lib("libref_rcnn.so")
    w4 = (10.0, 10.0, 5.0, 5.0)
    sd, dd, pd = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (scores, deltas, props))
    o = [_sent((B, N), dev), _sent((B, N, 4), dev), _sent((B, N), dev)]
    assert P.PredictorDecodePlugin(N, IMG_H, IMG_W, w4, Cc).enqueue(B, [sd, dd, pd], o, _ws(dev)) == 0
    r = [None] * 3
    if lib is not None:
        r = [_sent((B, N), dev), _sent((B, N, 4), dev), _sent((B, N), dev)]
        assert lib.ref_predictor_decode(B, _p(sd), _p(dd), _p(pd), *map(_p, r), N, Cc, IMG_H, IMG_W, (C.c_float * 4)(*w4)) == 0
    from oracle import oracle as O
    e = O.predictor_decode(scores, deltas, props, IMG_H, IMG_W, np.asarray(w4, np.float32))
    g = [_np(t) for t in o]
    for name, gi, ei, ri in zip(("scores", "boxes", "classes"), g, e, r):
        if name == "boxes" and not exact:
            np.testing.assert_allclose(gi, ei, rtol=2e-6, atol=1e-4)
            G.close(f"{key}.boxes", gi, _np(ri), rtol=3e-7, atol=1e-4)
            continue
        _same(f"{key}.{name} vs oracle", gi, ei)
        G.equal(f"{key}.{name}", _bits(gi), None if ri is None else _bits(_np(ri)))
    return g


@pytest.mark.parametrize("N,Cc,fams", [
    (1000, 80, ("fp16", "zeros", "late")),     # 80 000 scores > 65 536: the index select uses three bytes
    (8192, 10, ("fp16", "equal", "special")),  # the 8192-key limit, 81 920 scores
    (3000, 1, FAMILIES),                       # one class: nothing to select, all n sorted
])
def test_predictor_decode_ties(dev, N, Cc, fams):
    rng = np.random.default_rng(2000 + N + Cc)
    k = N
    scores = np.stack([class_probs(f, N, Cc, k, rng) for f in fams])
    n = N * Cc
    for f, s in zip(fams, scores):
        if n > k and f in ("fp16", "late", "zeros", "equal"):
            tied, where = _tie_block_at_cut(s, k)
            assert tied > 1024, (f, tied)
            if n > 65536:
                assert where.min() < 65536 <= where.max(), f
        if f == "zeros" and n > k:
            assert (s.reshape(-1) > 0).sum() < k                  # the cut lies in the block of zeros
        if f == "late":
            f64 = s.reshape(-1)
            assert np.flatnonzero(f64 == f64.max())[k - 1] >= 65536
    g = _predictor_decode(f"predictor.{N}.{Cc}", scores, np.zeros((len(fams), n, 4), np.float32),
                          _proposals(len(fams), N, rng), dev)
    for b, f in enumerate(fams):
        if f == "equal":
            assert np.array_equal(g[2][b], np.arange(N) % Cc)     # indices 0 .. N-1 in order


def test_predictor_decode_random_deltas(dev):
    N, Cc = 1000, 80
    rng = np.random.default_rng(2100)
    scores = np.stack([class_probs(f, N, Cc, N, rng) for f in ("fp16", "zeros")])
    deltas = (rng.standard_normal((2, N * Cc, 4)) * 0.5).astype(np.float32)
    _predictor_decode("predictor_deltas", scores, deltas, _proposals(2, N, rng), dev, exact=False)


# ---------------------------------------------------------------------------------------------------------------------
# RpnNms
# ---------------------------------------------------------------------------------------------------------------------
def _boxes(kind, B, n, rng):
    """integer corners (every IoU the same float on every side); distinct boxes per image"""
    if kind == "near_same":      # every pair overlaps with IoU > 0.9: one box survives, the rest is the tail
        x2 = 100000 + np.arange(n)
        b = np.stack([np.zeros(n), np.zeros(n), x2, np.full(n, 1000)], -1)
        return np.broadcast_to(b, (B, n, 4)).astype(np.float32).copy()
    if kind == "zero_area":      # half the boxes have zero width: IoU 0/0 with each other, which never suppresses
        b = _boxes("random", B, n, rng)
        z = rng.random((B, n)) < 0.5
        b[..., 2] = np.where(z, b[..., 0], b[..., 2])
        return b
    x1 = rng.integers(0, 700, (B, n)); y1 = rng.integers(0, 500, (B, n))
    w = rng.integers(4, 160, (B, n)); h = rng.integers(4, 160, (B, n))
    if kind == "cluster":        # 6 groups of ~100 x 80 boxes a few pixels apart (IoU > 0.75): most are suppressed
        g, u = rng.integers(0, 6, (B, n)), np.arange(n)
        x1, y1 = g * 150 + u % 8, g * 90 + (u // 8) % 8
        w, h = 100 + (u // 64) % 8, 80 + u // 512
    return np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)


def _distinct(b):
    return all(len(np.unique(x, axis=0)) == len(x) for x in b)


@pytest.mark.parametrize("pre,post,kind", [
    (1, 1, "random"), (1, 5, "random"), (31, 31, "random"), (31, 50, "random"), (33, 1, "random"), (33, 20, "random"),
    (1000, 300, "random"), (1000, 1, "random"), (1000, 1017, "random"), (1000, 1000, "near_same"),
    (1000, 600, "zero_area"), (8192, 1000, "random"), (8192, 1, "random"), (8192, 4000, "near_same"),
])
def test_rpn_nms_ties(dev, pre, post, kind):
    B = 4
    rng = np.random.default_rng(3000 + pre + post)
    scores = np.stack([rpn_scores(f, pre, max(1, min(post, pre)), rng) for f in FAMILIES])
    boxes = _boxes(kind, B, pre, rng)
    assert _distinct(boxes)
    thr = 0.7
    sd, bd = torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev)
    ob = _sent((B, post, 4), dev)
    assert P.RpnNmsPlugin(thr, post, pre).enqueue(B, [sd, bd], [ob], _ws(dev)) == 0
    got = _np(ob)
    from oracle import oracle as O
    exp = O.rpn_nms(scores, boxes, post, thr)
    n_out = min(post, pre)
    _same("rpn_nms vs oracle", got[:, :n_out], exp[:, :n_out])
    assert np.all(_bits(got[:, n_out:]) == _bits(np.float32(SENT)))
    key = f"rpn_nms.{pre}.{post}.{kind}"
    if pre <= REF_MAX:
        lib = G.lib("libref_rcnn.so")
        ref = None
        if lib is not None:
            rb = _sent((B, post, 4), dev)
            for b in range(B):
                assert lib.ref_rpn_nms(1, _p(sd[b]), _p(bd[b]), _p(rb[b]), pre, post, C.c_float(thr)) == 0
            ref = _bits(_np(rb))
        G.equal(key, _bits(got), ref)
    if kind == "near_same":   # one survivor per image, then every other box in first-sort order
        for b in range(B):
            order = np.lexsort((np.arange(pre), -(scores[b].astype(np.float64) + 0.0)))
            alive = order[scores[b][order] > -FMAX]
            tail = [i for i in order if i != alive[0]]
            assert np.array_equal(got[b, :n_out], boxes[b][[alive[0]] + tail][:n_out])


# ---------------------------------------------------------------------------------------------------------------------
# BatchedNms
# ---------------------------------------------------------------------------------------------------------------------
def _classes(B, n, rng):
    """float class ids, many of them non-integer: the plugin compares (int) truncations and outputs the floats"""
    return (rng.integers(0, 3, (B, n)) + rng.choice(np.float32([0.0, 0.25, 0.5, 0.999]), (B, n))).astype(np.float32)


@pytest.mark.parametrize("method", [0, 1, 2])
@pytest.mark.parametrize("count,dets,kind", [
    (33, 50, "random"), (33, 10, "random"), (33, 40, "cluster"), (1000, 100, "random"), (1000, 1000, "cluster"), (1000, 1200, "random"),
    (1025, 300, "random"), (4095, 100, "random"), (4096, 4096, "cluster"), (4096, 5000, "random"),
])
def test_batched_nms_ties(dev, method, count, dets, kind):
    B = 4
    rng = np.random.default_rng(4000 + count + dets + method)
    scores = np.stack([rpn_scores(f, count, max(1, min(dets, count)), rng) for f in FAMILIES])
    scores[0] = np.abs(scores[0])                 # fp16 family: all suppressors, many ties
    boxes = _boxes(kind, B, count, rng)
    assert _distinct(boxes)
    classes = _classes(B, count, rng)
    thr = 0.5
    sd, bd, cd = (torch.from_numpy(x).to(dev) for x in (scores, boxes, classes))
    o = [_sent((B, dets), dev), _sent((B, dets, 4), dev), _sent((B, dets), dev)]
    assert P.BatchedNmsPlugin(method, thr, dets, count).enqueue(B, [sd, bd, cd], o, _ws(dev)) == 0
    gs, gb, gc = (_np(t) for t in o)
    from oracle import oracle as O
    es, eb, ec = O.batched_nms(method, scores, boxes, classes, dets, thr)
    n_out = min(dets, count)
    if method == 2:   # glibc vs CUDA expf (<= 2 ulp) in each of up to dozens of gaussian decays of one score
        np.testing.assert_allclose(gs, es, rtol=1e-5, atol=3e-45)
        _same("batched_nms zero scores vs oracle", gs == 0, es == 0)
    else:
        _same("batched_nms scores vs oracle", gs, es)
    _same("batched_nms boxes vs oracle", gb[:, :n_out], eb[:, :n_out])
    _same("batched_nms classes vs oracle", gc[:, :n_out], ec[:, :n_out])
    assert np.all(_bits(gb[:, n_out:]) == _bits(np.float32(SENT))) and np.all(_bits(gc[:, n_out:]) == _bits(np.float32(SENT)))
    if kind == "cluster" and method == 0:
        assert ((gs[:, :n_out] > 0).sum(1) < n_out).all()      # fewer survivors than outputs: a zero-score tail
    key = f"batched_nms.{method}.{count}.{dets}.{kind}"
    if count <= REF_MAX:
        lib = G.lib("libref_rcnn.so")
        r = [None] * 3
        if lib is not None:
            rt = [_sent((B, dets), dev), _sent((B, dets, 4), dev), _sent((B, dets), dev)]
            for b in range(B):
                assert lib.ref_batched_nms(method, 1, _p(sd[b]), _p(bd[b]), _p(cd[b]), *(_p(t[b]) for t in rt), count, dets,
                                           C.c_float(thr)) == 0
            r = [_bits(_np(t)) for t in rt]
        for name, g, ri in zip(("scores", "boxes", "classes"), (gs, gb, gc), r):
            G.equal(f"{key}.{name}", _bits(g), ri)


# ---------------------------------------------------------------------------------------------------------------------
# YOLO NMS: equal class and conf, x0 = +0.0 at the lower row and -0.0 at the higher
# ---------------------------------------------------------------------------------------------------------------------
def test_yolo_nms_signed_zero_x0(dev, oracle):
    F, max_rows = 90, 1000
    buf = np.zeros((1, 1 + max_rows * F), np.float32)
    rows = buf[0, 1:].reshape(max_rows, F)
    rows[0, :6] = [0.0, 10, 100, 110, 0.9, 3]
    rows[1, :6] = [-0.0, 12, 100, 111, 0.9, 3]         # IoU > 0.45 with row 0: the first of the two in sort order is kept
    rows[2, :6] = [0.0, 200, 50, 260, 0.8, 3]
    rows[3, :6] = [-0.0, 201, 50, 262, 0.8, 5]         # another class: kept as well
    rows[4, :6] = [-0.0, 400, 50, 460, 0.7, 7]
    rows[5, :6] = [0.0, 401, 50, 461, 0.7, 7]          # -0.0 at the lower row this time
    buf[0, 0] = 6
    comp, idx = P.batch_nms(torch.from_numpy(buf).to(dev), 1, buf.shape[1], 0.5, 0.45, box_format=L.BOX_LTRB, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    res, src = oracle.nms(0, buf[0], max_rows, F, 0.5, 0.45)
    n = int(comp[0, 0])
    assert n == len(res) == 4 and list(src) == [0, 2, 3, 4]
    assert np.array_equal(idx[0, :n], src)
    _same("yolo nms rows", comp[0, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6])


# ---------------------------------------------------------------------------------------------------------------------
# arguments past the limits
# ---------------------------------------------------------------------------------------------------------------------
def test_out_of_range_arguments_write_nothing(dev):
    lib = L.load()
    ws = _ws(dev)
    nws = C.c_size_t(ws.numel())
    big = torch.zeros(8 * 8193 * 8, dtype=torch.float32, device=dev)
    outs = [_sent((8 * 8193 * 4,), dev) for _ in range(3)]

    def untouched():
        torch.cuda.synchronize()
        return all(bool((t == SENT).all()) for t in outs)

    anc = (C.c_float * (65 * 4))(*np.concatenate([anchors64(), anchors64()[:4]]))
    o0, o1, o2 = (_p(t) for t in outs)
    rc = lib.trtx_rpn_decode(1, _p(big), _p(big), o0, o1, 2, 2, IMG_H, IMG_W, C.c_float(STRIDE), anc, 65, 100, _p(ws), nws, None)
    assert rc == -L.ERR_UNSUPPORTED and untouched()
    rc = lib.trtx_rpn_decode(1, _p(big), _p(big), o0, o1, 2, 2, IMG_H, IMG_W, C.c_float(STRIDE), anc, 64, 8193, _p(ws), nws, None)
    assert rc == -L.ERR_UNSUPPORTED and untouched()
    rc = lib.trtx_rpn_nms(1, _p(big), _p(big), o0, 8193, 100, C.c_float(0.7), _p(ws), nws, None)
    assert rc == -L.ERR_UNSUPPORTED and untouched()
    rc = lib.trtx_predictor_decode(1, _p(big), _p(big), _p(big), o0, o1, o2, 8193, 1, IMG_H, IMG_W,
                                   (C.c_float * 4)(10, 10, 5, 5), _p(ws), nws, None)
    assert rc == -L.ERR_UNSUPPORTED and untouched()
    rc = lib.trtx_batched_nms(0, 1, _p(big), _p(big), _p(big), o0, o1, o2, 4097, 100, C.c_float(0.5), _p(ws), nws, None)
    assert rc == -L.ERR_UNSUPPORTED and untouched()
    # at the limits the same calls run
    for rc in (lib.trtx_rpn_nms(1, _p(big), _p(big), o0, 8192, 100, C.c_float(0.7), _p(ws), nws, None),
               lib.trtx_batched_nms(0, 1, _p(big), _p(big), _p(big), o0, o1, o2, 4096, 100, C.c_float(0.5), _p(ws), nws, None)):
        assert rc == 0
    torch.cuda.synchronize()
