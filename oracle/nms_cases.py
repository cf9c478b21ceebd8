"""Inputs of the NMS edge tests, shared by tests/test_nms_paths_gpu.py (the kernel against the oracle) and
tests/test_nms_edges_cpu.py (the oracle against the reference's own host code), so that both pin the same cases.

TEST INFRASTRUCTURE ONLY.  Every builder returns (box [n, 4], conf [n], cls [n]) as float32, the box in the variant's
format.  Variants are the oracle's: 0 v8 LTRB, 1 v5 CXCYWH, 2 RetinaFace (LTRB, `+ 1e-6` in the denominator), 3 oriented."""
from __future__ import annotations

import numpy as np

F32 = np.float32
EPS_RETINA = F32(1e-6)
FLOAT_IDS = (-1.0, -3.0, -0.0, 0.0, 2.0, 2.5, 1e9, 3e9, 5e9)


def boxes(variant, x1, y1, x2, y2):
    """Corners -> the variant's four box floats (CXCYWH and oriented: cx, cy, w, h)."""
    x1, y1, x2, y2 = (np.asarray(v, np.float64) for v in (x1, y1, x2, y2))
    if variant in (1, 3):
        return np.stack([(x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1], 1).astype(F32)
    return np.stack([x1, y1, x2, y2], 1).astype(F32)


def distinct_conf(rng, n, lo=0.3, hi=0.99):
    return (lo + (hi - lo) * (rng.permutation(n) + 1) / (n + 1)).astype(F32)


def random_rows(rng, variant, n, classes, conf):
    """n boxes in 16 clusters (so that many overlap), with the given class ids and confidences."""
    centres = rng.uniform(60, 580, (16, 2))
    c = centres[rng.integers(0, 16, n)] + rng.normal(0, 12, (n, 2))
    wh = rng.uniform(20, 110, (n, 2))
    return boxes(variant, c[:, 0] - wh[:, 0] / 2, c[:, 1] - wh[:, 1] / 2, c[:, 0] + wh[:, 0] / 2, c[:, 1] + wh[:, 1] / 2), \
        np.asarray(conf, F32), np.asarray(classes, F32)


def float_id_rows(rng, variant, n=240):
    """Class ids FLOAT_IDS in turn: negative, both zeros, 2.0 next to 2.5 on the same boxes, 1e9 and ids past 2^31.  The
    reference groups them with std::map<float, ...>: -3 < -1 < 0 (-0.0 == +0.0) < 2 < 2.5 < 1e9 < 3e9 < 5e9."""
    box, conf, _ = random_rows(rng, variant, n, np.zeros(n), distinct_conf(rng, n))
    cls = np.asarray(FLOAT_IDS, F32)[np.arange(n) % len(FLOAT_IDS)]
    i2, i25 = np.flatnonzero(cls == 2.0), np.flatnonzero(cls == 2.5)
    k = min(len(i2), len(i25))
    box[i25[:k]] = box[i2[:k]]                      # 2.5 rows sit exactly on 2.0 rows: they must not suppress each other
    conf[i25[:k]] = conf[i2[:k]] - F32(1e-3)
    return box, conf, cls


def degenerate_rows(rng, variant, n=160):
    """Normal boxes mixed with zero-area ones (every other one on the point (100, 100): IoU 0/0), inverted ones (x2 < x1;
    CXCYWH w < 0), 1e30 coordinates (the intersection overflows), +inf and -inf coordinates and a NaN in one coordinate."""
    box, conf, cls = random_rows(rng, variant, n, rng.integers(0, 3, n), distinct_conf(rng, n))
    kind = np.arange(n) % 8
    x = box.copy()
    z, point = kind == 1, (kind == 1) & (np.arange(n) % 16 == 1)
    if variant == 1:
        x[z, 2:4] = 0.0
        x[point, 0:2] = 100.0
        x[kind == 2, 2] = -x[kind == 2, 2]
    else:
        x[z, 2:4] = x[z, 0:2]
        x[point] = 100.0
        x[kind == 2, 0], x[kind == 2, 2] = box[kind == 2, 2], box[kind == 2, 0]
    x[kind == 3] *= F32(1e30)
    x[kind == 4, 2] = np.inf
    x[kind == 5, 1] = -np.inf
    nan_rows = np.flatnonzero(kind == 6)
    x[nan_rows, rng.integers(0, 4, len(nan_rows))] = np.nan
    return x, conf, cls


def pair_iou(a, b, variant, eps=True):
    """The reference's float IoU of [0, 0, b, 1] (kept) and [0, 0, a, 1] (a <= b): inter = a, denominator
    fl(fl(b + a) - a) (+ 1e-6 for RetinaFace) -> (iou, denominator).  CXCYWH forms the same corners and areas exactly."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    den = (b + a) - a
    if variant == 2 and eps:
        den = den + EPS_RETINA
    return a / den, den


def _in_band(a, den, t):
    """|inter - thr * denom| <= 1e-5 * denom: overlaps() takes the IEEE division, not its sign test."""
    return np.abs(a.astype(np.float64) - np.float64(t) * den.astype(np.float64)) <= 1e-5 * den.astype(np.float64)


def threshold_pair(target, variant, thr, above=False):
    """Integers a < b < 2^24 whose IoU (pair_iou) is `target`, inside the band where overlaps() divides.  above=True: also
    with the exact quotient a / denom strictly above fl(thr) -- the sign of t = fma(-thr, denom, inter) says "overlaps" while
    the rounded division equals thr and says it does not, so only the division gives the reference's answer.  -> (a, b) or
    None (no such pair: for thr = 0.5 every quotient that rounds to 0.5 is exactly 0.5)."""
    t = F32(thr)
    b = np.arange(2 ** 23, 2 ** 24, 97).astype(F32)
    for da in (0, -1, 1, -2, 2):
        a = (np.round(float(target) * b.astype(np.float64)) + da).astype(F32)
        iou, den = pair_iou(a, b, variant)
        ok = (iou == target) & _in_band(a, den, t)
        if above:
            ok &= a.astype(np.float64) > np.float64(t) * den.astype(np.float64)   # exact: 24-bit x 24-bit products
        hit = np.flatnonzero(ok)
        if len(hit):
            k = hit[0]
            if above:  # t = fma(-thr, denom, inter) rounded once (the exact value fits a double): its sign and the division disagree
                t_fma = F32(np.float64(a[k]) - np.float64(t) * np.float64(den[k]))
                assert t_fma > 0 and not a[k] / den[k] > t
            return float(a[k]), float(b[k])
    if above:
        return None
    raise AssertionError(f"no integer pair with IoU {target!r}")


def retina_epsilon_pairs(thr, bs=(3.0, 4.0, 5.0)):
    """Small boxes [0, 0, a, 1] against [0, 0, b, 1] where RetinaFace's `+ 1e-6` decides: the IoU without it is above thr,
    with it not (the epsilon is more than half an ulp of these denominators)."""
    t = F32(thr)
    out = []
    for bb in bs:
        b = F32(bb)
        a0 = F32(t * b)
        a = a0 + np.arange(-64, 65).astype(F32) * np.spacing(a0)
        with_eps, den = pair_iou(a, np.full_like(a, b), 2)
        without, _ = pair_iou(a, np.full_like(a, b), 2, eps=False)
        k = np.flatnonzero((without > t) & ~(with_eps > t) & _in_band(a, den, t))
        assert len(k), (thr, bb)
        out.append((float(a[k[0]]), float(b)))
    return out


def threshold_rows(variant, thr):
    """Pairs, each in a y band of its own, whose IoU is fl(thr) moved by d = -3..3 ulps; the d = 0 pair has its exact
    quotient above fl(thr) where such a pair exists (threshold_pair(above=True)); RetinaFace adds retina_epsilon_pairs.
    -> ((box, conf, cls), rows greedy NMS keeps, whether the d = 0 pair defeats the sign test)"""
    t = F32(thr)
    pairs, sign_test_wrong = [], False
    for d in range(-3, 4):
        v = t
        for _ in range(abs(d)):
            v = np.nextafter(v, F32(np.inf if d > 0 else -np.inf))
        p = threshold_pair(v, variant, thr, above=True) if d == 0 else None
        sign_test_wrong |= p is not None
        pairs.append(p or threshold_pair(v, variant, thr))
    if variant == 2:
        pairs += retina_epsilon_pairs(thr)
    bx, conf = [], []
    for j, (a, b) in enumerate(pairs):
        bx += [(0, 2 * j, b, 2 * j + 1), (0, 2 * j, a, 2 * j + 1)]
        conf += [0.9 - 0.001 * j, 0.5 - 0.001 * j]
    x1, y1, x2, y2 = np.asarray(bx, np.float64).T
    a, b = np.asarray(pairs, F32).T
    kept = len(pairs) + int((~(pair_iou(a, b, variant)[0] > t)).sum())
    return (boxes(variant, x1, y1, x2, y2), np.asarray(conf, F32), np.zeros(len(conf), F32)), kept, sign_test_wrong
