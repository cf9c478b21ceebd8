"""Mask R-CNN instance outlines without a GPU:
  - the oracle (oracle_find_contours_external) equals cv2.findContours(img, RETR_EXTERNAL, CHAIN_APPROX_NONE) exactly --
    same list, same order, same points -- on seeded random images, structured cases and paste-like masks up to 1920 x 1080;
  - the facts the restatement rests on, each checked against cv2 directly;
  - trtx_rcnn_contours_enqueue's argument checks and trtx_rcnn_contours_workspace_size."""
import ctypes as C

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import contours as CO  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402


def _cv2(img):
    cs, _ = cv2.findContours(img, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)
    return cs


def _same(img):
    lengths, points = CO.cv2_contours(_cv2(img))
    n, total, ln, pt = CO.find_contours_external(img)
    assert n == len(lengths) and total == len(points)
    np.testing.assert_array_equal(ln, lengths)
    np.testing.assert_array_equal(pt, points)
    return n


def _pts(img):
    return [[tuple(p) for p in c.reshape(-1, 2).tolist()] for c in _cv2(img)]


def test_random_images_equal_cv2():
    rng = np.random.default_rng(2024)
    contours = 0
    for _ in range(5000):
        h, w = (int(v) for v in rng.integers(1, 65, 2))
        d = rng.uniform(0.05, 0.95)
        img = ((rng.random((h, w)) < d) * rng.integers(1, 256, (h, w))).astype(np.uint8)
        contours += _same(img)
    assert contours > 100000


def _ring(n, x0, y0, size, width):
    img = np.zeros((n, n), np.uint8)
    img[y0:y0 + size, x0:x0 + size] = 1
    img[y0 + width:y0 + size - width, x0 + width:x0 + size - width] = 0
    return img


def structured():
    out = [np.zeros((5, 7), np.uint8), np.full((6, 4), 9, np.uint8), np.full((1, 1), 1, np.uint8)]
    for y, x in ((0, 0), (0, 6), (4, 0), (4, 6)):
        img = np.zeros((5, 7), np.uint8)
        img[y, x] = 200
        out.append(img)
    h = np.zeros((4, 8), np.uint8)
    h[1, 1:5] = 1
    v = np.zeros((8, 4), np.uint8)
    v[1:6, 2] = 1
    dg = np.zeros((6, 6), np.uint8)
    for i in range(1, 5):
        dg[i, i] = 1
    ad = np.fliplr(dg).copy()
    out += [h, v, dg, ad]
    for width in (1, 2):
        r = _ring(16, 2, 2, 12, width)
        r[7, 7] = 1                                  # an island in the hole
        r[5:7, 9:11] = 3
        out.append(r)
    nested = _ring(24, 1, 1, 22, 1) | _ring(24, 4, 4, 16, 2) | _ring(24, 9, 9, 6, 1)
    nested[11, 11] = 1
    out.append(nested)
    joins = np.zeros((8, 8), np.uint8)               # components joined only diagonally
    joins[1, 1] = joins[2, 2] = joins[2, 0] = joins[3, 3] = joins[4, 2] = joins[5, 5] = joins[6, 4] = 1
    out.append(joins)
    cb = (np.indices((9, 11)).sum(0) % 2).astype(np.uint8)   # a checkerboard: one 8-connected component
    out.append(cb)
    return out


def test_structured_cases_equal_cv2():
    for img in structured():
        _same(np.ascontiguousarray(img))


def test_paste_like_masks_equal_cv2():
    rng = np.random.default_rng(7)
    for w, h in ((28, 28), (640, 480), (333, 777), (1280, 720), (1920, 1080)):
        for _ in range(3):
            m = (1 / (1 + np.exp(-rng.standard_normal((14, 14)) * 2))).astype(np.float32)
            img = ((cv2.resize(m, (w, h), interpolation=cv2.INTER_LINEAR) > 0.5) * 255).astype(np.uint8)
            _same(img)


def test_truncated_lists_are_prefixes():
    rng = np.random.default_rng(3)
    img = ((rng.random((40, 50)) < 0.3) * 255).astype(np.uint8)
    n, total, ln, pt = CO.find_contours_external(img)
    for mc, mp in ((1, 1), (3, 17), (n, total), (n + 5, total + 9)):
        n2, t2, l2, p2 = CO.find_contours_external(img, mc, mp)
        assert (n2, t2) == (n, total)
        np.testing.assert_array_equal(l2, ln[:mc])
        np.testing.assert_array_equal(p2, pt[:mp])


def test_facts():
    # foreground is any nonzero byte; 8-connected; pixels outside are 0, so edge components are traced
    a = np.zeros((5, 5), np.uint8)
    a[0, 0], a[1, 1], a[4, 4] = 3, 250, 1
    assert _pts(a) == [[(4, 4)], [(0, 0), (1, 1)]]
    # outer borders of top-level components only, equal to RETR_TREE's contours with parent -1, same order and points
    rng = np.random.default_rng(11)
    for _ in range(300):
        img = ((rng.random(tuple(rng.integers(1, 40, 2))) < rng.uniform(0.2, 0.8)) * 1).astype(np.uint8)
        tree, hier = cv2.findContours(img, cv2.RETR_TREE, cv2.CHAIN_APPROX_NONE)
        top = [c for c, h in zip(tree, hier[0] if hier is not None else []) if h[3] == -1]
        ext = _cv2(img)
        assert len(top) == len(ext) and all(np.array_equal(p, q) for p, q in zip(top, ext))
    # an island in a 1-px ring's hole is not reported
    r = _ring(9, 1, 1, 7, 1)
    r[4, 4] = 1
    assert len(_cv2(r)) == 1
    # each contour starts at its component's raster-first pixel, contours in descending raster order of their starts
    for _ in range(200):
        img = ((rng.random(tuple(rng.integers(2, 40, 2))) < 0.3) * 1).astype(np.uint8)
        starts = [tuple(c[0, 0][::-1]) for c in _cv2(img)]          # (y, x)
        assert starts == sorted(starts, reverse=True)
        n, lab = cv2.connectedComponents(img, connectivity=8)
        for c in _cv2(img):
            x, y = c[0, 0]
            ys, xs = np.nonzero(lab == lab[y, x])
            assert (ys[0], xs[0]) == (y, x)
    # down the left side first
    sq = np.zeros((5, 5), np.uint8)
    sq[1:4, 1:4] = 1
    assert _pts(sq) == [[(1, 1), (1, 2), (1, 3), (2, 3), (3, 3), (3, 2), (3, 1), (2, 1)]]
    # pixels are revisited on thin structures
    one = np.zeros((3, 3), np.uint8)
    one[1, 1] = 1
    assert _pts(one) == [[(1, 1)]]
    ln = np.zeros((3, 6), np.uint8)
    ln[1, 1:5] = 1
    assert _pts(ln) == [[(1, 1), (2, 1), (3, 1), (4, 1), (3, 1), (2, 1)]]
    dg = np.zeros((5, 5), np.uint8)
    dg[1, 1] = dg[2, 2] = dg[3, 3] = 1
    assert _pts(dg) == [[(1, 1), (2, 2), (3, 3), (2, 2)]]
    # and the oracle agrees on each of them
    for img in (a, r, sq, one, ln, dg):
        _same(img)


# ------------------------------------------------------------------ host checks of the C entry points
OK = dict(net_w=0, net_h=0, img_w=0, img_h=0, detections_per_im=100, mask_size=1, max_masks=20, score_thresh=0.0)


def _frames(sizes, pitch_extra=0):
    d = (L.Frame * len(sizes))()
    for i, (w, h) in enumerate(sizes):
        d[i].img_w, d[i].img_h = w, h
        d[i].masks_dev = 4096 * (i + 1)
        d[i].pitch = w + pitch_extra
    return d


def _size(params=None, frames=None, batch=None):
    q = L.RcnnPostParams(**{**OK, **(params or {})})
    frames = _frames([(640, 480), (1920, 1080)]) if frames is None else frames
    return L.load().trtx_rcnn_contours_workspace_size(C.byref(q), frames, len(frames) if batch is None else batch)


# rows, counts, lengths, points, workspace: fake device addresses, never dereferenced by a rejected call
PTRS = [0x10000, 0x20000, 0x30000, 0x40000, 0x100000]


def _call(params=None, frames=None, batch=None, ptrs=PTRS, caps=(8, 1000), wbytes=None):
    q = L.RcnnPostParams(**{**OK, **(params or {})})
    frames = _frames([(640, 480), (1920, 1080)]) if frames is None else frames
    batch = len(frames) if batch is None else batch
    if wbytes is None:
        wbytes = _size(params, frames, batch) if batch > 0 else 1 << 40
    p = [None if v is None else C.c_void_p(v) for v in ptrs]
    return L.load().trtx_rcnn_contours_enqueue(C.byref(q), frames, batch, p[0], caps[0], caps[1], p[1], p[2], p[3], p[4],
                                               wbytes, None)


def _slot(w, h):
    return (((w + 2) * (h + 2) + 15) // 16 * 16, ((w + 1) // 2) * ((h + 1) // 2) * 8, 32 * ((w + 1) // 2) * 8)


def test_workspace_size():
    for sizes, M in (([(640, 480)] * 8, 20), ([(1920, 1080)] * 8, 20), ([(640, 480), (17, 2000), (3000, 5)], 100),
                     ([(64, 48)] * 70, 1), ([(5, 5)], 3)):
        regions = [_slot(w, h) for w, h in sizes]
        slot = sum(max(r[i] for r in regions) for i in range(3))
        slot = (slot + 255) // 256 * 256
        slots = min(min(len(sizes), 64) * M, 128)
        assert _size({"max_masks": M}, _frames(sizes)) == slots * slot, (sizes, M)
    # the value does not depend on the pitch or the canvas address
    assert _size(frames=_frames([(640, 480)], pitch_extra=77)) == _size(frames=_frames([(640, 480)]))
    # rejected arguments give 0
    assert _size({"max_masks": 0}) == 0
    assert _size({"detections_per_im": -1}) == 0
    assert _size(batch=0) == 0
    assert L.load().trtx_rcnn_contours_workspace_size(None, _frames([(4, 4)]), 1) == 0


def test_null_pointers_batch_and_capacities():
    inv = L.ERR_INVALID
    lib = L.load()
    q = L.RcnnPostParams(**OK)
    assert lib.trtx_rcnn_contours_enqueue(None, _frames([(8, 8)]), 1, *[C.c_void_p(v) for v in PTRS[:1]], 4, 4,
                                          *[C.c_void_p(v) for v in PTRS[1:]], 1 << 30, None) == inv
    assert lib.trtx_rcnn_contours_enqueue(C.byref(q), None, 1, C.c_void_p(PTRS[0]), 4, 4,
                                          *[C.c_void_p(v) for v in PTRS[1:]], 1 << 30, None) == inv
    for i in range(5):
        ptrs = list(PTRS)
        ptrs[i] = None
        assert _call(ptrs=ptrs) == inv, i
    assert _call(batch=0) == inv
    assert _call(batch=-3) == inv
    for caps in ((0, 10), (-1, 10), (10, 0), (10, -7)):
        assert _call(caps=caps) == inv, caps
    for k in ("detections_per_im", "max_masks"):
        assert _call({k: 0}) == inv, k
        assert _call({k: -2}) == inv, k


def test_frames_and_workspace():
    inv = L.ERR_INVALID
    for bad in ((0, 480), (640, 0), (-1, 480)):
        assert _call(frames=_frames([(640, 480), bad])) == inv, bad   # every frame is checked
    f = _frames([(640, 480), (64, 48)])
    f[1].masks_dev = None                                             # a frame without canvases
    assert _call(frames=f) == inv
    f = _frames([(640, 480), (64, 48)])
    f[1].pitch = 63                                                   # pitch < img_w
    assert _call(frames=f) == inv
    assert _call(ptrs=PTRS[:4] + [PTRS[4] + 8]) == inv                # a misaligned workspace
    need = _size()
    assert _call(wbytes=need - 1) == L.ERR_WORKSPACE
    assert _call(frames=_frames([(30000, 20000)])) == L.ERR_UNSUPPORTED   # more than 2^29 pixels
    # an invalid frame is INVALID even when the workspace is also too small
    assert _call(frames=_frames([(640, 480), (0, 4)]), wbytes=1) == inv


def test_python_wrapper_validates_shapes():
    import torch

    from tensorrtx_b200 import plugins as P
    with pytest.raises(ValueError):
        P.rcnn_contours(torch.zeros((2, 1 + 10 * 7)), [], frames=[(64, 48)], detections_per_im=10, max_masks=2,
                        max_contours=4, max_points=10)
    with pytest.raises(ValueError):
        P.rcnn_contours(torch.zeros((1, 1 + 10 * 7)), [torch.zeros((3, 48, 64), dtype=torch.uint8)], frames=[(64, 48)],
                        detections_per_im=10, max_masks=2, max_contours=4, max_points=10)
