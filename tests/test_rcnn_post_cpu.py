"""Mask R-CNN post-process (rcnn/rcnn.cpp:516-550) on the CPU: the letterbox pads against the reference's compiled
preprocessImg (oracle/_ref/libref_rcnn_host.so, or tests/golden/ref_rcnn_host.npz where it was not built), the oracle's mask
paste against cv2, and the rescale / rectangle arithmetic against an independent numpy float32 restatement."""
import ctypes as C

import numpy as np
import pytest

from oracle import rcnn_post as RP
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

G = RefOutputs("ref_rcnn_host")
F = np.float32


def calculate_size(img_w, img_h, min_size=800.0, max_size=1333.0):
    """calculateSize, rcnn/rcnn.cpp:349-366 (float arithmetic, `+ 0.5` in double, int truncation) -> (INPUT_W, INPUT_H)."""
    ratio = F(min_size) / F(min(img_h, img_w))
    if img_h < img_w:
        newh, neww = F(min_size), F(ratio * F(img_w))
    else:
        newh, neww = F(ratio * F(img_h)), F(min_size)
    if max(newh, neww) > max_size:
        ratio = F(max_size) / F(max(newh, neww))
        newh, neww = F(newh * ratio), F(neww * ratio)
    return int(float(neww) + 0.5), int(float(newh) + 0.5)


def _pad_cases():
    cases = []
    for w, h in ((640, 480), (480, 640), (1920, 1080), (1080, 1920), (640, 640), (1, 1), (3, 1001), (1001, 3), (333, 517),
                 (1279, 721), (4096, 2160), (17, 13)):
        cases.append((w, h) + calculate_size(w, h))
        cases.append((w, h, 1067, 800))
    rng = np.random.default_rng(11)
    for _ in range(130):   # portrait, landscape, square, odd and even
        w, h = (int(v) for v in rng.integers(1, 2500, 2))
        cases.append((w, h, 1067, 800) if rng.random() < 0.5 else (w, h) + calculate_size(w, h))
    for s in range(1, 60, 3):
        cases.append((s, s, 800, 800))
    # odd gaps: x = k + 0.5, so round(x - 0.1) and round(x + 0.1) differ
    for w in range(600, 640, 3):
        cases.append((w, 480, 1067, 800))
        cases.append((480, w, 1067, 800))
    return cases


def test_letterbox_pads_equal_reference():
    """trtx_rcnn_letterbox_pads and the oracle's restatement = preprocessImg's four int& outputs (rcnn/common.hpp:79-102)."""
    ref = G.lib("libref_rcnn_host.so")
    lib = L.load()
    cases = _pad_cases()
    assert len(cases) >= 200
    mine, refs = [], []
    for (w, h, nw, nh) in cases:
        p = (C.c_int * 4)()
        assert lib.trtx_rcnn_letterbox_pads(w, h, nw, nh, p) == 0
        assert tuple(p) == RP.rcnn_letterbox_pads(w, h, nw, nh), (w, h, nw, nh)
        mine.append(list(p) + [w, h, nw, nh])
        if ref is not None:
            r = np.zeros(4, np.int32)
            ref.ref_rcnn_preprocess_pads(w, h, nw, nh, r.ctypes.data_as(C.c_void_p))
            refs.append(list(r) + [w, h, nw, nh])
    mine = np.array(mine, np.int32)
    assert (mine[:, 0] != mine[:, 1]).sum() > 20   # cases where x -/+ 0.1 round apart
    G.equal("rcnn_pads", mine, np.array(refs, np.int32) if ref is not None else None)
    # the sizes quoted in the design notes
    for (w, h, pads) in ((640, 480, (0, 1, 0, 0)), (480, 640, (233, 234, 0, 0)), (1920, 1080, (0, 0, 100, 100))):
        assert RP.rcnn_letterbox_pads(w, h, 1067, 800) == pads
    assert calculate_size(640, 480) == (1067, 800)


# ------------------------------------------------------------------ paste vs cv2 ------------------------------
def _cv2_canvas(cv2, mask, rect, img_w, img_h):
    """rcnn.cpp:547-550 in cv2: resize to the rectangle, threshold at 0.5 to 0/255, add into a zero u8 ROI.
    Also returns the float resize placed on the canvas (NaN outside r) for the near-threshold check."""
    x, y, w, h = rect
    part = cv2.resize(mask, (w, h), interpolation=cv2.INTER_LINEAR)
    _, t = cv2.threshold(part, 0.5, 255, cv2.THRESH_BINARY)
    cur = np.zeros((img_h, img_w), np.uint8)
    cur[y:y + h, x:x + w] = cv2.add(cur[y:y + h, x:x + w], t, dtype=cv2.CV_8U)
    val = np.full((img_h, img_w), np.nan, np.float32)
    val[y:y + h, x:x + w] = part
    return cur, val


def _paste_vs_cv2(cv2, rects, img_w, img_h, seed):
    """Boxes that give exactly `rects` (net = image size: pads 0, ratio 1), pasted by the oracle, against cv2.
    Returns the number of pixels that differ, all of them within 1 ulp of the 0.5 threshold in cv2's float value."""
    rng = np.random.default_rng(seed)
    near = 0
    lo, hi = np.nextafter(F(0.5), F(0)), np.nextafter(F(0.5), F(1))
    for i0 in range(0, len(rects), 128):
        chunk = rects[i0:i0 + 128]
        D = len(chunk)
        boxes = np.array([[x + 1.5, y + 1.25, x + w - 1.5, y + h - 1.75] for (x, y, w, h) in chunk], np.float32)
        masks = (1 / (1 + np.exp(-rng.standard_normal((D, 14, 14)) * 2))).astype(np.float32)
        masks[:, 3, 3] = 0.5
        rows, canv = RP.rcnn_postprocess(np.full(D, 0.9, F), boxes, np.zeros(D, F), masks, img_w, img_h, img_w, img_h)
        assert rows[0] == D
        for k, rect in enumerate(chunk):
            assert RP.rcnn_mask_rect(rows[1 + k * 7:5 + k * 7], img_w, img_h) == tuple(rect)
            ref, val = _cv2_canvas(cv2, masks[k], rect, img_w, img_h)
            diff = canv[k] != ref
            if diff.any():
                v = val[diff]
                assert np.all((v >= lo) & (v <= hi)), (rect, v[(v < lo) | (v > hi)][:5])
                near += int(diff.sum())
    return near


@pytest.fixture(scope="module")
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(ipp)


def test_paste_small_rects_equal_cv2(cv2_no_ipp):
    """Every rectangle size 1..64 x 1..64 (7 x 7 is OpenCV's INTER_AREA fast path, 14 x 14 a plain copy there)."""
    rects = [(3 + (w * 7) % 20, 2 + (h * 5) % 13, w, h) for w in range(1, 65) for h in range(1, 65)]
    near = _paste_vs_cv2(cv2_no_ipp, rects, 100, 80, seed=1)
    print(f"pixels within 1 ulp of 0.5 that differ from cv2: {near}")


def test_paste_large_and_clamped_rects_equal_cv2(cv2_no_ipp):
    rects = [(0, 0, 1920, 1080), (100, 50, 1000, 700), (5, 3, 1911, 1075), (1800, 900, 120, 180), (0, 500, 259, 39),
             (700, 0, 97, 1080), (13, 17, 480, 255), (1000, 1000, 7, 7), (30, 40, 14, 14)]
    near = _paste_vs_cv2(cv2_no_ipp, rects, 1920, 1080, seed=2)
    print(f"pixels within 1 ulp of 0.5 that differ from cv2: {near}")
    # rectangles clamped at the four borders: boxes that leave the image on one side
    img_w, img_h = 640, 480
    boxes = np.array([[-30, 100, 50, 200], [600, 100, 700, 200], [100, -20, 300, 60], [100, 400, 300, 520],
                      [-5, -5, 700, 600], [0.2, 0.7, 639.5, 479.1]], np.float32)
    D = len(boxes)
    masks = np.random.default_rng(3).uniform(0, 1, (D, 14, 14)).astype(np.float32)
    rows, canv = RP.rcnn_postprocess(np.full(D, 0.9, F), boxes, np.zeros(D, F), masks, img_w, img_h, img_w, img_h)
    for k in range(D):
        rect = RP.rcnn_mask_rect(rows[1 + k * 7:5 + k * 7], img_w, img_h)
        x, y, w, h = rect
        assert x == 0 or y == 0 or x + w == img_w or y + h == img_h
        ref, val = _cv2_canvas(cv2_no_ipp, masks[k], rect, img_w, img_h)
        d = canv[k] != ref
        assert np.all(np.abs(val[d] - 0.5) <= 6e-8)


# ------------------------------------------------------------------ rescale and rectangle arithmetic -----------
def _np_rows(scores, boxes, classes, img_w, img_h, net_w, net_h, pads, thr):
    l, r, t, b = pads
    h_ratio = F(F(img_h) / F(net_h - (t + b)))
    w_ratio = F(F(img_w) / F(net_w - (l + r)))
    rows = []
    for i in range(len(scores)):
        if not scores[i] > F(thr):
            continue
        bx = boxes[i]
        rows.append([F(F(bx[0] - F(l)) * w_ratio), F(F(bx[1] - F(t)) * h_ratio), F(F(bx[2] - F(l)) * w_ratio),
                     F(F(bx[3] - F(t)) * h_ratio), scores[i], classes[i], F(i)])
    return np.array(rows, np.float32).reshape(-1, 7)


def _np_rect(box, img_w, img_h):
    """rcnn.cpp:543-546 in float64 (floor / ceil of a float are exact), then the conditions under which OpenCV throws."""
    if not np.all(np.isfinite(box)):
        return None
    out = []
    for c0, c1, size in ((box[0], box[2], img_w), (box[1], box[3], img_h)):
        p = max(np.floor(np.float64(c0)) - 1, 0.0)
        q = min(np.ceil(np.float64(c1)) + 1, float(size))
        o, n = min(p, q), abs(q - p)
        if o < 0 or o + n > size or n == 0:   # Mat::operator()(Rect) / cv::resize throw
            return None
        out.append((int(o), int(n)))
    return (out[0][0], out[1][0], out[0][1], out[1][1])


def _edge_boxes(rng, net_w, net_h, pads, n=300):
    l, r, t, b = pads
    boxes = []
    for _ in range(n):
        x1, y1 = rng.uniform(-50, net_w + 50), rng.uniform(-50, net_h + 50)
        boxes.append([x1, y1, x1 + rng.uniform(-20, 400), y1 + rng.uniform(-20, 300)])
    boxes += [
        [0, 0, max(l - 1, 0), max(t - 1, 0)],                                # inside the top-left padding
        [net_w - r + 0.5, net_h - b + 0.5, net_w, net_h],                    # inside the bottom-right padding
        [l - 10, t - 10, l + 10, t + 10],                                    # straddling the padding border
        [net_w - r - 10, net_h - b - 10, net_w + 5, net_h + 5],
        [100, 100, 100, 100], [100.5, 100.5, 100.5, 100.5], [200, 200, 150, 150],   # degenerate, inverted
        [np.nan, 10, 50, 50], [10, np.inf, 50, 50], [10, 10, -np.inf, 50], [10, 10, 50, np.nan],
        [1e30, 10, 2e30, 50], [-1e30, -1e30, 1e30, 1e30], [10, 10, 3e9, 4e9], [-3e9, 10, -2e9, 50],
    ]
    return np.array(boxes, np.float32)


@pytest.mark.parametrize("img_w,img_h", [(640, 480), (480, 640), (1920, 1080), (637, 479)])
def test_rows_and_rects_equal_numpy(img_w, img_h):
    net_w, net_h = calculate_size(img_w, img_h)
    pads = RP.rcnn_letterbox_pads(img_w, img_h, net_w, net_h)
    rng = np.random.default_rng(img_w * 7 + img_h)
    boxes = _edge_boxes(rng, net_w, net_h, pads)
    D = len(boxes)
    scores = rng.uniform(0, 1, D).astype(np.float32)
    scores[::7] = F(0.6)                      # exactly at the threshold: not kept (score > SCORE_THRESH)
    scores[3::11] = np.nan                    # a NaN score is not kept
    scores[-15:] = 0.9                        # every edge box is kept
    classes = rng.integers(0, 80, D).astype(np.float32)
    rows, _ = RP.rcnn_postprocess(scores, boxes, classes, None, img_w, img_h, net_w, net_h, 0.6)
    exp = _np_rows(scores, boxes, classes, img_w, img_h, net_w, net_h, pads, 0.6)
    n = int(rows[0])
    assert n == len(exp) and 15 < n < D
    got = rows[1:1 + n * 7].reshape(n, 7)
    assert np.array_equal(got, exp, equal_nan=True)
    assert not np.any(rows[1 + n * 7:])
    kinds = {"none": 0, "rect": 0}
    for k in range(n):
        want = _np_rect(got[k, :4], img_w, img_h)
        assert RP.rcnn_mask_rect(got[k, :4], img_w, img_h) == want, got[k, :4]
        kinds["none" if want is None else "rect"] += 1
    assert kinds["none"] > 8 and kinds["rect"] > 8


# ------------------------------------------------------------------ argument validation ------------------------
def test_rcnn_postprocess_argument_validation():
    """Invalid arguments are rejected before anything is launched (the pointers here are never dereferenced)."""
    lib = L.load()
    ok = dict(net_w=1067, net_h=800, img_w=640, img_h=480, detections_per_im=100, mask_size=14, max_masks=100, score_thresh=0.6)

    def call(params=None, batch=1, ptrs=(16, 32, 48, 64, 80, 96)):
        q = L.RcnnPostParams(**{**ok, **(params or {})})
        p = [None if v is None else C.c_void_p(v) for v in ptrs]
        return lib.trtx_rcnn_postprocess_enqueue(C.byref(q), batch, *p, None)

    inv = L.ERR_INVALID
    assert lib.trtx_rcnn_postprocess_enqueue(None, 1, 16, 32, 48, 64, 80, 96, None) == inv
    assert call(batch=0) == inv
    for i in (0, 1, 2, 4):                                        # scores, boxes, classes, rows are required
        ptrs = [16, 32, 48, 64, 80, 96]
        ptrs[i] = None
        assert call(ptrs=tuple(ptrs)) == inv
    assert call(ptrs=(16, 32, 48, None, 80, 96)) == inv          # masks without canvases and the other way round
    assert call(ptrs=(16, 32, 48, 64, 80, None)) == inv
    for k in ("net_w", "net_h", "img_w", "img_h", "detections_per_im", "mask_size", "max_masks"):
        assert call({k: 0}) == inv, k
        assert call({k: -3}) == inv, k
    assert call({"mask_size": 33}) == inv                         # larger than the shared-memory stage
    p = (C.c_int * 4)()
    assert lib.trtx_rcnn_letterbox_pads(0, 480, 1067, 800, p) == inv
    assert lib.trtx_rcnn_letterbox_pads(640, 480, 1067, -1, p) == inv
    assert lib.trtx_rcnn_letterbox_pads(640, 480, 1067, 800, None) == inv
    assert L.load().trtx_abi_sizeof(5) == C.sizeof(L.RcnnPostParams)
