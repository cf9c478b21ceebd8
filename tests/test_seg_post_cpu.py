"""The YOLO segmentation post-process without a GPU: the CPU oracle (oracle/seg_post_oracle.c) against a cv2 restatement of
process_mask -> scale_mask -> draw_mask_bbox's selection, the oracle's selection against the reference's own compiled
draw_mask_bbox (live, or through tests/golden/ref_seg_post_host.npz), and the argument validation of
trtx_yolo_seg_postprocess_enqueue."""
import ctypes as C

import numpy as np
import pytest

from oracle import seg_post as SP
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

F = np.float32
G = RefOutputs("ref_seg_post_host")
SIZES = [(1920, 1080), (1080, 1920), (1280, 720), (640, 480), (480, 640), (640, 640), (333, 1001), (1, 1), (3000, 100)]


@pytest.fixture(scope="module")
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(ipp)


def _boxes(variant, img_w, img_h):
    """Boxes (network pixels) inside the frame, across its borders, in the letterbox padding and degenerate."""
    x, y, w, h = SP.scale_mask_rect(img_w, img_h)   # the frame inside the 640 x 640 input
    ltrb = [[x + w * 0.2, y + h * 0.25, x + w * 0.7, y + h * 0.8], [x - 30, y - 20, x + w * 0.3, y + h * 0.4],
            [x + w * 0.6, y + h * 0.5, x + w + 25, y + h + 25], [x, y, x + w, y + h], [5, 2, 60, max(y - 1, 8)],
            [x + w * 0.5, y + h * 0.5, x + w * 0.5, y + h * 0.5], [x + 3.3, y + 2.7, x + 9.1, y + 7.9]]
    if variant == 0:
        return np.array(ltrb, F)
    b = np.array(ltrb, F)
    return np.stack([(b[:, 0] + b[:, 2]) / 2, (b[:, 1] + b[:, 3]) / 2, b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], 1).astype(F)


def _dets(rng, boxes, R=39, off=7):
    K = len(boxes)
    d = np.zeros(1 + K * R, F)
    d[0] = K
    rows = d[1:].reshape(K, R)
    rows[:, :4] = boxes
    rows[:, 4] = 0.9
    rows[:, 5] = rng.integers(0, 80, K)
    rows[:, off:off + 32] = rng.standard_normal((K, 32)) * 0.6
    return d


def _low_res(variant, proto, bbox, coeffs):
    """process_mask's 160 x 160 sigmoid(coeffs . proto) inside get_downscale_rect (float32, the same summation order)."""
    mh, mw = proto.shape[1:]
    b = bbox.astype(F)
    if variant == 0:
        l, t = max(b[0], F(0)), max(b[1], F(0))
        r, bt = min(F(b[0] + b[2]), F(640)), min(F(b[1] + b[3]), F(640))
        l, t, r, bt = l / F(4), t / F(4), r / F(4), bt / F(4)
        rx, ry, rw, rh = int(l), int(t), int(F(r - l)), int(F(bt - t))
    else:
        l, t = F(b[0] - b[2] / F(2)) / F(4), F(b[1] - b[3] / F(2)) / F(4)
        r, bt = F(b[0] + b[2] / F(2)) / F(4), F(b[1] + b[3] / F(2)) / F(4)
        rx, ry, rw, rh = (int(np.copysign(np.floor(abs(float(v)) + 0.5), float(v))) for v in (l, t, F(r - l), F(bt - t)))  # C round()
    m = np.zeros((mh, mw), F)
    x0, x1, y0, y1 = max(rx, 0), min(rx + rw, mw), max(ry, 0), min(ry + rh, mh)
    if x0 < x1 and y0 < y1:
        e = np.zeros((y1 - y0, x1 - x0), F)
        for j in range(32):
            e = e + coeffs[j] * proto[j, y0:y1, x0:x1]
        m[y0:y1, x0:x1] = F(1) / (F(1) + np.exp(-e))
    return m


def _cv2_select(cv2, variant, proto, bbox, coeffs, img_w, img_h):
    M = cv2.resize(_low_res(variant, proto, bbox, coeffs), (640, 640), interpolation=cv2.INTER_LINEAR)
    x, y, w, h = SP.scale_mask_rect(img_w, img_h)
    S = cv2.resize(np.ascontiguousarray(M[y:y + h, x:x + w]), (img_w, img_h), interpolation=cv2.INTER_LINEAR)
    rx, ry, rw, rh = P.get_rect(img_w, img_h, bbox, variant=variant)
    sel = np.zeros((img_h, img_w), np.uint8)
    x0, y0, x1, y1 = max(rx, 0), max(ry, 0), min(rx + rw, img_w), min(ry + rh, img_h)
    if x0 < x1 and y0 < y1:
        sel[y0:y1, x0:x1] = np.where(S[y0:y1, x0:x1] <= 0.5, 0, 255)
    return sel, S


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("img_w,img_h", SIZES)
def test_oracle_equals_cv2(cv2_no_ipp, variant, img_w, img_h):
    """resize -> crop -> resize -> `> 0.5` inside get_rect, in cv2 (IPP off) = the oracle, except where S lies within 1e-5 of
    0.5 (numpy's expf and OpenCV's own arithmetic vs the C restatement)."""
    rng = np.random.default_rng(img_w * 3 + img_h + variant)
    proto = rng.standard_normal((32, 160, 160)).astype(F)
    boxes = _boxes(variant, img_w, img_h)
    d = _dets(rng, boxes)
    K = len(boxes)
    rows, canv, _ = SP.seg_postprocess(variant, proto, d, img_w, img_h, max_rows=K, max_masks=K)
    src = d[1:].reshape(K, 39)
    near, selected = 0, 0
    for k in range(K):
        ref, S = _cv2_select(cv2_no_ipp, variant, proto, src[k, :4], src[k, 7:39], img_w, img_h)
        diff = canv[k] != ref
        assert np.all(np.abs(S[diff] - 0.5) <= 1e-5), (k, int(diff.sum()))
        near += int(diff.sum())
        selected += int((ref == 255).sum())
        assert tuple(int(v) for v in rows[1 + k * 6:1 + k * 6 + 4]) == P.get_rect(img_w, img_h, src[k, :4], variant=variant)
    if img_w * img_h > 1:
        assert selected > 0
    print(f"{img_w}x{img_h} v{variant}: {near} pixels within 1e-5 of 0.5 differ, {selected} selected")


def test_oracle_undefined_boxes_select_nothing():
    """Non-finite boxes and boxes whose rescaled corners leave the int range: rect {0, 0, 0, 0}, an all-zero canvas."""
    rng = np.random.default_rng(5)
    for variant in (0, 1):
        # (V8 clamps l and t at 0 first, so a -inf left edge is defined there)
        boxes = np.array([[np.nan, 5, 50, 50], [5, 5, np.inf, 50], [5, np.nan, 50, 50], [1e30, 5, 2e30, 50]], F)
        d = _dets(rng, boxes)
        canv = np.full((4, 100, 120), 9, np.uint8)
        rows, canv, _ = SP.seg_postprocess(variant, rng.standard_normal((32, 160, 160)).astype(F), d, 120, 100, max_rows=4,
                                           max_masks=4, canvases=canv)
        assert not canv.any()
        assert not rows[1:].reshape(4, 6)[:, :4].any()
        for b in boxes:
            assert P.get_rect(120, 100, b, variant=variant) == (0, 0, 0, 0)


def _ref_cases():
    """(variant, img_w, img_h, box index, bbox) of the reference pin; V5 rects that leave the image are left out (the
    reference's loop reads outside img_mask there)."""
    cases = []
    for variant in (0, 1):
        for img_w, img_h in SIZES[:7] + [(3000, 100)]:
            for i, b in enumerate(_boxes(variant, img_w, img_h)):
                if variant == 1:
                    x, y, w, h = P.get_rect(img_w, img_h, b, variant=1)
                    if x < 0 or y < 0 or x + w > img_w or y + h > img_h:
                        continue
                cases.append((variant, img_w, img_h, i, b))
    return cases


def _ref_selection(variant, img_w, img_h, bbox, seed):
    """The oracle's selection of one detection and the 640 x 640 mask it starts from."""
    rng = np.random.default_rng(seed)
    proto = rng.standard_normal((32, 160, 160)).astype(F)
    d = _dets(rng, bbox[None])
    if seed % 5 == 0:
        d[1 + 7 + 4] = np.nan    # a NaN coefficient: NaN S values, which `val <= 0.5 -> continue` keeps
    from oracle import oracle as O
    M = O.process_mask(variant, proto, d[1:5], d[8:40])
    _, canv, _ = SP.seg_postprocess(variant, proto, d, img_w, img_h, max_rows=1, max_masks=1)
    return M, canv[0] != 0


def test_oracle_selection_equals_reference_draw_mask_bbox():
    """The reference's own draw_mask_bbox + scale_mask + get_rect (compiled against a header shim whose cv::resize is the
    oracle's) colours exactly the pixels the oracle selects: live where oracle/_ref was built, else the stored digests."""
    ref = SP.load_ref()
    counts, ref_counts = [], []
    for variant, w, h, i, b in _ref_cases():
        M, sel = _ref_selection(variant, w, h, b, w + h + i)
        want = None
        if ref is not None:
            want = SP.ref_draw_mask_select(variant, M, b, w, h)
            ref_counts.append(int(want.sum()))
        # packed: the same verdict, an eighth of the bytes to hash
        G.equal(f"select.v{variant}.{w}x{h}.{i}", np.packbits(sel), ref=None if want is None else np.packbits(want))
        counts.append(int(sel.sum()))
    G.equal("counts", counts, ref=ref_counts or None)
    assert sum(counts) > 0


def _fake(n):
    return C.c_void_p(0x1000 * n)


def test_argument_validation():
    """Rejected before anything is launched (the device pointers here are never dereferenced)."""
    lib = L.load()
    assert lib.trtx_abi_sizeof(6) == C.sizeof(L.Frame) == 24

    def call(p=None, imgs=None, batch=1, proto=_fake(1), dets=_fake(2), max_rows=10, rows=_fake(3), **kw):
        q = L.MaskParams(0, 640, 640, 160, 160, 32, 39, 7, 20)
        for k, v in kw.items():
            setattr(q, k, v)
        if imgs is None:
            imgs = [(1920, 1080, _fake(4).value, 1920)]
        arr = (L.Frame * max(len(imgs), 1))()
        for i, (w, h, m, pitch) in enumerate(imgs):
            arr[i].img_w, arr[i].img_h, arr[i].masks_dev, arr[i].pitch = w, h, m, pitch
        return lib.trtx_yolo_seg_postprocess_enqueue(C.byref(q) if p is None else p, arr, batch, proto, dets, max_rows,
                                                     rows, None)

    INV, UNS = L.ERR_INVALID, L.ERR_UNSUPPORTED
    assert lib.trtx_yolo_seg_postprocess_enqueue(None, None, 1, _fake(1), _fake(2), 10, _fake(3), None) == INV
    assert call(batch=0) == INV
    assert call(max_rows=0) == INV
    assert call(dets=None) == INV
    assert call(rows=None) == INV
    assert call(proto=None) == INV                                        # canvases need the prototypes
    assert call(variant=2) == INV
    assert call(row_floats=5, coeff_offset=0, num_coeffs=4) == INV        # conf and class are floats 4 and 5
    assert call(coeff_offset=8) == INV                                    # 8 + 32 > 39
    assert call(num_coeffs=0) == INV
    assert call(max_masks=0) == INV
    assert call(mask_w=0) == INV
    assert call(mask_w=150) == UNS                                        # net = 4 x mask
    assert call(imgs=[(0, 1080, _fake(4).value, 1920)]) == INV
    assert call(imgs=[(1920, -1, _fake(4).value, 1920)]) == INV
    assert call(imgs=[(1920, 1080, _fake(4).value, 1919)]) == INV         # pitch < img_w
    assert call(imgs=[(64, 64, _fake(4).value, 64), (64, 64, None, 64)], batch=2) == INV   # NULL and non-NULL canvases
    assert call(imgs=[(64, 64, _fake(4).value, 64), (1, 5000, _fake(5).value, 1)], batch=2) == UNS  # empty scale_mask crop
    assert call(imgs=[(5000, 1, _fake(4).value, 5000)]) == UNS
    # rows only: the mask fields are not read, and any frame size works
    assert call(imgs=[(1, 5000, None, 0)], proto=None, num_coeffs=0, mask_w=0, dets=None) == INV
    # the Python wrapper: one canvas per frame
    import torch
    for n in (1, 3):
        with pytest.raises(ValueError, match="expected 2 canvases"):
            P.yolo_seg_postprocess(torch.zeros((2, 1, 160, 160)), torch.zeros((2, 1 + 39)), [(64, 48), (48, 64)], variant=0,
                                   max_rows=1, max_masks=1, canvases_out=[torch.zeros((1, 48, 64), dtype=torch.uint8)] * n)
