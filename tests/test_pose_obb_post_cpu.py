"""The pose and oriented-box geometry without a GPU: the library's host trtx_get_corner and trtx_get_rect_adapt_landmark
(whose expressions the device post-process shares, common.cuh) against the reference's own draw_bbox_obb and
draw_bbox_keypoints_line (yolov8 at net 640, yolo11's get_rect_obb at net 1024), compiled against a header shim whose drawing
calls record their points: live where oracle/_ref was built, else through tests/golden/ref_pose_obb_host.npz.  Also the
reference's undefined cases as the library defines them, and the argument validation of
trtx_yolo_pose_obb_postprocess_enqueue."""
import ctypes as C

import numpy as np
import pytest

from oracle import pose_obb as PO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

F = np.float32
G = RefOutputs("ref_pose_obb_host")
# portrait, landscape, square, extreme aspect, a single pixel
SIZES = [(1920, 1080), (1080, 1920), (1280, 720), (640, 480), (480, 640), (640, 640), (1024, 1024), (333, 1001),
         (5000, 20), (17, 3000), (1, 1)]
TREES = [("v8", 640), ("v11", 1024)]
N_OBB, N_POSE = 2500, 600


def obb_boxes(net, img_w, img_h):
    """[N_OBB, 5] (cx, cy, w, h, angle) in network pixels: random boxes inside, across and wholly outside the input, with
    h >= w swaps (h == w included), negative angles, angles at and next to 0 and +-pi/2, non-finite angles and boxes, boxes
    whose rescaled corners wrap get_corner's integer centre, and degenerate boxes."""
    rng = np.random.default_rng(net + 7 * img_w + img_h)
    b = np.zeros((N_OBB, 5), F)
    b[:, 0:2] = rng.uniform(-0.2 * net, 1.2 * net, (N_OBB, 2))
    b[:, 2:4] = rng.uniform(0, 0.7 * net, (N_OBB, 2))
    b[:, 4] = rng.uniform(-np.pi, np.pi, N_OBB)
    half = F(np.pi / 2)
    specials = [F(0), half, -half, F(np.pi), -F(np.pi), np.nextafter(half, F(0)), np.nextafter(half, F(4)),
                np.nextafter(-half, F(0)), np.nextafter(F(0), F(1)), -np.nextafter(F(0), F(1))]
    b[0:200, 4] = np.resize(np.array(specials, F), 200)
    b[100:300, 3] = b[100:300, 2]                              # h == w: swapped
    b[300:400, 3] = b[300:400, 2] + rng.uniform(1, 50, 100)    # h > w
    b[400:450, 0] = rng.uniform(-3 * net, -0.8 * net, 50)      # wholly outside
    b[450:500, 1] = rng.uniform(1.8 * net, 4 * net, 50)
    b[500:510, 4] = np.nan
    b[510:515, 4] = np.inf
    b[515:520, 4] = -np.inf
    b[520:525, 0] = np.nan
    b[525:530, 3] = np.inf
    b[530:540, 0] = 5e8                                        # 2 * rect.x leaves int (for some frames)
    b[540:545, 1] = 4e8
    b[545:550, 2] = 1e12
    b[550:560, 2:4] = 0                                        # degenerate
    return b


def pose_boxes(img_w, img_h):
    """[N_POSE, 4] l, t, r, b and [N_POSE, 51] keypoints (x, y, conf) in network pixels, inside and outside the input."""
    rng = np.random.default_rng(3 * img_w + img_h)
    x, y = rng.uniform(-100, 700, N_POSE), rng.uniform(-100, 700, N_POSE)
    ltrb = np.stack([x, y, x + rng.uniform(0, 400, N_POSE), y + rng.uniform(0, 400, N_POSE)], 1).astype(F)
    k = rng.uniform(-150, 790, (N_POSE, 51)).astype(F)
    k[:, 2::3] = rng.uniform(0, 1, (N_POSE, 17))
    k[:20, 4] = np.nan
    k[20:30, 0] = np.inf
    return ltrb, k


def _round(v):
    return np.copysign(np.floor(abs(float(v)) + 0.5), float(v))


def rect_defined(net, img_w, img_h, ltrb):
    """Whether get_rect's float -> int conversions are defined for a V8 box (the reference's arithmetic, float32)."""
    with np.errstate(all="ignore"):
        l, t, r, b = (F(v) for v in ltrb)
        r_w, r_h = F(net / (img_w * 1.0)), F(net / (img_h * 1.0))
        if r_h > r_w:
            pad = (F(net) - r_w * F(img_h)) / F(2)
            t, b, ratio = t - pad, b - pad, r_w
        else:
            pad = (F(net) - r_h * F(img_w)) / F(2)
            l, r, ratio = l - pad, r - pad, r_h
        l, r, t, b = l / ratio, r / ratio, t / ratio, b / ratio
        l = F(0) if F(0) > l else l
        t = F(0) if F(0) > t else t
        vals = [l, t, r - l, b - t]
    return all(np.isfinite(v) and -2.0 ** 31 <= _round(v) <= 2.0 ** 31 - 1 for v in vals)


def obb_rect_defined(net, img_w, img_h, box5):
    cx, cy, w, h = (F(v) for v in box5[:4])
    if h >= w:
        w, h = h, w
    with np.errstate(all="ignore"):
        ltrb = [cx - w / F(2), cy - h / F(2), cx + w / F(2), cy + h / F(2)]
    return rect_defined(net, img_w, img_h, ltrb)


def lib_corners(net, img_w, img_h, boxes5):
    lib = L.load()
    out = np.zeros((len(boxes5), 8), np.int32)
    c = (C.c_int * 8)()
    for i, b in enumerate(boxes5):
        bb = (C.c_float * 4)(*[float(v) for v in b[:4]])
        assert lib.trtx_get_corner(net, net, img_w, img_h, bb, float(b[4]), c) == 0
        out[i] = list(c)
    return out


def lib_landmarks(img_w, img_h, ltrb, kpts, net=640):
    lib = L.load()
    rects = np.zeros((len(ltrb), 4), np.int32)
    mapped = np.ascontiguousarray(kpts, F).copy()
    r = (C.c_int * 4)()
    for i in range(len(ltrb)):
        bb = (C.c_float * 4)(*[float(v) for v in ltrb[i]])
        k = mapped[i]
        assert lib.trtx_get_rect_adapt_landmark(net, net, img_w, img_h, bb, k.ctypes.data_as(C.POINTER(C.c_float)),
                                                len(k) // 3, r) == 0
        rects[i] = list(r)
    return rects, mapped


def check_corners(g, tree, net, ref_draw):
    """trtx_get_corner at `net` = the corners `ref_draw(img_w, img_h, boxes5) -> (corners, printed text)` hands to
    cv::polylines, for every box whose get_rect is defined, on every frame size: live when ref_draw is given (also the 3
    debug lines printed per box), else g's stored digests."""
    for w, h in SIZES:
        b = obb_boxes(net, w, h)
        keep = np.array([obb_rect_defined(net, w, h, x) for x in b])
        want = None
        if ref_draw is not None:
            want, log = ref_draw(w, h, b)
            want = want[keep]
            assert log.count("Original angle: ") == log.count("Adjusted angle: ") == log.count("Normal angle: ") == len(b)
            assert keep.sum() > 0.9 * len(b)
        g.equal(f"obb.{tree}.{w}x{h}", lib_corners(net, w, h, b)[keep], ref=want)


@pytest.mark.parametrize("tree,net", TREES)
def test_get_corner_equals_reference_draw_bbox_obb(tree, net):
    """trtx_get_corner = the corners the reference's draw_bbox_obb hands to cv::polylines, for every box whose get_rect is
    defined, on 11 frame sizes: live where oracle/_ref was built (also the 3 debug lines printed per box), else the
    stored digests."""
    ref = PO.load_ref()
    check_corners(G, tree, net, None if ref is None else lambda w, h, b: PO.ref_draw_bbox_obb(tree, w, h, b))


@pytest.mark.parametrize("tree", ["v8", "v11"])
def test_get_rect_adapt_landmark_equals_reference_draw_bbox_keypoints_line(tree):
    """trtx_get_rect_adapt_landmark = draw_bbox_keypoints_line's rectangle (for boxes whose get_rect is defined) and its
    in-place keypoint mapping (all, NaN and inf included), on 11 frame sizes."""
    ref = PO.load_ref()
    for w, h in SIZES:
        ltrb, k = pose_boxes(w, h)
        keep = np.array([rect_defined(640, w, h, x) for x in ltrb])
        got_r, got_k = lib_landmarks(w, h, ltrb, k)
        want_r = want_k = None
        if ref is not None:
            want_r, want_k = PO.ref_draw_bbox_keypoints_line(tree, w, h, ltrb, k)
            want_r, want_k = want_r[keep], want_k.view(np.int32)
            # the rectangle is get_rect's V8 branch
            assert all(tuple(got_r[i]) == P.get_rect(w, h, ltrb[i]) for i in range(0, len(ltrb), 7))
        G.equal(f"rect.{tree}.{w}x{h}", got_r[keep], ref=want_r)
        G.equal(f"kpts.{tree}.{w}x{h}", got_k.view(np.int32), ref=want_k)   # bit for bit, NaN payloads too


def test_undefined_cases():
    """Where the reference's conversions are undefined: a NaN / infinite angle makes every corner's float -> int conversion
    undefined (INT_MIN on x86-64, which the clamp turns into 0); a box whose get_rect is undefined (NaN, infinite or huge)
    gets four (0, 0) corners; 2 * rect.x leaving the int range wraps, as in the compiled reference."""
    for net in (640, 1024):
        for angle in (np.nan, np.inf, -np.inf):
            assert P.get_corner(1920, 1080, (300, 280, 120, 40), angle, net, net) == ((0, 0),) * 4
        for box in ((np.nan, 280, 120, 40), (300, np.inf, 120, 40), (300, 280, 1e12, 40), (4e9, 280, 120, 40)):
            assert P.get_corner(1920, 1080, box, 0.3, net, net) == ((0, 0),) * 4, box
    # rect.x = 1.5e9 at 1920 x 1080 / 640: the centre (2 * x + w) / 2 wraps negative, every x clamps to 0 (not 1919)
    assert obb_rect_defined(640, 1920, 1080, (5e8, 300, 100, 50))
    corners = P.get_corner(1920, 1080, (5e8, 300, 100, 50), 0.3)
    assert [c[0] for c in corners] == [0] * 4 and all(0 < c[1] < 1080 for c in corners)
    # get_rect_adapt_landmark: an undefined rectangle is {0, 0, 0, 0} (trtx_get_rect's definition); keypoints still map
    rect, k = P.get_rect_adapt_landmark(1920, 1080, (np.nan, 5, 50, 50), [320.0, 300.0, 0.7])
    r_w = F(640 / 1920.0)
    pad = (F(640) - r_w * F(1080)) / F(2)
    assert rect == (0, 0, 0, 0) and k == [F(320) / r_w, (F(300) - pad) / r_w, F(0.7)]


def test_nets_640_and_1024_give_different_corners():
    """The two trees pin different mappings: on the same boxes, get_corner at net 640 and at net 1024 differ (except at
    1 x 1, where every corner is clamped to (0, 0))."""
    for w, h in SIZES:
        b = obb_boxes(640, w, h)
        assert np.array_equal(lib_corners(640, w, h, b), lib_corners(1024, w, h, b)) == (w * h == 1), (w, h)


def _fake(n):
    return C.c_void_p(0x1000 * n)


def test_argument_validation():
    """Rejected before anything is launched (the device pointers here are never dereferenced)."""
    lib = L.load()
    assert lib.trtx_abi_sizeof(7) == C.sizeof(L.PoseObbParams) == 24
    INV = L.ERR_INVALID

    def call(sizes=((1920, 1080),), batch=None, dets=_fake(1), max_rows=10, rows=_fake(2), **kw):
        q = L.PoseObbParams(L.TASK_POSE, 640, 640, 58, 7, 17)
        for k, v in kw.items():
            setattr(q, k, v)
        wh = (C.c_int32 * max(2 * len(sizes), 2))(*[v for s in sizes for v in s])
        return lib.trtx_yolo_pose_obb_postprocess_enqueue(C.byref(q), wh, len(sizes) if batch is None else batch, dets,
                                                          max_rows, rows, None)

    assert lib.trtx_yolo_pose_obb_postprocess_enqueue(None, None, 1, _fake(1), 10, _fake(2), None) == INV
    assert call(batch=0) == INV
    assert call(max_rows=0) == INV
    assert call(dets=None) == INV
    assert call(rows=None) == INV
    assert call(task=0) == INV
    assert call(task=3) == INV
    assert call(net_w=0) == INV
    assert call(row_floats=6, extra_offset=0, num_kpts=2) == INV     # the keep flag is float 6
    assert call(extra_offset=8) == INV                               # 8 + 51 > 58
    assert call(extra_offset=-1) == INV
    assert call(num_kpts=-1) == INV
    assert call(num_kpts=65, row_floats=7 + 195) == INV
    assert call(task=L.TASK_OBB, row_floats=8, extra_offset=8) == INV  # the angle lies outside the row
    assert call(sizes=((1920, 1080), (0, 5))) == INV
    assert call(sizes=((1920, 1080), (5, -1))) == INV
    bb = (C.c_float * 4)(1, 2, 3, 4)
    c = (C.c_int * 8)()
    assert lib.trtx_get_corner(640, 640, 0, 5, bb, 0.0, c) == INV
    assert lib.trtx_get_corner(640, 640, 5, 5, None, 0.0, c) == INV
