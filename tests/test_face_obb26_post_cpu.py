"""The RetinaFace and yolo26-obb geometry without a GPU.

- RetinaFace: the library's host trtx_retina_get_rect_adapt_landmark (whose expressions the device face post-process
  shares, common.cuh) against the reference's compiled get_rect_adapt_landmark (retinaface/common.hpp, at -O2 and -O0), on
  ordinary faces and on the cases the reference leaves undefined (NaN, infinite and out-of-int corners, r - l overflow),
  at 640x480 (retinaface) and 640x640 (retinafaceAntiCov's identical copy, BASELINE config 3).
- yolo26-obb: trtx_get_corner at net 1024 against yolo26's own compiled draw_bbox_obb.
Both live where oracle/_ref was built, else through tests/golden/ref_face_obb26_host.npz.  Also the argument validation of
trtx_retina_postprocess_enqueue and of the NMS-free OBB task, without a device."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import face_obb26 as FO
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

import test_pose_obb_post_cpu as T

F = np.float32
G = RefOutputs("ref_face_obb26_host")
INPUTS = [(640, 480), (640, 640)]   # retinaface's decodeplugin::INPUT_W x INPUT_H; retinafaceAntiCov's
SIZES = T.SIZES                     # 11 frame sizes: portrait, landscape, square, extreme aspect, a single pixel
N_FACE = 600
INT_MIN = -2 ** 31
# box coordinates whose mapped value is NaN, infinite, outside the int range, or inside it but far enough apart to make
# r - l wrap
SPECIAL = [np.nan, np.inf, -np.inf, 3e9, -3e9, 1e38, -1e38, 7.1e8, -7.1e8, 1.4e9, -1.4e9, 2.1e9, -2.1e9]


def face_cases(in_w, in_h, img_w, img_h):
    """bbox [N_FACE, 4] (x1, y1, x2, y2) and landmarks [N_FACE, 10] in network pixels: ordinary faces inside and around the
    input, then boxes with one or two special coordinates, NaN / infinite landmarks."""
    rng = np.random.default_rng(in_h + 5 * img_w + img_h)
    x1, y1 = rng.uniform(-30, in_w + 10, N_FACE), rng.uniform(-30, in_h + 10, N_FACE)
    bb = np.stack([x1, y1, x1 + rng.uniform(-5, 400, N_FACE), y1 + rng.uniform(-5, 400, N_FACE)], 1).astype(F)
    lmk = rng.uniform(-20, 660, (N_FACE, 10)).astype(F)
    s = np.array(SPECIAL, F)
    for i in range(300, 300 + 4 * len(s)):           # every special value in every corner
        bb[i, (i - 300) % 4] = s[(i - 300) // 4]
    for i in range(400, 560):                        # random pairs: l and r (or t and b) both special
        c = int(rng.integers(0, 2))
        bb[i, c], bb[i, c + 2] = rng.choice(s), rng.choice(s)
    lmk[560:570, 3] = np.nan
    lmk[570:575, 0] = np.inf
    lmk[575:580, 9] = -np.inf
    lmk[580:590] = rng.uniform(-3e9, 3e9, (10, 10))
    return bb, lmk


def lib_faces(in_w, in_h, img_w, img_h, bb, lmk):
    lib = L.load()
    rects = np.zeros((len(bb), 4), np.int32)
    mapped = np.ascontiguousarray(lmk, F).copy()
    r = (C.c_int * 4)()
    for i in range(len(bb)):
        b = (C.c_float * 4)(*[float(v) for v in bb[i]])
        assert lib.trtx_retina_get_rect_adapt_landmark(in_w, in_h, img_w, img_h, b,
                                                       mapped[i].ctypes.data_as(C.POINTER(C.c_float)), r) == 0
        rects[i] = list(r)
    return rects, mapped


def ref_faces(lib, in_w, in_h, img_w, img_h, bb, lmk):
    rects = np.zeros((len(bb), 4), np.int32)
    mapped = np.ascontiguousarray(lmk, F).copy()
    for i in range(len(bb)):
        b = np.ascontiguousarray(bb[i], F).copy()
        lib.ref_retina_get_rect_adapt_landmark(img_w, img_h, in_w, in_h, b.ctypes.data_as(C.c_void_p),
                                               mapped[i].ctypes.data_as(C.c_void_p), rects[i].ctypes.data_as(C.c_void_p))
    return rects, mapped


def _ref_retina():
    return [(opt, RefOutputs.lib(name)) for opt, name in (("O2", "libref_retina_host.so"), ("O0", "libref_retina_host_O0.so"))
            if RefOutputs.lib(name) is not None]


@pytest.mark.parametrize("in_w,in_h", INPUTS)
def test_retina_get_rect_adapt_landmark_equals_reference_undefined_cases(in_w, in_h):
    """trtx_retina_get_rect_adapt_landmark = the reference's compiled get_rect_adapt_landmark at -O2 and at -O0 on 600 faces
    x 11 frame sizes, every rectangle and every landmark bit, including the corners the reference cannot convert (INT_MIN
    on x86-64) and the widths and heights that overflow (wrap): live where oracle/_ref was built, else the stored digests."""
    refs = _ref_retina()
    undefined = wrapped = 0
    for w, h in SIZES:
        bb, lmk = face_cases(in_w, in_h, w, h)
        got_r, got_k = lib_faces(in_w, in_h, w, h, bb, lmk)
        key = f"face.{in_w}x{in_h}.{w}x{h}"
        if not refs:
            G.equal(key + ".rect", got_r)
            G.equal(key + ".lmk", got_k.view(np.int32))
        for opt, ref in refs:
            want_r, want_k = ref_faces(ref, in_w, in_h, w, h, bb, lmk)
            G.equal(key + ".rect", got_r, ref=want_r, msg=opt)
            G.equal(key + ".lmk", got_k.view(np.int32), ref=want_k.view(np.int32), msg=opt)   # bit for bit, NaN payloads too
            undefined += int((got_r[:, :2] == INT_MIN).sum())
            l, t, wd, ht = (got_r[:, k].astype(np.int64) for k in range(4))
            r, b = l + wd, t + ht
            wrapped += int(((r < INT_MIN) | (r > 2 ** 31 - 1) | (b < INT_MIN) | (b > 2 ** 31 - 1)).sum())
    if refs:
        assert undefined > 100 and wrapped > 10, (undefined, wrapped)


def test_retina_definitions():
    """The definitions stated in trtx_hot.h, without the reference: a corner that is NaN, infinite or outside the int range
    is INT_MIN; w = r - l wraps modulo 2^32; an ordinary corner truncates toward zero and is not clamped."""
    def face(box, img=(1920, 1080)):
        return lib_faces(640, 640, img[0], img[1], np.array([box], F), np.zeros((1, 10), F))[0][0].tolist()

    assert face((np.nan, 10, 20, 30))[0] == INT_MIN
    assert face((10, np.inf, 20, 30))[1] == INT_MIN
    assert face((-1e30, 10, 20, 30))[0] == INT_MIN
    # 1920x1080 in 640x640: r_w = 1/3, so x = 7e8 maps to 2.1e9 and x = -7e8 to -2.1e9: r - l = 4.2e9 wraps
    l, _, w, _ = face((-7e8, 10, 7e8, 30))
    r_w = F(640 / 1920.0)
    want_l, want_r = int(F(-7e8) / r_w), int(F(7e8) / r_w)
    assert l == want_l and w == (want_r - want_l + 2 ** 31) % 2 ** 32 - 2 ** 31 and w < 0
    # truncation toward zero, no clamp: x = -1.5 / r_w -> -4 (not -5, not 0)
    assert face((F(-1.5), 10, 20, 30))[0] == int(F(-1.5) / r_w) == -4


def test_get_corner_equals_yolo26_draw_bbox_obb():
    """trtx_get_corner at net 1024 = the corners yolo26's own draw_bbox_obb (get_corner over get_rect_obb) hands to
    cv::polylines, for every box of test_pose_obb_post_cpu's 2,500 x 11 frame sizes whose get_rect is defined (NaN and
    infinite angles, wrapping centres and h >= w swaps included): live where oracle/_ref was built (also yolo26's 3 debug
    lines per box), else the stored digests."""
    ref = FO.load_obb26()
    T.check_corners(G, "v26", 1024, None if ref is None else lambda w, h, b: FO.ref_draw_bbox_obb_v26(w, h, b))


def test_inputs_640x480_and_640x640_give_different_faces():
    """The two input sizes pin different mappings: on the same faces, trtx_retina_get_rect_adapt_landmark at 640x480 and at
    640x640 differs on every frame size."""
    for w, h in SIZES:
        bb, lmk = face_cases(640, 480, w, h)
        a_r, a_k = lib_faces(640, 480, w, h, bb, lmk)
        b_r, b_k = lib_faces(640, 640, w, h, bb, lmk)
        assert not (np.array_equal(a_r, b_r) and np.array_equal(a_k.view(np.int32), b_k.view(np.int32))), (w, h)


def test_conf_threshold_as_float():
    """CONF_THRESH is a double literal: c < T exactly when c < the smallest float >= T."""
    assert P.float_ge_threshold(0.75) == 0.75
    t = P.float_ge_threshold(0.1)
    assert F(t) == t and t >= 0.1 and float(np.nextafter(F(t), F(0))) < 0.1
    for c in (np.nextafter(F(t), F(0)), F(t), np.nextafter(F(t), F(1))):
        assert (float(c) < 0.1) == (c < F(t))
    assert P.float_ge_threshold(-math.inf) == -math.inf


def _fake(n):
    return C.c_void_p(0x1000 * n)


def test_face_argument_validation():
    """Rejected before anything is launched (the device pointers here are never dereferenced)."""
    lib = L.load()
    assert lib.trtx_abi_sizeof(9) == C.sizeof(L.FacePostParams) == 24
    INV = L.ERR_INVALID

    def call(sizes=((1920, 1080),), batch=None, dets=_fake(1), max_rows=10, rows=_fake(2), **kw):
        q = L.FacePostParams(L.RETINA_FACE, 640, 480, 17, 7, 0.75)
        for k, v in kw.items():
            setattr(q, k, v)
        wh = (C.c_int32 * max(2 * len(sizes), 2))(*[v for s in sizes for v in s])
        return lib.trtx_retina_postprocess_enqueue(C.byref(q), wh, len(sizes) if batch is None else batch, dets, max_rows,
                                                   rows, None)

    assert lib.trtx_retina_postprocess_enqueue(None, None, 1, _fake(1), 10, _fake(2), None) == INV
    q = L.FacePostParams(L.RETINA_FACE, 640, 480, 17, 7, 0.75)
    assert lib.trtx_retina_postprocess_enqueue(C.byref(q), None, 1, _fake(1), 10, _fake(2), None) == INV
    assert call(batch=0) == INV
    assert call(max_rows=0) == INV
    assert call(dets=None) == INV
    assert call(rows=None) == INV
    assert call(variant=2) == INV
    assert call(variant=-1) == INV
    assert call(in_w=0) == INV
    assert call(in_h=-640) == INV
    assert call(row_floats=6, lmk_offset=0) == INV                          # the keep flag is float 6
    assert call(lmk_offset=8) == INV                                        # 8 + 10 > 17
    assert call(lmk_offset=-1) == INV
    assert call(variant=L.RETINA_ANTICOV) == INV                            # mask_confidence would be float 17 of 17
    assert call(variant=L.RETINA_ANTICOV, row_floats=18, lmk_offset=8) == INV
    assert call(sizes=((1920, 1080), (0, 5))) == INV
    assert call(sizes=((1920, 1080), (5, -1))) == INV


def test_obb_nms_free_argument_validation():
    """TASK_OBB_NMS_FREE takes yolo26's plugin rows, whose angle is the last float; rejected before any launch otherwise."""
    lib = L.load()
    assert L.TASK_OBB_NMS_FREE == 3

    def call(row_floats=90, extra_offset=89, sizes=((1920, 1080),)):
        q = L.PoseObbParams(L.TASK_OBB_NMS_FREE, 1024, 1024, row_floats, extra_offset, 0)
        wh = (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])
        return lib.trtx_yolo_pose_obb_postprocess_enqueue(C.byref(q), wh, len(sizes), _fake(1), 10, _fake(2), None)

    assert call(extra_offset=7) == L.ERR_INVALID
    assert call(extra_offset=90) == L.ERR_INVALID
    assert call(row_floats=6, extra_offset=5) == L.ERR_INVALID
    assert call(sizes=((1920, 1080), (0, 1))) == L.ERR_INVALID
