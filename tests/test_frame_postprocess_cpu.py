"""The contract the per-frame post-processes share, through ctypes: the call, its parameters, every frame size or descriptor
and the workspace's alignment are checked first (TRTX_ERR_INVALID), then the parameter and per-frame limits
(TRTX_ERR_UNSUPPORTED), then the workspace's size (TRTX_ERR_WORKSPACE), all before the first launch.  So a call that fails
two ways is TRTX_ERR_INVALID whichever frame fails first, and a bad frame past the first 64-frame launch still leaves
nothing written.  The pointers are fake: every call here is rejected before a launch (one would fail with TRTX_ERR_CUDA on
a machine without a GPU)."""
import ctypes as C

import pytest

from tensorrtx_b200 import _lib as L

P = 4096        # a fake device pointer, 256-byte aligned
BIG = 1 << 40   # workspace bytes no call here outgrows
FRAME = (640, 480)
HUGE_SIDE = (1 << 24) + 1


def _wh(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


def _frames(sizes):
    d = (L.Frame * len(sizes))()
    for i, (w, h) in enumerate(sizes):
        d[i].img_w, d[i].img_h, d[i].masks_dev, d[i].pitch = w, h, P, max(w, 1)
    return d


def _pose(sizes):
    q = L.PoseObbParams(L.TASK_POSE, 640, 640, 57, 6, 17)
    return L.load().trtx_yolo_pose_obb_postprocess_enqueue(C.byref(q), _wh(sizes), len(sizes), P, 100, P, None)


def _face(sizes):
    q = L.FacePostParams(L.RETINA_FACE, 640, 480, 17, 7, 0.5)
    return L.load().trtx_retina_postprocess_enqueue(C.byref(q), _wh(sizes), len(sizes), P, 100, P, None)


def _topk(sizes):
    q = L.YoloTopkParams(L.YOLO_V8, 640, 640, 6, 0.25)
    return L.load().trtx_yolo_topk_postprocess_enqueue(C.byref(q), _wh(sizes), len(sizes), P, 100, P, None)


def _detr(sizes, queries=100):
    q = L.DetrPostParams(queries, 92, 0.7)
    return L.load().trtx_detr_postprocess_enqueue(C.byref(q), _wh(sizes), len(sizes), P, P, P, None)


def _ufld(sizes):
    q = L.UfldPostParams(101, 56, 4, 800, 288, 8)
    anchors = (C.c_int32 * 56)(*range(64, 288, 4))
    return L.load().trtx_ufld_postprocess_enqueue(C.byref(q), anchors, _wh(sizes), len(sizes), P, P, None)


def _pyrunner(sizes, max_rows=1000):
    q = L.PyrunnerParams(L.BOX_LTRB, 640, 640, 6, 5, -1, 0.5, 0.4)
    return L.load().trtx_pyrunner_postprocess_enqueue(C.byref(q), _wh(sizes), len(sizes), P, max_rows, P, None)


def _centernet(sizes, classes=80, ws=P, ws_bytes=BIG):
    q = L.CenternetParams(classes, 128, 128, 100, 512, 4, 0.5)
    return L.load().trtx_centernet_decode_enqueue(C.byref(q), len(sizes), P, P, P, ws, ws_bytes, P, _wh(sizes), P, None)


def _refinedet(sizes, top_k=1000, ws=P, ws_bytes=BIG):
    q = L.RefinedetParams(320, 25, 0.01, 0.01, 0.45, top_k, 24000, 0.2)
    return L.load().trtx_refinedet_postprocess_enqueue(C.byref(q), len(sizes), P, P, P, P, ws, ws_bytes, P, _wh(sizes), P,
                                                       None)


def _seg(sizes, mask_side=160):
    q = L.MaskParams(L.YOLO_V8, 640, 640, mask_side, mask_side, 32, 38, 6, 100)
    return L.load().trtx_yolo_seg_postprocess_enqueue(C.byref(q), _frames(sizes), len(sizes), P, P, 100, P, None)


def _rcnn_frames(sizes, max_masks=100):
    q = L.RcnnPostParams(1344, 1344, 0, 0, 100, 28, max_masks, 0.6)
    return L.load().trtx_rcnn_postprocess_frames_enqueue(C.byref(q), _frames(sizes), len(sizes), P, P, P, P, P, None)


def _contours(sizes):
    q = L.RcnnPostParams(1344, 1344, 0, 0, 100, 28, 100, 0.6)
    return L.load().trtx_rcnn_contours_enqueue(C.byref(q), _frames(sizes), len(sizes), P, 16, 256, P, P, P, P, BIG, None)


def _yolop(sizes):
    q = L.YolopPostParams(640, 640, 640, 640, 7)
    return L.load().trtx_yolop_postprocess_enqueue(C.byref(q), _frames(sizes), len(sizes), P, 100, P, P, P, None)


ENTRIES = {
    "pose_obb": _pose, "face": _face, "topk": _topk, "detr": _detr, "ufld": _ufld, "pyrunner": _pyrunner,
    "centernet": _centernet, "refinedet": _refinedet, "seg": _seg, "rcnn_frames": _rcnn_frames, "contours": _contours,
    "yolop": _yolop,
}

# (entry, keyword arguments, frame 0): a call of frame 0 alone is TRTX_ERR_UNSUPPORTED, by a parameter limit or frame 0's size
UNSUPPORTED = {
    "detr_queries": ("detr", {"queries": HUGE_SIDE}, FRAME),
    "ufld_side": ("ufld", {}, (HUGE_SIDE, 720)),
    "pyrunner_rows": ("pyrunner", {"max_rows": 4096}, FRAME),
    "centernet_classes": ("centernet", {"classes": 2048}, FRAME),
    "refinedet_side": ("refinedet", {}, (HUGE_SIDE, 480)),
    "refinedet_top_k": ("refinedet", {"top_k": 2048}, FRAME),
    "seg_mask_side": ("seg", {"mask_side": 100}, FRAME),
    "rcnn_frames_ctas": ("rcnn_frames", {"max_masks": 1 << 30}, (1000, 1000)),
    "contours_area": ("contours", {}, (30000, 30000)),
    "yolop_smem": ("yolop", {}, (100000, 480)),
}


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_bad_frame_past_the_first_launch_is_invalid(entry):
    """Frame 64, the first of the second launch, has width 0: the call is refused before the first launch."""
    sizes = [FRAME] * 64 + [(0, 480)]
    assert ENTRIES[entry](sizes) == L.ERR_INVALID


@pytest.mark.parametrize("case", list(UNSUPPORTED))
def test_invalid_frame_wins_over_unsupported_call(case):
    entry, kw, frame0 = UNSUPPORTED[case]
    fn = ENTRIES[entry]
    assert fn([frame0], **kw) == L.ERR_UNSUPPORTED
    assert fn([frame0, (0, 480)], **kw) == L.ERR_INVALID


@pytest.mark.parametrize("entry", ["centernet", "refinedet"])
def test_misaligned_workspace_wins_over_small_workspace(entry):
    fn = ENTRIES[entry]
    assert fn([FRAME], ws_bytes=0) == L.ERR_WORKSPACE
    assert fn([FRAME], ws=P + 16, ws_bytes=0) == L.ERR_INVALID
