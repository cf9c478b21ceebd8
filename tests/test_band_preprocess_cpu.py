"""The contract the band pre-processes share (trtx_rcnn / cls / yolop / detr / ufld / refinedet / cubic / linear
_preprocess_enqueue), through ctypes: the call and every descriptor are checked first (TRTX_ERR_INVALID), then every frame's
rectangle and every launch's shared memory (TRTX_ERR_UNSUPPORTED), so a call that fails both ways is TRTX_ERR_INVALID
whichever frame fails first.  The pointers are fake: every call here is rejected before a launch."""
import pytest

from tensorrtx_b200 import _lib as L

EMPTY = (1, 5000)  # a frame whose letterbox rectangle is 0 pixels wide: cv::resize throws there


def _descs(*sizes):
    d = (L.ImageDesc * len(sizes))()
    for i, (w, h) in enumerate(sizes):
        d[i].data_dev, d[i].width, d[i].height, d[i].pitch = 4096, w, h, 3 * w
    return d


# (entry, its arguments before the descriptors, after the count, frame 0): frame 0 alone is TRTX_ERR_UNSUPPORTED, by an empty
# rectangle or by a net too wide for the kernel's staged rows
CASES = {
    "rcnn": ("trtx_rcnn_preprocess_enqueue", (), (1067, 800), EMPTY),
    "cls_v8": ("trtx_cls_preprocess_enqueue", (L.YOLO_V8,), (5000, 8), (640, 480)),
    "cls_v5": ("trtx_cls_preprocess_enqueue", (L.YOLO_V5,), (224, 224), EMPTY),
    "yolop": ("trtx_yolop_preprocess_enqueue", (), (640, 384), EMPTY),
    "detr": ("trtx_detr_preprocess_enqueue", (), (5000, 8), (640, 480)),
    "ufld": ("trtx_ufld_preprocess_enqueue", (), (5000, 8), (640, 480)),
    "refinedet": ("trtx_refinedet_preprocess_enqueue", (), (5000,), (640, 480)),
    "cubic_yolov3_tiny": ("trtx_cubic_preprocess_enqueue", (L.CUBIC_YOLOV3_TINY,), (608, 608), EMPTY),
    "cubic_anticov": ("trtx_cubic_preprocess_enqueue", (L.CUBIC_ANTICOV,), (640, 640), EMPTY),
    "linear_yolov3": ("trtx_linear_preprocess_enqueue", (L.LINEAR_YOLOV3,), (608, 608, 608), EMPTY),
    "linear_retina": ("trtx_linear_preprocess_enqueue", (L.LINEAR_RETINA,), (640, 480, 0), EMPTY),
    "linear_yolov3_spp": ("trtx_linear_preprocess_enqueue", (L.LINEAR_YOLOV3_SPP,), (608, 608, 608), EMPTY),
    "linear_py": ("trtx_linear_preprocess_enqueue", (L.LINEAR_PY,), (640, 640, 0), EMPTY),
}


@pytest.mark.parametrize("case", list(CASES))
def test_invalid_descriptor_wins_over_unsupported_frame(case):
    entry, lead, trail, frame0 = CASES[case]
    fn = getattr(L.load(), entry)
    assert fn(*lead, _descs(frame0), 1, *trail, 4096, None) == L.ERR_UNSUPPORTED
    bad = _descs(frame0, (640, 480))
    bad[1].pitch = 3 * 640 - 1
    assert fn(*lead, bad, 2, *trail, 4096, None) == L.ERR_INVALID


def test_rcnn_rejects_rectangles_past_its_shared_memory():
    """4 840 pixels is the widest R-CNN rectangle: 8 staged int16 rows of 3 * 4 840 plus the band's 128 B of static arrays fill
    the 227 KB opt-in, so 4 841 is refused before anything reaches the device."""
    assert L.load().trtx_rcnn_preprocess_enqueue(_descs((4841, 8)), 1, 4841, 8, 4096, None) == L.ERR_UNSUPPORTED
