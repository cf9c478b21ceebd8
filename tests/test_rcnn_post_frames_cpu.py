"""Mask R-CNN post-process for frames of mixed sizes (trtx_rcnn_postprocess_frames_enqueue) without a GPU: every argument
check returns its error before anything is launched, and the ctypes mirror of trtx_frame has the C layout."""
import ctypes as C
import subprocess
from pathlib import Path

import pytest

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

ROOT = Path(__file__).resolve().parents[1]
OK = dict(net_w=1067, net_h=800, img_w=0, img_h=0, detections_per_im=100, mask_size=14, max_masks=100, score_thresh=0.6)
# scores, boxes, classes, masks, rows: fake device addresses, never dereferenced by a rejected call
PTRS = (16, 32, 48, 64, 80)


def _frames(sizes, canvases=True, pitch_extra=0):
    d = (L.Frame * len(sizes))()
    for i, (w, h) in enumerate(sizes):
        d[i].img_w, d[i].img_h = w, h
        d[i].masks_dev = (4096 * (i + 1)) if canvases else None
        d[i].pitch = w + pitch_extra
    return d


def _call(params=None, frames=None, batch=None, ptrs=PTRS):
    q = L.RcnnPostParams(**{**OK, **(params or {})})
    frames = _frames([(640, 480), (1920, 1080)]) if frames is None else frames
    batch = len(frames) if batch is None else batch
    p = [None if v is None else C.c_void_p(v) for v in ptrs]
    return L.load().trtx_rcnn_postprocess_frames_enqueue(C.byref(q), frames, batch, *p, None)


def test_null_pointers_and_batch():
    lib = L.load()
    inv = L.ERR_INVALID
    frames = _frames([(640, 480)])
    assert lib.trtx_rcnn_postprocess_frames_enqueue(None, frames, 1, *PTRS, None) == inv
    q = L.RcnnPostParams(**OK)
    assert lib.trtx_rcnn_postprocess_frames_enqueue(C.byref(q), None, 1, *PTRS, None) == inv
    assert _call(batch=0) == inv
    assert _call(batch=-2) == inv
    for i in (0, 1, 2, 4):                                  # scores, boxes, classes, rows are required
        ptrs = list(PTRS)
        ptrs[i] = None
        assert _call(ptrs=tuple(ptrs)) == inv, i
        assert _call(frames=_frames([(64, 48)], canvases=False), ptrs=tuple(ptrs)) == inv, i


def test_params():
    inv = L.ERR_INVALID
    for k in ("net_w", "net_h", "detections_per_im", "mask_size", "max_masks"):
        assert _call({k: 0}) == inv, k
        assert _call({k: -3}) == inv, k
    assert _call({"mask_size": 33}) == inv                 # larger than the paste's shared-memory stage
    assert _call({"mask_size": 33}, frames=_frames([(64, 48)], canvases=False)) == inv


def test_frame_sizes_and_pitch():
    inv = L.ERR_INVALID
    for bad in ((0, 480), (640, 0), (-1, 480), (640, -7)):
        assert _call(frames=_frames([(640, 480), bad])) == inv, bad           # checked for every frame, not the first
        assert _call(frames=_frames([(640, 480), bad], canvases=False)) == inv, bad
    f = _frames([(640, 480), (1920, 1080), (17, 23)])
    f[2].pitch = 16                                                           # pitch < img_w
    assert _call(frames=f) == inv
    f[2].pitch = -1
    assert _call(frames=f) == inv


def test_canvases_for_every_frame_or_none():
    inv = L.ERR_INVALID
    f = _frames([(640, 480), (480, 640), (64, 48)])
    f[1].masks_dev = None                                                     # NULL among non-NULL
    assert _call(frames=f) == inv
    f = _frames([(640, 480), (480, 640)], canvases=False)
    f[1].masks_dev = 4096                                                     # non-NULL among NULL
    assert _call(frames=f) == inv
    assert _call(ptrs=(16, 32, 48, None, 80)) == inv                          # canvases without a mask input


def test_grid_over_int_max_is_unsupported():
    # 2^30 slots x 10 bands of a 640 x 480 frame (40 chunks: 6 rows per pass, 48-row bands)
    assert _call({"max_masks": 1 << 30}, frames=_frames([(640, 480)])) == L.ERR_UNSUPPORTED
    # the sum over the frames of one launch counts: 2^24 x 10 CTAs per frame, 13 frames pass INT_MAX
    assert _call({"max_masks": 1 << 24}, frames=_frames([(640, 480)] * 13)) == L.ERR_UNSUPPORTED
    # an invalid frame after the oversized grid is still INVALID: every frame is checked first
    assert _call({"max_masks": 1 << 30}, frames=_frames([(640, 480), (0, 5)])) == L.ERR_INVALID


def test_python_wrapper_validates_shapes():
    import torch

    s, bx, c = torch.zeros((2, 10)), torch.zeros((2, 10, 4)), torch.zeros((2, 10))
    with pytest.raises(ValueError):
        P.rcnn_postprocess_frames(s, bx, c, frames=[(64, 48)], net_w=100, net_h=80)           # 2 rows, 1 frame
    with pytest.raises(ValueError):
        P.rcnn_postprocess_frames(s, bx[:, :5], c, frames=[(64, 48), (48, 64)], net_w=100, net_h=80)
    with pytest.raises(ValueError):
        P.rcnn_postprocess_frames(s, bx, c, torch.zeros((2, 10, 14, 14)), frames=[(64, 48), (48, 64)], net_w=100, net_h=80,
                                  canvases=[torch.zeros((10, 48, 64), dtype=torch.uint8)])   # one canvas for two frames
    with pytest.raises(ValueError):
        P.rcnn_postprocess_frames(s, bx, c, torch.zeros((2, 10, 14, 14)), frames=[(64, 48), (48, 64)], net_w=100, net_h=80,
                                  canvases=[torch.zeros((10, 48, 64), dtype=torch.uint8),
                                            torch.zeros((10, 48, 64), dtype=torch.uint8)])   # frame 1 is 48 x 64


def test_rcnn_image_layout_equals_the_mirror(tmp_path):
    """trtx_frame has the layout of the ctypes mirror, and the earlier names trtx_seg_image and trtx_rcnn_image are the
    same type (a pointer to one assigns to a pointer to the other under -Werror)."""
    assert L.load().trtx_abi_sizeof(8) == L.load().trtx_abi_sizeof(6) == C.sizeof(L.Frame) == 24
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "trtx_hot.h"\nint main(void) {\n'
                   '  trtx_rcnn_image r = {0};\n  trtx_seg_image* s = &r;\n  trtx_frame* f = s;\n  (void)f;\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(trtx_frame), offsetof(trtx_frame, img_w),\n'
                   '         offsetof(trtx_frame, img_h), offsetof(trtx_frame, masks_dev),\n'
                   '         offsetof(trtx_frame, pitch), offsetof(trtx_frame, reserved));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(L.Frame)] + [getattr(L.Frame, n).offset for n in ("img_w", "img_h", "masks_dev", "pitch", "reserved")]
    assert got == want
