"""The exact CPU model of the letterbox pre-process (trtx_preprocess_batch_enqueue), and its argument checks, without a device.

The model is the oracle's warpaffine with contracted=True: the reference's arithmetic with the bilinear sum evaluated as nvcc's
default FMA contraction evaluates it, fmaf(w4, v4, fmaf(w3, v3, fmaf(w1, v1, w2 * v2))), in the reference's compiled
warpaffine_kernel and in both paths of letterbox_kernel.  It is pinned here to the reference's own outputs (digests recorded
on the GPU from oracle/_ref/libref_yolov8.so), and tests/test_letterbox_paths_gpu.py holds every kernel path to it bit for
bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.golden import RefOutputs, digest
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

INV = L.ERR_INVALID

# (src h, src w): the frames of test_vs_reference_gpu.py::test_preprocess_vs_reference_kernel, into 640 x 640
REF_640 = [(640, 640), (1080, 1920), (375, 500), (480, 640), (640, 480), (416, 640), (640, 500), (639, 640), (640, 624)]

# (src h, src w, dst w, dst h): other destination sizes and shrink ratios, run through the reference's cuda_preprocess on the
# GPU (test_letterbox_paths_gpu.py::test_letterbox_vs_reference_sweep); every frame fits the reference's staging buffer
# (kMaxInputImageSize = 3000 x 3000 pixels)
SWEEP = [(1080, 1920, 320, 320), (1080, 1920, 1280, 1280), (1080, 1920, 608, 416), (720, 1280, 416, 608),
         (3000, 3000, 640, 640), (2999, 1999, 640, 640), (2160, 3840, 640, 640), (480, 640, 333, 517),
         (600, 600, 640, 640), (660, 660, 640, 640), (33, 47, 320, 320), (1, 2999, 640, 640), (2999, 1, 640, 640),
         (517, 333, 1280, 1280)]


def sweep_key(h, w, dw, dh):
    return f"letterbox.{h}x{w}.{dw}x{dh}"


def sweep_frame(h, w):
    return synth.frames(1, seed=7919 + 3 * h + w, h=h, w=w)[0]


def test_model_reproduces_the_reference_at_640(oracle):
    G = RefOutputs("ref_gpu")
    for h, w in REF_640:
        img = synth.frames(1, seed=h, h=h, w=w)[0]
        model = oracle.warpaffine(img, 640, 640, contracted=True)
        assert np.array_equal(digest(model), G.stored[f"preprocess.{h}x{w}"]), (h, w)
    # the plain IEEE restatement is not enough once the image is resampled
    img = synth.frames(1, seed=1080, h=1080, w=1920)[0]
    assert not np.array_equal(oracle.warpaffine(img, 640, 640), oracle.warpaffine(img, 640, 640, contracted=True))


def test_model_reproduces_the_reference_sweep(oracle):
    G = RefOutputs("ref_letterbox_gpu")
    for h, w, dw, dh in SWEEP:
        model = oracle.warpaffine(sweep_frame(h, w), dw, dh, contracted=True)
        assert np.array_equal(digest(model), G.stored[sweep_key(h, w, dw, dh)]), (h, w, dw, dh)


@pytest.mark.parametrize("h,w,dw,dh", [(640, 640, 640, 640), (480, 640, 640, 640), (640, 607, 640, 640), (607, 640, 640, 640),
                                       (640, 320, 640, 640), (720, 1280, 1280, 1280), (240, 320, 320, 320), (9, 16, 16, 16),
                                       (480, 640, 640, 642), (640, 500, 640, 640), (640, 624, 640, 640)])
def test_model_at_scale_1_is_the_uncontracted_oracle(oracle, h, w, dw, dh):
    """At scale 1 every weight is 0, 0.5 or 1 and every partial sum is exact: the order of evaluation does not matter."""
    img = synth.frames(1, seed=h * w + dw, h=h, w=w)[0]
    m = oracle.letterbox_matrix(w, h, dw, dh)
    assert m[0] == m[4] == 1
    model = oracle.warpaffine(img, dw, dh, contracted=True)
    assert np.array_equal(model.view(np.uint32), oracle.warpaffine(img, dw, dh).view(np.uint32))


def test_model_reads_pitched_and_cropped_frames(oracle):
    big = synth.frames(1, seed=5, h=300, w=500)[0]
    padded = np.zeros((300, 512, 3), np.uint8)
    padded[:, :500] = big
    for view, dense in ((padded[:, :500], big), (big[17:250, 33:480], np.ascontiguousarray(big[17:250, 33:480]))):
        for contracted in (False, True):
            got = oracle.warpaffine(view, 320, 320, contracted=contracted)
            assert np.array_equal(got.view(np.uint32), oracle.warpaffine(dense, 320, 320, contracted=contracted).view(np.uint32))


def _fake(n):
    """a non-null address that is never dereferenced: every call below is rejected before the first launch"""
    return 0x10000 * n


def test_c_argument_checks_before_the_first_launch():
    lib = L.load()
    descs = (L.ImageDesc * 2)()
    for i in range(2):
        descs[i].data_dev, descs[i].width, descs[i].height, descs[i].pitch = _fake(1 + i), 640, 480, 1920

    def call(dst=_fake(3), dtype=L.F32, batch=2, dw=640, dh=640):
        return lib.trtx_preprocess_batch_enqueue(descs, batch, dst, dw, dh, dtype, None)

    # dst not aligned to its element size
    assert call(dst=_fake(3) + 2) == call(dst=_fake(3) + 1) == call(dst=_fake(3) + 1, dtype=L.F16) == INV
    assert call(dst=_fake(3) + 3, dtype=L.F16) == INV
    assert call(dtype=2) == call(dtype=-1) == call(dst=None) == call(batch=0) == call(dw=0) == call(dh=-1) == INV
    descs[1].pitch = 1919
    assert call(dst=_fake(3) + 2, dtype=L.F16) == INV                # aligned for halves, but a bad descriptor
    descs[1].pitch, descs[1].data_dev = 1920, None
    assert call() == INV


def test_python_wrappers_check_dst_before_the_call():
    frames = [torch.zeros((48, 64, 3), dtype=torch.uint8) for _ in range(3)]
    for bad in (torch.float64, torch.bfloat16, torch.int32):
        dst = torch.zeros((3, 3, 32, 32), dtype=bad)
        with pytest.raises(L.TrtxError, match="not accepted"):
            P.cuda_batch_preprocess(frames, dst, 32, 32)
        with pytest.raises(L.TrtxError, match="not accepted"):
            P.PreprocessPlan(frames, dst, 32, 32)
    for dt in (torch.float32, torch.float16):
        for shape in ((2, 3, 32, 32), (3, 3, 32, 33), (3, 3, 33, 32), (3, 32, 32, 3), (3, 3 * 32 * 32), (4, 3, 32, 32)):
            dst = torch.zeros(shape, dtype=dt)
            with pytest.raises(ValueError, match=r"\[3, 3, 32, 32\]"):
                P.cuda_batch_preprocess(frames, dst, 32, 32)
            with pytest.raises(ValueError, match=r"\[3, 3, 32, 32\]"):
                P.PreprocessPlan(frames, dst, 32, 32)
        # the right dtype and shape pass the check; these host tensors are then refused as device pointers
        dst = torch.zeros((3, 3, 32, 32), dtype=dt)
        with pytest.raises(L.TrtxError, match="CUDA tensor"):
            P.cuda_batch_preprocess(frames, dst, 32, 32)
        with pytest.raises(L.TrtxError, match="CUDA tensor"):
            P.PreprocessPlan(frames, dst, 32, 32).enqueue()
