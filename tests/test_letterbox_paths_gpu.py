"""Every path of the letterbox pre-process (trtx_preprocess_batch_enqueue), bit for bit against the exact CPU model.

The host sends each frame to one of two kernels: letterbox_unit_kernel (TMA row bands) for a scale-1 frame whose base and
row pitch are 16-byte aligned, whose horizontal offset is a multiple of 16 pixels, into a 16-byte aligned dst with dst_w % 4
== 0; letterbox_kernel (fast and general strips) for every other frame.  Each case below names the kernel the rules must
pick, runs in fp32 and fp16, and compares every output with oracle.warpaffine(contracted=True) -- fp16 outputs with that
value rounded to nearest -- bit for bit.  dst is filled with NaN and sits between sentinel elements, so a missed or a stray
write shows.  The kernels that ran, and how often, are read from the names torch.profiler records."""
import ctypes as C
import math
import warnings

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from oracle.golden import RefOutputs
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth
from test_letterbox_paths_cpu import SWEEP, sweep_frame, sweep_key

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_letterbox_gpu")

U, GEN = "unit", "general"
MAX_UNIT, MAX_GENERAL = 64, 128     # frames per launch of each kernel
GUARD = 64                          # sentinel elements on either side of dst
SENTINEL = -3.0


def _dev_frame(fr, dev, pitch=None, lead=0):
    """A device copy of host frame fr [h, w, 3] whose rows are `pitch` bytes apart, `lead` bytes into its buffer (the
    allocation is 256-byte aligned); the bytes between the rows are 0xA5, which no frame row may show."""
    h, w, _ = fr.shape
    pitch = pitch or 3 * w
    buf = torch.full((lead + (h - 1) * pitch + 3 * w,), 0xA5, dtype=torch.uint8, device=dev)
    v = torch.as_strided(buf, (h, w, 3), (pitch, 3, 1), lead)
    v.copy_(torch.from_numpy(np.ascontiguousarray(fr)))
    return v


def _pad16(w):
    return (3 * w + 15) // 16 * 16 + (16 if (3 * w) % 16 == 0 else 0)  # a pitch with padding, multiple of 16


class _Kernels:
    """Counts the letterbox kernels launched inside the block, by the names the profiler records; traced is False where it
    recorded no CUDA activity at all."""

    def __enter__(self):
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        names = [e.name for e in self.prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        self.traced = bool(names)
        self.unit = sum("letterbox_unit_kernel" in n for n in names)
        self.general = sum("letterbox_kernel" in n for n in names)
        return False


def _run(views, dw, dh, odt, dev, shift=0, plan=False):
    """The letterbox of `views` into a [B, 3, dh, dw] dst `shift` elements past a 256-byte boundary -> (dst on the host,
    _Kernels).  Asserts that no element around dst changed."""
    B = len(views)
    n = B * 3 * dh * dw
    buf = torch.full((GUARD + shift + n + GUARD,), SENTINEL, dtype=odt, device=dev)
    dst = buf[GUARD + shift:GUARD + shift + n].view(B, 3, dh, dw)
    dst.fill_(float("nan"))
    torch.cuda.synchronize()
    with _Kernels() as k:
        if plan:
            P.PreprocessPlan(views, dst, dw, dh).enqueue()
        else:
            P.cuda_batch_preprocess(views, dst, dw, dh)
    out = buf.cpu()
    assert torch.all(out[:GUARD + shift] == SENTINEL) and torch.all(out[GUARD + shift + n:] == SENTINEL), "stray write"
    return out[GUARD + shift:GUARD + shift + n].view(B, 3, dh, dw).numpy(), k


def _model(oracle, fr, dw, dh, odt):
    m = oracle.warpaffine(fr, dw, dh, contracted=True)
    return m if odt == torch.float32 else m.astype(np.float16)


def _bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint16)


def _expect_exact(oracle, got, frames, dw, dh, odt, cache, what):
    for b, fr in enumerate(frames):
        key = (id(fr), dw, dh, odt)
        if key not in cache:
            cache[key] = _model(oracle, fr, dw, dh, odt)
        ref = cache[key]
        bad = _bits(got[b]) != _bits(ref)
        assert not bad.any(), (what, b, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def _expect_launches(runs):
    """runs: (_Kernels, kind per frame) of each call of a test.  Each call launches ceil(n / 64) unit and ceil(n / 128) general
    kernels for its n frames of each kind.  A call in whose window the profiler recorded no CUDA activity at all is not judged
    (CUPTI can drop a window's records); the test skips, once the outputs are checked, where no window was recorded."""
    traced = [(k, kinds) for k, kinds in runs if k.traced]
    if not traced:
        pytest.skip("torch.profiler recorded no CUDA kernel on this machine (no CUPTI activity tracing): outputs were checked, "
                    "the kernel choice was not")
    if len(traced) < len(runs):
        warnings.warn(f"{len(runs) - len(traced)} of {len(runs)} profiler windows recorded nothing; the others were checked")
    for k, kinds in traced:
        nu, ng = kinds.count(U), kinds.count(GEN)
        assert (k.unit, k.general) == (math.ceil(nu / MAX_UNIT), math.ceil(ng / MAX_GENERAL)), (k.unit, k.general, nu, ng)


# ----------------------------------------------------------------------------------------------------------------------
# Cases: build(dev) -> (host frames (the model's input, may be pitched views), device views, dst w, dst h, kind per frame)
def _single(h, w, pitch=None, seed=None):
    def build(dev):
        fr = synth.frames(1, seed=seed if seed is not None else 31 * h + w, h=h, w=w)[0]
        return [fr], [_dev_frame(fr, dev, pitch)]
    return build


def _crops(boxes, h=1080, w=1920, seed=3):
    """crops (x, y, cw, ch) of one pitched frame"""
    def build(dev):
        big = synth.frames(1, seed=seed, h=h, w=w)[0]
        bd = _dev_frame(big, dev, pitch=3 * w + 64)
        return [big[y:y + ch, x:x + cw] for x, y, cw, ch in boxes], [bd[y:y + ch, x:x + cw] for x, y, cw, ch in boxes]
    return build


def _batch(B, h, w, spaced=False, seed=17):
    """B frames in one [B, h, w, 3] tensor, or each in a buffer of its own"""
    def build(dev):
        fr = synth.frames(B, seed=seed, h=h, w=w)
        if spaced:
            return list(fr), [_dev_frame(f, dev, lead=16 * (i % 5)) for i, f in enumerate(fr)]
        return list(fr), list(torch.from_numpy(fr).to(dev).unbind(0))
    return build


def _repeated(dev):
    fr = synth.frames(1, seed=23, h=480, w=640)[0]
    v = _dev_frame(fr, dev)
    return [fr] * 3, [v, v, v]


def _reversed(dev):
    fr = synth.frames(5, seed=29, h=480, w=640)
    return list(fr[::-1]), list(torch.from_numpy(fr).to(dev).unbind(0))[::-1]


UNIT_CASES = {
    # lx = 0 / ly = 0: odd width / height, reachable only with a padded pitch
    "607x640_padded": (_single(640, 607, pitch=_pad16(607)), 640, 640),
    "640x607_padded": (_single(607, 640, pitch=_pad16(640)), 640, 640),
    "crops_x16_of_1920x1080": (_crops([(0, 0, 640, 480), (16, 100, 640, 480), (640, 300, 640, 480), (1280, 600, 640, 480)]),
                               640, 640),
    "portrait_320x640": (_single(640, 320), 640, 640),           # left boxes wholly outside the image
    "dst_320x320": (_single(240, 320), 320, 320),                 # CTAs narrower than 160 threads
    "dst_644x644_padded": (_single(484, 644, pitch=_pad16(644)), 644, 644),
    "dst_1280x1280": (_single(720, 1280), 1280, 1280),           # the column loop
    "dst_640x642": (_single(480, 640), 640, 642),                 # a last band of 2 rows
    "dst_16x16": (_single(9, 16), 16, 16),
    "b70_one_tensor": (_batch(70, 480, 640), 640, 640),           # one tensor map, two launches
    "b70_per_frame_maps": (_batch(70, 416, 640, spaced=True), 640, 640),
    "one_buffer_3_times": (_repeated, 640, 640),
    "reversed_unbind": (_reversed, 640, 640),
    "overlapping_crops": (_crops([(0, 0, 640, 480), (16, 0, 640, 480), (32, 0, 640, 480)]), 640, 640),
}


@pytest.mark.parametrize("case", list(UNIT_CASES))
def test_unit_kernel_cases(oracle, dev, case):
    """Each case on the unit kernel, then with dst 1 element past 16-byte alignment, which sends the same frames to the
    general kernel: both equal the model, hence each other."""
    build, dw, dh = UNIT_CASES[case]
    frames, views = build(dev)
    cache, traced = {}, []
    for odt in (torch.float32, torch.float16):
        got, k = _run(views, dw, dh, odt, dev)
        _expect_exact(oracle, got, frames, dw, dh, odt, cache, (case, odt))
        shifted, ks = _run(views, dw, dh, odt, dev, shift=1)
        _expect_exact(oracle, shifted, frames, dw, dh, odt, cache, (case, odt, "shifted"))
        assert np.array_equal(_bits(got), _bits(shifted))
        traced += [(k, [U] * len(views)), (ks, [GEN] * len(views))]
    _expect_launches(traced)


def _solid(h, w, v):
    def build(dev):
        fr = np.full((h, w, 3), v, np.uint8)
        return [fr], [_dev_frame(fr, dev)]
    return build


def _checker(h, w, cell=1):
    def build(dev):
        y, x = np.mgrid[0:h, 0:w]
        fr = np.repeat((((y // cell + x // cell) & 1) * 255).astype(np.uint8)[:, :, None], 3, axis=2)
        fr[:, :, 1] = 255 - fr[:, :, 1]
        return [fr], [_dev_frame(fr, dev)]
    return build


def _unaligned_crop(dev):
    return _crops([(1, 0, 640, 480), (5, 7, 640, 480)])(dev)


GENERAL_CASES = {
    # scale 1, but not for the unit kernel
    "crop_x1_and_x5": (_unaligned_crop, 640, 640),
    "packed_500_wide": (_single(640, 500), 640, 640),             # pitch 1500: not a multiple of 16
    "624_wide": (_single(640, 624), 640, 640),                    # horizontal offset 8 pixels
    "dst_w_638_scale_1": (_single(480, 638), 638, 640),          # dst_w % 4 != 0
    # shrinks
    "1080x1920": (_single(1080, 1920), 640, 640),
    "3000x4000": (_single(3000, 4000), 640, 640),
    "1x4000": (_single(1, 4000), 640, 640),
    "4000x1": (_single(4000, 1), 640, 640),
    # enlargements (600x600: fast and general strips in one image)
    "33x47": (_single(33, 47), 640, 640),
    "1x1": (_single(1, 1), 640, 640),
    "600x600": (_single(600, 600), 640, 640),
    "660x660": (_single(660, 660), 640, 640),
    # other dst sizes
    "dst_608x416": (_batch(3, 1080, 1920, seed=41), 608, 416),
    "dst_638x640": (_batch(2, 720, 1280, seed=43), 638, 640),
    "dst_333x517": (_batch(2, 480, 640, seed=47), 333, 517),
    # flat and worst-case frames
    "all_0": (_solid(720, 1280, 0), 640, 640),
    "all_255": (_solid(600, 600, 255), 640, 640),
    "checkerboard": (_checker(720, 1280), 640, 640),
    "checkerboard_600": (_checker(600, 600, 3), 640, 640),
    # two launches
    "b130": (_batch(130, 96, 128, seed=53), 640, 640),
}


@pytest.mark.parametrize("case", list(GENERAL_CASES))
def test_general_kernel_cases(oracle, dev, case):
    build, dw, dh = GENERAL_CASES[case]
    frames, views = build(dev)
    cache, traced = {}, []
    for odt in (torch.float32, torch.float16):
        for shift in (0, 1):
            got, k = _run(views, dw, dh, odt, dev, shift=shift)
            _expect_exact(oracle, got, frames, dw, dh, odt, cache, (case, odt, shift))
            traced.append((k, [GEN] * len(views)))
    _expect_launches(traced)


def test_unit_and_general_frames_interleaved(oracle, dev):
    """70 unit and 70 general frames alternating in one call: two unit launches (the first flushed at 64 while general
    frames are still being collected), one general launch, every frame in its own slot."""
    uni = synth.frames(70, seed=61, h=480, w=640)
    gen = synth.frames(70, seed=62, h=48, w=64)
    ud = list(torch.from_numpy(uni).to(dev).unbind(0))
    gd = list(torch.from_numpy(gen).to(dev).unbind(0))
    frames, views, kinds = [], [], []
    for i in range(70):
        frames += [uni[i], gen[i]]
        views += [ud[i], gd[i]]
        kinds += [U, GEN]
    cache, traced = {}, []
    for odt in (torch.float32, torch.float16):
        got, k = _run(views, 640, 640, odt, dev, plan=odt == torch.float16)
        _expect_exact(oracle, got, frames, 640, 640, odt, cache, odt)
        traced.append((k, kinds))
    _expect_launches(traced)


def test_plan_replayed_from_a_cuda_graph_reads_the_new_frames(oracle, dev):
    """PreprocessPlan.enqueue captured in a CUDA graph, as the pipeline and the benchmark run it: after the frame buffers
    are overwritten in place, a replay letterboxes the new bytes (unit frames through a tensor map made at capture time)."""
    uni = torch.empty((4, 480, 640, 3), dtype=torch.uint8, device=dev)
    big = torch.empty((2, 1080, 1920, 3), dtype=torch.uint8, device=dev)
    views = list(uni.unbind(0)) + list(big.unbind(0))
    for odt in (torch.float32, torch.float16):
        dst = torch.full((6, 3, 640, 640), float("nan"), dtype=odt, device=dev)
        plan = P.PreprocessPlan(views, dst, 640, 640)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            plan.enqueue()
        for seed in (71, 72):
            a, b = synth.frames(4, seed=seed, h=480, w=640), synth.frames(2, seed=seed + 10, h=1080, w=1920)
            uni.copy_(torch.from_numpy(a))
            big.copy_(torch.from_numpy(b))
            dst.fill_(float("nan"))
            g.replay()
            torch.cuda.synchronize()
            _expect_exact(oracle, dst.cpu().numpy(), list(a) + list(b), 640, 640, odt, {}, (odt, seed))
        del g


def test_letterbox_vs_reference_sweep(dev, oracle):
    """The reference's cuda_preprocess (oracle/_ref/libref_yolov8.so) on other dst sizes and shrink ratios: ours equals it
    bit for bit, live where the library was built and through tests/golden/ref_letterbox_gpu.npz elsewhere."""
    lib = G.lib("libref_yolov8.so")
    for h, w, dw, dh in SWEEP:
        img = sweep_frame(h, w)
        ref = None
        if lib is not None:
            r = torch.zeros((3, dh, dw), dtype=torch.float32, device=dev)
            assert lib.ref_v8_preprocess(img.ctypes.data_as(C.c_void_p), w, h, C.c_void_p(r.data_ptr()), dw, dh, None) == 0
            ref = r.cpu().numpy()
        dst = torch.zeros((1, 3, dh, dw), dtype=torch.float32, device=dev)
        P.cuda_batch_preprocess([torch.from_numpy(img).to(dev)], dst, dw, dh)
        G.equal(sweep_key(h, w, dw, dh), dst[0].cpu().numpy(), ref, msg=(h, w, dw, dh))
