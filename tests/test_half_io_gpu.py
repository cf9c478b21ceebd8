"""Half-precision tensors through RoIAlign, MaskRcnnInference and Decode_TRT (include/trtx_hot.h: trtx_roi_align_typed,
trtx_mask_rcnn_inference_typed, trtx_retina_params.in_dtype), the mode an FP16 engine uses so that no reformat copy sits
around the plugins.  Each result is DEFINED by the fp32 mode on the widened halves, so every comparison here is against
the fp32 path (itself pinned to the reference's kernels by tests/test_vs_reference_gpu.py) or the fp32 CPU oracle, fed the
half-rounded inputs -- the way tests/test_yolo_gpu.py::test_v8_fp16_inputs does it."""
import ctypes as C

import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth
from tensorrtx_b200.pipeline import RetinaPipeline

pytestmark = pytest.mark.gpu
ATOL = 1e-4
RTOL_EXP = 2e-6  # columns that pass through expf (CUDA expf vs glibc expf), as tests/test_others_gpu.py
PP = 14


def _roi(dev, rois, feat, sampling, out):
    """RoiAlignPlugin.enqueue in the dtype of `feat` and `out`."""
    B, N = rois.shape[:2]
    _, c, fh, fw = feat.shape
    plug = P.RoiAlignPlugin(PP, 1 / 16, sampling, N, c, fh, fw)
    assert plug.enqueue(B, [rois, feat], [out]) == 0
    torch.cuda.synchronize()
    return out


def _expected_and_got(dev, rois, feat_half, sampling):
    """(half(roi_align_fp32(float(features))), roi_align_half(features)): the two sides of the definition."""
    B, N = rois.shape[:2]
    c = feat_half.shape[1]
    ref = _roi(dev, rois, feat_half.float(), sampling, torch.full((B, N, c, PP, PP), -3.0, device=dev))
    got = _roi(dev, rois, feat_half, sampling, torch.full((B, N, c, PP, PP), -3.0, dtype=torch.float16, device=dev))
    return ref.half(), got


def _assert_same_halves(got, exp, msg=""):
    """bit for bit; NaNs (degenerate proposals, inf * 0 taps) at the same places"""
    nan = torch.isnan(exp)
    assert torch.equal(torch.isnan(got), nan), msg
    g, e = got.view(torch.int16)[~nan], exp.view(torch.int16)[~nan]
    assert torch.equal(g, e), (msg, int((g != e).sum()))


def _case_rois(rng, B, N):
    """the proposals of test_roi_align_and_mask_rcnn_inference_vs_reference_functions"""
    x1 = rng.uniform(-40, 1000, (B, N)); y1 = rng.uniform(-40, 760, (B, N))
    w = np.exp(rng.uniform(np.log(8), np.log(900), (B, N))); h = np.exp(rng.uniform(np.log(8), np.log(700), (B, N)))
    rois = np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)
    rois[0, 0] = [100, 100, 100, 100]        # zero-size proposal: count = 0 -> NaN
    rois[0, 1] = [300, 300, 200, 250]        # negative size
    rois[1, 0] = [-500, -500, -300, -300]    # entirely outside the feature map
    rois[1, 1] = [0, 0, 1067, 800]           # the whole map: 3350 cells, passes of 8 channels at 16 bytes per cell
    rois[1, 2] = [5, 5, 9, 9]                # a fraction of one cell
    rois[1, 3] = [1060, 790, 1200, 900]      # hangs over the bottom-right corner
    return rois


# channels, map height: which kernel trtx_roi_align_typed picks for halves
SHAPES = {"c80.window": (80, 50),            # 64 + 16 channels: the second CTA runs one full tap round of 16
          "c72.window": (72, 50),            # 64 + 8: a multiple of 4 and of 8 but not of the 16 of a tap round -> partial round
          "c76.direct": (76, 50),            # a multiple of 4 (the fp32 window kernel's rule) but not of 8: direct for halves
          "c78.direct": (78, 50),
          "c80.70x67.direct": (80, 70)}      # more than 4096 cells


@pytest.mark.parametrize("sampling", [0, 2, 5, 19])   # 19: 14 * 19 table entries per axis > 256 -> coordinates on the fly
def test_roi_align_half_is_the_rounded_fp32_result_bit_for_bit(dev, oracle, sampling):
    rng = np.random.default_rng(470)
    B, N, W = 2, 96, 67
    rd = torch.from_numpy(_case_rois(rng, B, N)).to(dev)
    for tag, (c, fh) in SHAPES.items():
        feat = torch.from_numpy(rng.standard_normal((B, c, fh, W)).astype(np.float32)).to(dev).half()
        exp, got = _expected_and_got(dev, rd, feat, sampling)
        assert not torch.isnan(exp[1]).any() and (sampling > 0 or torch.isnan(exp[0, 0]).all())   # zero-size proposal: 0 / 0
        _assert_same_halves(got, exp, (tag, sampling))
    if sampling > 2:
        return
    # and against the CPU oracle (no FMA contraction: a few fp32 ulps) on proposals inside the map, within half rounding
    xi = rng.uniform(0, 700, N); yi = rng.uniform(0, 500, N)
    wi = np.exp(rng.uniform(np.log(8), np.log(300), N)); hi = np.exp(rng.uniform(np.log(8), np.log(250), N))
    rois_in = np.stack([xi, yi, xi + wi, yi + hi], -1).astype(np.float32)
    feat = rng.standard_normal((1, 80, 50, W)).astype(np.float16)
    orc = oracle.roi_align(rois_in, feat[0].astype(np.float32), PP, 1 / 16, sampling)
    got = _roi(dev, torch.from_numpy(rois_in[None]).to(dev), torch.from_numpy(feat).to(dev), sampling,
               torch.empty((1, N, 80, PP, PP), dtype=torch.float16, device=dev))
    np.testing.assert_allclose(got[0].float().cpu().numpy(), orc, rtol=2.0 ** -11, atol=2e-5)


@pytest.mark.parametrize("fh", [50, 70], ids=["window", "direct"])
def test_roi_align_half_final_rounding(dev, fh):
    """The one rounding of the half mode, at its edges: bins that round to half subnormals and to zero, bins at +-65504 (a
    bin is a convex combination of taps, so a finite bin never exceeds the largest half: it cannot overflow), and +-inf taps
    (inf bins; NaN where a zero weight meets an inf), all equal to torch's round-to-nearest-even of the fp32 bins."""
    rng = np.random.default_rng(471)
    B, N, c, W = 2, 64, 16, 67
    feat = rng.standard_normal((B, c, fh, W)).astype(np.float32)
    feat[:, 0] *= 1e-5           # subnormal halves in (taps) and out
    feat[:, 1] *= 3e-8           # around the smallest subnormal 5.96e-8: ties between 0 and the first subnormal
    feat[:, 2] *= 6.1e-5         # across the normal / subnormal boundary
    feat[:, 3] = 65504.0
    feat[:, 4] = -65504.0
    feat[:, 5] = np.where(rng.random((B, fh, W)) < 0.5, 65504.0, 65472.0)
    feat[:, 6] = np.inf
    feat[:, 7] = -np.inf
    feat[:, 8] = np.where(rng.random((B, fh, W)) < 0.05, np.inf, feat[:, 8])
    feat[:, 9] *= 30000.0        # overflows to +-inf when narrowed to the half INPUT
    rois = _case_rois(rng, B, N)
    rois[0, 2] = [160, 160, 160 + 14 * 16, 160 + 14 * 16]   # samples exactly on cell centres: weights 0 and 1
    fd, rd = torch.from_numpy(feat).to(dev).half(), torch.from_numpy(rois).to(dev)
    for sampling in (0, 2):
        exp, got = _expected_and_got(dev, rd, fd, sampling)
        _assert_same_halves(got, exp, sampling)
        fin = got[1, 4:]          # image 1 has no degenerate proposal
        sub = fin[:, :3].float().abs()
        assert ((sub > 0) & (sub < 6.1e-5)).any() and (fin[:, 1] == 0).any()                    # subnormal and flushed-by-rounding bins
        assert (fin[:, 3] == 65504).any() and (fin[:, 4] == -65504).any() and not torch.isinf(fin[:, 3:6]).any()
        assert torch.isinf(fin[:, 6]).any() and torch.isinf(fin[:, 7]).any() and torch.isinf(got[:, :, 9]).any()


def test_roi_align_half_full_shape(dev):
    """The reference's configuration (rcnn.cpp:39-43,150): 1000 proposals x 1024 channels x 14 x 14 on the 50 x 67 map."""
    rng = np.random.default_rng(472)
    B, N, c, H, W = 2, 1000, 1024, 50, 67
    feat = torch.from_numpy(rng.standard_normal((B, c, H, W)).astype(np.float32)).to(dev).half()
    x1 = rng.uniform(0, 900, (B, N)); y1 = rng.uniform(0, 700, (B, N))
    w = np.exp(rng.uniform(np.log(16), np.log(600), (B, N))); h = np.exp(rng.uniform(np.log(16), np.log(500), (B, N)))
    rd = torch.from_numpy(np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)).to(dev)
    for sampling in (0, 2):
        exp, got = _expected_and_got(dev, rd, feat, sampling)
        assert not torch.isnan(exp).any()
        assert torch.equal(got.view(torch.int16), exp.view(torch.int16)), sampling
        del exp, got


def _fill(t, byte):
    t.view(torch.uint8).fill_(byte)
    return t


def test_typed_fp32_calls_equal_the_untyped_ones_byte_for_byte(dev):
    lib = L.load()
    rng = np.random.default_rng(473)
    B, N, c, H, W = 2, 40, 24, 50, 67
    rd = torch.from_numpy(_case_rois(rng, B, N)).to(dev)
    fd = torch.from_numpy(rng.standard_normal((B, c, H, W)).astype(np.float32)).to(dev)
    a, b = _fill(torch.empty((B, N, c, PP, PP), device=dev), 0x5a), _fill(torch.empty((B, N, c, PP, PP), device=dev), 0x5a)
    for sampling in (0, 2):
        assert lib.trtx_roi_align(B, rd.data_ptr(), fd.data_ptr(), a.data_ptr(), PP, 1 / 16, sampling, N, c, H, W, None) == 0
        assert lib.trtx_roi_align_typed(L.F32, B, rd.data_ptr(), fd.data_ptr(), b.data_ptr(), PP, 1 / 16, sampling, N, c, H, W, None) == 0
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    D, nc, S = 20, 7, 14
    md = torch.from_numpy(rng.standard_normal((B, D, nc, S, S)).astype(np.float32)).to(dev)
    idd = torch.from_numpy(rng.integers(-1, nc + 1, (B, D)).astype(np.float32)).to(dev)
    a, b = _fill(torch.empty((B, D, S, S), device=dev), 0x5a), _fill(torch.empty((B, D, S, S), device=dev), 0x5a)
    assert lib.trtx_mask_rcnn_inference(B, idd.data_ptr(), md.data_ptr(), a.data_ptr(), D, S, nc, None) == 0
    assert lib.trtx_mask_rcnn_inference_typed(L.F32, B, idd.data_ptr(), md.data_ptr(), b.data_ptr(), D, S, nc, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_mask_rcnn_inference_half_masks(dev, oracle):
    rng = np.random.default_rng(474)
    B, D, nc, S = 2, 100, 80, 14
    masks = (rng.standard_normal((B, D, nc, S, S)).astype(np.float32) * 3).astype(np.float16)
    idx = rng.integers(0, nc, (B, D)).astype(np.float32)
    idx[0, 5] = -1.0
    idx[1, 7] = float(nc)                      # out of range: the row is not written
    md, idd = torch.from_numpy(masks).to(dev), torch.from_numpy(idx).to(dev)
    plug = P.MaskRcnnInferencePlugin(D, S, nc)
    got = torch.full((B, D, S, S), 9.0, device=dev)
    assert plug.enqueue(B, [idd, md], [got]) == 0
    ref = torch.full((B, D, S, S), 9.0, device=dev)
    assert plug.enqueue(B, [idd, md.float()], [ref]) == 0
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))          # the fp32 kernel on the widened masks
    assert torch.all(got[0, 5] == 9.0) and torch.all(got[1, 7] == 9.0) and not torch.any(got[0, 4] == 9.0)
    for b in range(B):
        exp = oracle.mask_rcnn_inference(idx[b], masks[b].astype(np.float32), out=np.full((D, S, S), 9.0, np.float32))
        np.testing.assert_allclose(got[b].cpu().numpy(), exp, rtol=3e-7, atol=1e-7)


@pytest.mark.parametrize("anticov", [False, True], ids=["retinaface", "anticov"])
@pytest.mark.parametrize("B,h,w", [(1, 640, 640), (16, 640, 640), (1, 480, 640), (16, 480, 640)])
def test_decode_trt_half_heads(oracle, dev, anticov, B, h, w):
    gen = synth.anticov_heads if anticov else synth.retina_heads
    heads16 = [x.astype(np.float16) for x in gen(B, seed=480 + B, in_h=h, in_w=w)]
    wide = [x.astype(np.float32) for x in heads16]
    ref, _ = oracle.anticov_decode(wide, in_h=h, in_w=w) if anticov else oracle.retina_decode(wide, in_h=h, in_w=w, gate=0.02)
    F = 16 if anticov else 15
    plug = P.DecodePlugin(h, w, anticov=anticov)
    ws = torch.empty(max(plug.getWorkspaceSize(B), 256), dtype=torch.uint8, device=dev)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in heads16], [out], ws) == 0
    out32 = torch.zeros_like(out)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in wide], [out32], ws) == 0
    got, got32 = out.cpu().numpy(), out32.cpu().numpy()
    assert plug.params.in_dtype == L.F32                       # enqueue works on a copy of the parameters
    assert np.array_equal(got[:, 0], ref[:, 0]) and ref[:, 0].min() > 20
    for b in range(B):
        n = int(ref[b, 0])
        np.testing.assert_allclose(got[b, 1:1 + n * F], ref[b, 1:1 + n * F], atol=ATOL, rtol=RTOL_EXP)
        assert np.array_equal(got[b, :1 + n * F], got32[b, :1 + n * F])      # the same code on the same floats
    # unaligned head pointers (one cell per load) give the same rows
    shifted = []
    for x in heads16:
        buf = torch.empty(x.size + 1, dtype=torch.float16, device=dev)
        buf[1:] = torch.from_numpy(x).to(dev).flatten()
        shifted.append(buf[1:].view(x.shape))
    out1 = torch.zeros_like(out)
    assert plug.enqueue(B, shifted, [out1], ws) == 0
    assert torch.equal(out1, out)


def test_retina_pipeline_half_heads_equal_the_widened_fp32_heads(dev):
    B = 4
    heads16 = [torch.from_numpy(x.astype(np.float16)).to(dev) for x in synth.retina_heads(B, seed=481)]
    pipe = RetinaPipeline(B, device=dev)
    a = pipe.run_device(heads16, overlap=False).clone()
    b = pipe.run_device([x.float() for x in heads16], overlap=False).clone()
    torch.cuda.synchronize()
    assert (a[:, 0] > 5).all() and torch.equal(a[:, 0], b[:, 0])
    for i in range(B):
        n = int(a[i, 0])
        assert torch.equal(a[i, :1 + n * 17], b[i, :1 + n * 17])


def test_rejections_write_nothing(dev):
    """Unknown dtype and misaligned pointers through the C ABI -> TRTX_ERR_INVALID; other or mixed dtypes through the Python
    wrappers -> TrtxError before the library is called.  The poisoned outputs stay as they were."""
    lib = L.load()
    INV = L.ERR_INVALID
    B, N, c, H, W = 1, 8, 8, 20, 27
    rois = torch.tensor([[[16.0, 16.0, 200.0, 180.0]] * N], device=dev)
    feat = torch.randn((B, c, H, W), device=dev)
    feat16 = torch.empty(feat.numel() + 8, dtype=torch.float16, device=dev)
    out16 = _fill(torch.empty(B * N * c * PP * PP + 8, dtype=torch.float16, device=dev), 0x5a)
    out32 = _fill(torch.empty(B * N * c * PP * PP + 8, dtype=torch.float32, device=dev), 0x5a)

    def roi(dtype, r, f, o):
        return lib.trtx_roi_align_typed(dtype, B, r, f, o, PP, 1 / 16, 2, N, c, H, W, None)

    assert roi(2, rois.data_ptr(), feat.data_ptr(), out32.data_ptr()) == INV and roi(-1, rois.data_ptr(), feat.data_ptr(), out32.data_ptr()) == INV
    assert roi(L.F16, rois.data_ptr(), feat16.data_ptr() + 1, out16.data_ptr()) == INV      # half features on an odd address
    assert roi(L.F16, rois.data_ptr(), feat16.data_ptr(), out16.data_ptr() + 1) == INV
    assert roi(L.F32, rois.data_ptr(), feat.data_ptr() + 2, out32.data_ptr()) == INV        # float features on a 2-byte boundary
    assert roi(L.F32, rois.data_ptr(), feat.data_ptr(), out32.data_ptr() + 2) == INV
    assert roi(L.F16, rois.data_ptr() + 4, feat16.data_ptr(), out16.data_ptr()) == INV      # a proposal is one 16-byte load
    assert roi(L.F16, rois.data_ptr(), feat16.data_ptr() + 2, out16.data_ptr() + 2) == 0     # 2-byte alignment is all halves need
    torch.cuda.synchronize()
    out16[1:] = out16[0]                                                                     # re-poison after the accepted call
    D, nc, S = 4, 3, 14
    idx = torch.zeros((B, D), device=dev)
    masks16 = torch.zeros(B * D * nc * S * S + 8, dtype=torch.float16, device=dev)
    mout = _fill(torch.empty(B * D * S * S + 8, dtype=torch.float32, device=dev), 0x5a)

    def mask(dtype, i, m, o):
        return lib.trtx_mask_rcnn_inference_typed(dtype, B, i, m, o, D, S, nc, None)

    assert mask(5, idx.data_ptr(), masks16.data_ptr(), mout.data_ptr()) == INV
    assert mask(L.F16, idx.data_ptr(), masks16.data_ptr() + 1, mout.data_ptr()) == INV
    assert mask(L.F32, idx.data_ptr(), masks16.data_ptr() + 2, mout.data_ptr()) == INV
    assert mask(L.F16, idx.data_ptr(), masks16.data_ptr(), mout.data_ptr() + 2) == INV
    assert mask(L.F16, idx.data_ptr() + 2, masks16.data_ptr(), mout.data_ptr()) == INV
    # Decode_TRT
    plug = P.DecodePlugin(480, 640)
    heads16 = [torch.from_numpy(x.astype(np.float16)).to(dev) for x in synth.retina_heads(B, seed=482, in_h=480, in_w=640)]
    ws = torch.empty(max(plug.getWorkspaceSize(B), 256), dtype=torch.uint8, device=dev)
    rows = _fill(torch.empty((B, plug.output_elems()), dtype=torch.float32, device=dev), 0x5a)
    p = L.RetinaParams.from_buffer_copy(plug.params)

    def decode(ptrs, o=None):
        return lib.trtx_retina_decode_enqueue(C.byref(p), B, L.ptr_array(ptrs), rows.data_ptr() if o is None else o, ws.data_ptr(),
                                              ws.numel(), None)

    good = [t.data_ptr() for t in heads16]
    p.in_dtype = 2
    assert decode(good) == INV
    p.in_dtype = L.F16
    assert decode([good[0], good[1] + 1, good[2]]) == INV
    assert decode(good, rows.data_ptr() + 2) == INV
    p.in_dtype = L.F32
    assert decode([good[0] + 2, good[1], good[2]]) == INV
    # the Python wrappers: the tensors' dtype is the selector; a mix or another dtype never reaches the library
    ra = P.RoiAlignPlugin(PP, 1 / 16, 2, N, c, H, W)
    f16 = feat.half()
    o16, o32 = out16[:B * N * c * PP * PP].view(B, N, c, PP, PP), out32[:B * N * c * PP * PP].view(B, N, c, PP, PP)
    for ins, outs in (([rois, f16], [o32]), ([rois, feat], [o16]), ([rois.half(), f16], [o16]), ([rois, feat.double()], [o32]),
                      ([rois, feat.bfloat16()], [o16])):
        with pytest.raises(L.TrtxError):
            ra.enqueue(B, ins, outs)
    mi = P.MaskRcnnInferencePlugin(D, S, nc)
    m16 = masks16[:B * D * nc * S * S].view(B, D, nc, S, S)
    mo = mout[:B * D * S * S].view(B, D, S, S)
    for ins, outs in (([idx.half(), m16], [mo]), ([idx, m16], [mo.half()]), ([idx, m16.to(torch.int16)], [mo])):
        with pytest.raises(L.TrtxError):
            mi.enqueue(B, ins, outs)
    for ins, outs in (([heads16[0], heads16[1].float(), heads16[2]], [rows]), ([h.bfloat16() for h in heads16], [rows]),
                      (heads16, [rows.half()])):
        with pytest.raises(L.TrtxError):
            plug.enqueue(B, ins, outs, ws)
    torch.cuda.synchronize()
    for t in (out16, out32, mout, rows):
        assert (t.view(torch.uint8) == 0x5a).all()
