"""The half-precision mode of RoIAlign, MaskRcnnInference and Decode_TRT, as far as it goes without a device: the ABI of
trtx_retina_params, the argument checks that come before the first launch, the dtype selection of the Python wrappers, the
TensorRT adapters' host surface (tests/trt_adapter_half_check.cpp against tests/mock_trt), and the index algebra of
roi_align_window_kernel<14, __half> replayed formula by formula on a flat array of the kernel's 32768 shared halves."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from test_roi_window_emulation_cpu import _axis_tap

ROOT = Path(__file__).resolve().parents[1]
F = np.float32
INV = L.ERR_INVALID


def _fake(n):
    """a non-null address that is never dereferenced: every call below is rejected before the first launch"""
    return 0x10000 * n


def test_retina_params_abi_and_zeroed_struct_is_fp32():
    lib = L.load()
    assert lib.trtx_abi_sizeof(2) == C.sizeof(L.RetinaParams) == 20
    assert [f[0] for f in L.RetinaParams._fields_] == ["in_h", "in_w", "gate", "variant", "in_dtype"]
    p = L.RetinaParams()
    assert (p.variant, p.in_dtype) == (L.RETINA_FACE, L.F32)
    assert P.DecodePlugin().params.in_dtype == L.F32
    # the struct's size does not change what the size queries answer
    p.in_h, p.in_w = 480, 640
    q = L.RetinaParams.from_buffer_copy(p)
    q.in_dtype = L.F16
    assert lib.trtx_retina_workspace_size(C.byref(p), 4) == lib.trtx_retina_workspace_size(C.byref(q), 4) > 0
    assert lib.trtx_retina_total_priors(C.byref(p)) == lib.trtx_retina_total_priors(C.byref(q)) == 12600


def test_argument_checks_before_the_first_launch():
    lib = L.load()

    def roi(dtype=L.F16, rois=_fake(1), feat=_fake(2), out=_fake(3), batch=1, pooler=14, n=10, c=8, h=20, w=27):
        return lib.trtx_roi_align_typed(dtype, batch, rois, feat, out, pooler, 1 / 16, 2, n, c, h, w, None)

    assert roi(dtype=2) == roi(dtype=-1) == roi(dtype=L.F32, feat=_fake(2) + 2) == INV
    assert roi(feat=_fake(2) + 1) == roi(out=_fake(3) + 1) == roi(rois=_fake(1) + 8) == INV
    assert roi(dtype=L.F32, out=_fake(3) + 2) == roi(rois=None) == roi(feat=None) == roi(out=None) == INV
    assert roi(batch=0) == roi(n=0) == roi(c=0) == roi(h=0) == roi(pooler=0) == INV
    assert roi(pooler=33) == L.ERR_UNSUPPORTED                      # sizes are judged as in the fp32 call
    assert lib.trtx_roi_align(1, _fake(1), _fake(2) + 2, _fake(3), 14, 1 / 16, 2, 10, 8, 20, 27, None) == INV

    def mask(dtype=L.F16, idx=_fake(1), masks=_fake(2), out=_fake(3), batch=1, d=4, s=14, nc=3):
        return lib.trtx_mask_rcnn_inference_typed(dtype, batch, idx, masks, out, d, s, nc, None)

    assert mask(dtype=3) == mask(masks=_fake(2) + 1) == mask(dtype=L.F32, masks=_fake(2) + 2) == INV
    assert mask(idx=_fake(1) + 2) == mask(out=_fake(3) + 2) == mask(masks=None) == mask(d=0) == mask(nc=0) == INV

    p = L.RetinaParams(480, 640, 0.02, L.RETINA_FACE, L.F16)

    def decode(ptrs=(_fake(1), _fake(2), _fake(3)), out=_fake(4), ws=_fake(5)):
        return lib.trtx_retina_decode_enqueue(C.byref(p), 1, L.ptr_array(ptrs), out, ws, 1 << 30, None)

    assert decode(ptrs=(_fake(1), _fake(2) + 1, _fake(3))) == decode(out=_fake(4) + 2) == decode(ptrs=(_fake(1), 0, _fake(3))) == INV
    p.in_dtype = 2
    assert decode() == INV
    p.in_dtype = L.F32
    assert decode(ptrs=(_fake(1) + 2, _fake(2), _fake(3))) == INV
    p.in_dtype, p.variant = L.F16, 2
    assert decode() == INV


def test_python_wrappers_take_the_dtype_from_the_tensors():
    f32, f16 = torch.zeros(4), torch.zeros(4, dtype=torch.float16)
    assert P._elem_dtype([f32, f32], "x") == L.F32 and P._elem_dtype([f16, f16, f16], "x") == L.F16
    assert P._elem_dtype([0x1000, f32], "x") == L.F32               # a raw address carries no dtype: fp32, as before
    for bad in ([f32, f16], [f16, 0x1000], [torch.zeros(4, dtype=torch.bfloat16)], [torch.zeros(4, dtype=torch.float64)],
                [torch.zeros(4, dtype=torch.int32)]):
        with pytest.raises(L.TrtxError):
            P._elem_dtype(bad, "x")
    with pytest.raises(L.TrtxError):
        P._elem_dtype([f16], "x", only=L.F32)
    # a mix is refused before any pointer is taken: these are host tensors, which _ptr would refuse with another message
    ra = P.RoiAlignPlugin(14, 1 / 16, 2, 1, 4, 20, 27)
    with pytest.raises(L.TrtxError, match="mixed dtypes"):
        ra.enqueue(1, [f32, f16], [f32])
    with pytest.raises(L.TrtxError, match="must be torch.float32"):
        ra.enqueue(1, [f16, f16], [f16])
    with pytest.raises(L.TrtxError, match="indices and output: must be torch.float32"):
        P.MaskRcnnInferencePlugin(1, 14, 1).enqueue(1, [f16, f16], [f16])
    with pytest.raises(L.TrtxError, match="mixed dtypes"):
        P.DecodePlugin().enqueue(1, [f16, f32, f16], [f32], f32)
    with pytest.raises(L.TrtxError, match="must be torch.float32"):
        P.DecodePlugin().enqueue(1, [f16, f16, f16], [f16], f32)


def _build_half_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda = Path(nvcc).resolve().parents[1]
    exe = tmp_path / "trt_adapter_half_check"
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-I", str(ROOT / "include"), "-I", str(ROOT / "tests" / "mock_trt"),
           "-I", str(cuda / "include"), str(ROOT / "tests" / "trt_adapter_half_check.cpp"), "-o", str(exe),
           str(L.LIB_PATH), f"-Wl,-rpath,{L.LIB_PATH.parent}", "-L", str(cuda / "lib64"), "-lcudart", f"-Wl,-rpath,{cuda / 'lib64'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_half_adapters_host_surface(tmp_path):
    """Format combinations accepted and refused at every position, output data types, configurePlugin -> serialize ->
    deserialize -> clone keeps the element type, a blob of the reference's length is an fp32 plugin."""
    r = subprocess.run([str(_build_half_check(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "trt adapter half check ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_half_adapters_enqueue_on_gpu(tmp_path, dev):
    """enqueue through each adapter equals the direct C call, halves and floats."""
    r = subprocess.run([str(_build_half_check(tmp_path)), "--gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "gpu half enqueue ok" in r.stdout, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# roi_align_window_kernel<14, __half>: kRoiWindowBytes / 2 halves, RoiWin<__half>::kCU / kGroup / kPad / kMin
WINDOW_HALVES, CU, GROUP, PAD, MIN, CPC, MAX_TABLE = 32768, 16, 16, 8, 8, 64, 256


def emulate_half(rois, feat, P_, scale, sampling):
    """feat: float16 [C, H, W] -> float16 [N, C, P, P]; the fill goes through 32-bit words of two halves as the kernel's does."""
    C_, H, W = feat.shape
    bits = feat.view(np.uint16)
    N = rois.shape[0]
    out = np.full((N, C_, P_, P_), np.nan, np.float16)
    scale = F(scale)
    used = {"passes": 0, "narrow": 0, "partial": 0, "full": 0, "pow2": 0, "div": 0}
    for n in range(N):
        r = rois[n].astype(F)
        start_w, start_h = F(r[0] * scale - F(0.5)), F(r[1] * scale - F(0.5))
        end_w, end_h = F(r[2] * scale - F(0.5)), F(r[3] * scale - F(0.5))
        roi_w, roi_h = F(end_w - start_w), F(end_h - start_h)
        bin_h, bin_w = F(roi_h / F(P_)), F(roi_w / F(P_))
        gh = sampling if sampling > 0 else int(np.ceil(F(roi_h / F(P_))))
        gw = sampling if sampling > 0 else int(np.ceil(F(roi_w / F(P_))))
        count = F(gh * gw)
        assert gh > 0 and gw > 0 and P_ * gh <= MAX_TABLE and P_ * gw <= MAX_TABLE, "the test only feeds tabulated proposals"
        s_y = [_axis_tap(F(F(start_h + F(ph * bin_h)) + F(F(F(iy + 0.5) * bin_h) / F(gh))), H) for ph in range(P_) for iy in range(gh)]
        s_x = [_axis_tap(F(F(start_w + F(pw * bin_w)) + F(F(F(ix + 0.5) * bin_w) / F(gw))), W) for pw in range(P_) for ix in range(gw)]
        vy, vx = [t for t in s_y if t[4]], [t for t in s_x if t[4]]
        if not vy or not vx:                    # every sample outside the map
            out[n] = np.float16(F(0) / count)
            continue
        y0, y1 = min(t[0] for t in vy), max(t[1] for t in vy)
        x0, x1 = min(t[0] for t in vx), max(t[1] for t in vx)
        wh, ww = y1 - y0 + 1, x1 - x0 + 1
        cells = wh * ww
        cpass = min(CPC, (WINDOW_HALVES // cells - PAD) & ~(GROUP - 1))
        pitch = cpass + PAD
        if cpass < GROUP:
            cpass, pitch = MIN, MIN
            used["narrow"] += 1
        assert cells * pitch <= WINDOW_HALVES and (pitch * 2) % 16 == 0 and (pitch * 2 // 16) % 2 == 1
        w_y = [(((t[0] - y0) * ww * pitch * 2) if t[4] else -1, (t[1] - y0) * ww * pitch * 2, t[2], t[3]) for t in s_y]
        w_x = [(((t[0] - x0) * pitch * 2) if t[4] else -1, (t[1] - x0) * pitch * 2, t[2], t[3]) for t in s_x]
        ngroups, m_ww = (cells + 7) >> 3, (65536 + ww - 1) // ww
        pow2 = (gh * gw) & (gh * gw - 1) == 0
        used["pow2" if pow2 else "div"] += 1
        for c_begin in range(0, C_, CPC):
            c_end = min(C_, c_begin + CPC)
            for cb in range(c_begin, c_end, cpass):
                nc = min(cpass, c_end - cb)
                used["passes"] += 1
                assert nc % 8 == 0, "the dispatcher only sends channel counts that are a multiple of 8 to this kernel"
                words = np.full(WINDOW_HALVES // 2, 0x7e007e00, np.uint32)      # stale shared memory: NaNs
                e = np.arange(ngroups * 32, dtype=np.int64)                     # every thread's fill items
                fx, fc = e & 7, (e >> 3) & 3                                    # 8 cells x 4 channel PAIRS
                cell = (e >> 5) * 8 + fx
                ok = cell < cells
                fx, fc, cell = fx[ok], fc[ok], cell[ok]
                y = (cell * m_ww) >> 16 if cells * ww <= 65536 else cell // ww
                x = cell - y * ww
                assert np.array_equal(y, cell // ww)
                for cq in range(nc >> 3):
                    lo = bits[cb + 2 * fc + 8 * cq, y0 + y, x0 + x].astype(np.uint32)
                    hi = bits[cb + 2 * fc + 8 * cq + 1, y0 + y, x0 + x].astype(np.uint32)
                    byte = (2 * fc) * 2 + cell * pitch * 2 + 16 * cq
                    assert np.all(byte % 4 == 0) and len(np.unique(byte)) == len(byte)
                    words[byte // 4] = lo | (hi << 16)
                smem = words.view(np.float16).astype(F)                          # a tap is widened exactly
                for k0 in range(0, nc, CU):
                    nch = nc - k0
                    used["full" if nch >= CU else "partial"] += 1
                    for ph in range(P_):
                        for pw in range(P_):
                            acc = np.zeros(CU, F)
                            for iy in range(gh):
                                ty = w_y[ph * gh + iy]
                                if ty[0] < 0:
                                    continue
                                for ix in range(gw):
                                    tx = w_x[pw * gw + ix]
                                    if tx[0] < 0:
                                        continue
                                    ly, hy, lx, hx = ty[2], ty[3], tx[2], tx[3]
                                    w1, w2, w3, w4 = F(hy * hx), F(hy * lx), F(ly * hx), F(ly * lx)
                                    for g in (g for g in range(CU // 8) if nch >= CU or 8 * g < nch):
                                        # one LDS.128 per tap: byte offset / 2 + k0 + 8g .. + 7
                                        i1, i2 = (ty[0] + tx[0]) // 2 + k0 + 8 * g, (ty[0] + tx[1]) // 2 + k0 + 8 * g
                                        i3, i4 = (ty[1] + tx[0]) // 2 + k0 + 8 * g, (ty[1] + tx[1]) // 2 + k0 + 8 * g
                                        assert max(i1, i2, i3, i4) + 7 < WINDOW_HALVES and (ty[0] + tx[0]) % 16 == 0
                                        v1, v2, v3, v4 = smem[i1:i1 + 8], smem[i2:i2 + 8], smem[i3:i3 + 8], smem[i4:i4 + 8]
                                        val = (w1 * v1 + w2 * v2) + w3 * v3
                                        val = val + w4 * v4
                                        acc[8 * g:8 * g + 8] += val
                            res = acc * F(F(1.0) / count) if (pow2 and nch >= CU) else acc / count
                            m = min(nch, CU)
                            out[n, cb + k0:cb + k0 + m, ph, pw] = res[:m].astype(np.float16)      # the one rounding
    return out, used


@pytest.mark.parametrize("shape,sampling", [((8, 50, 67), 0), ((24, 20, 23), 0), ((72, 12, 9), 2), ((16, 33, 3), 3)])
def test_half_window_kernel_algebra_reproduces_the_rounded_oracle(oracle, shape, sampling):
    C_, H, W = shape
    rng = np.random.default_rng(C_ * 1000 + H + sampling)
    feat = rng.standard_normal((C_, H, W)).astype(np.float16)
    sw, sh = W * 16.0, H * 16.0
    k = 6 if C_ > 24 else 12
    x1, y1 = rng.uniform(-40, sw, k), rng.uniform(-40, sh, k)
    w_, h_ = np.exp(rng.uniform(np.log(4), np.log(sw * 1.2), k)), np.exp(rng.uniform(np.log(4), np.log(sh * 1.2), k))
    rois = np.stack([x1, y1, x1 + w_, y1 + h_], -1).astype(F)
    extra = np.array([[0, 0, sw, sh],                    # the whole map: 3350 cells -> passes of 8 channels, row pitch 8
                      [5, 5, 9, 9],                      # a fraction of one cell
                      [sw - 8, sh - 8, sw + 90, sh + 70],  # hangs over the bottom-right corner
                      [-300, -300, -200, -100]], F)      # entirely outside
    rois = np.concatenate([rois, extra])
    if sampling == 0:                                    # keep the adaptive grids inside the 256-entry tables
        rois = rois[np.ceil((rois[:, 2] - rois[:, 0]) / 16 / 14) * 14 <= MAX_TABLE]
    got, used = emulate_half(rois, feat, 14, 1 / 16, sampling)
    ref = oracle.roi_align(rois, feat.astype(F), 14, 1 / 16, sampling).astype(np.float16)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.array_equal(got.view(np.uint16)[~np.isnan(got)], ref.view(np.uint16)[~np.isnan(ref)])
    assert used["passes"] >= len(rois) // 2
    if shape == (8, 50, 67):
        assert used["narrow"] > 0 and used["partial"] > 0 and used["pow2"] > 0
    if shape == (72, 12, 9):                             # 64 + 8 channels: full rounds of 16 and the partial round of 8
        assert used["full"] > 0 and used["partial"] > 0
