"""Decode_TRT (tensorrtx_b200/csrc/retina_decode.cu) on every scan it builds and every shape class, against the float64
reference of tests/test_retina_decode_paths_cpu.py.

Each case of gpu_cases() (both variants, fp32 and fp16 heads, nine input sizes from 32x32 to 4480x4480, batches 1 to 64,
sparse / dense / empty / non-finite heads) decodes through trtx_retina_decode_enqueue into an output and a workspace of
exactly the size the library asks for, the output filled with a sentinel, and checks:
  * the count of every image exactly, the kept priors in the reference's order, every finite value within its column's
    bound, non-finite values where the reference has them, and the copied AntiCov columns bit for bit (assert_matches);
  * that every float past an image's 1 + count * F still holds the sentinel: like the reference, the decode writes the
    count and its rows only;
  * the same heads one element off 16-byte alignment, which forces the one-cell-per-load scans, give the same output bit
    for bit, at every size, 4480x4480 included;
  * fp16 heads give bit for bit the output of the fp32 call on the widened heads (every NaN compared as NaN);
  * the images of the batch in another order give their outputs in that order, bit for bit.
The gate is tested at its boundary through trtx_retina_params.gate, and the scan each call should launch is checked by
name in a profiler trace."""
from __future__ import annotations

import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L

from test_retina_decode_paths_cpu import (ANTICOV, DET, DTYPE_SIZE, DTYPE_T, F32, FACE, GATE, KERNEL, VARIANTS, assert_matches,
                                          canonical_bits, case_id, dispatch, gate_heads, gpu_cases, make_heads, reference,
                                          total_priors)

pytestmark = pytest.mark.gpu
DEV = "cuda"
TORCH = {"f32": torch.float32, "f16": torch.float16}
SENTINEL = F32(-7777.25)


def to_device(heads, dtype, offset=False):
    """the heads as device tensors of `dtype`; offset: each one element past an aligned base, in a buffer of exactly one
    more element"""
    out = []
    for h in heads:
        t = torch.from_numpy(h).to(DEV, TORCH[dtype])
        if offset:
            buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=DEV)
            buf[1:].copy_(t.reshape(-1))
            t = buf[1:].view(t.shape)
            assert t.data_ptr() % 16 == DTYPE_SIZE[dtype]
        out.append(t)
    return out


def prepare(dev_heads, variant, in_h, in_w, dtype, gate=GATE):
    """a sentinel-filled output and a workspace of exactly the sizes the library gives -> (output, a function that makes
    one trtx_retina_decode_enqueue into them and returns its code)"""
    lib = L.load()
    B = dev_heads[0].shape[0]
    p = L.RetinaParams(in_h=in_h, in_w=in_w, gate=gate, variant=variant, in_dtype=L.F16 if dtype == "f16" else L.F32)
    ws_bytes = lib.trtx_retina_workspace_size(C.byref(p), B)
    ws = torch.full((ws_bytes,), 0x5A, dtype=torch.uint8, device=DEV)
    out = torch.full((B, 1 + total_priors(in_h, in_w) * DET[variant]), float(SENTINEL), dtype=torch.float32, device=DEV)
    ptrs = L.ptr_array([t.data_ptr() for t in dev_heads])
    return out, lambda: lib.trtx_retina_decode_enqueue(C.byref(p), B, ptrs, out.data_ptr(), ws.data_ptr(), ws_bytes,
                                                       torch.cuda.current_stream().cuda_stream)


def decode(dev_heads, variant, in_h, in_w, dtype, gate=GATE):
    """one trtx_retina_decode_enqueue (see prepare) -> output [B, 1 + total_priors * F] as numpy fp32"""
    out, run = prepare(dev_heads, variant, in_h, in_w, dtype, gate)
    rc = run()
    assert rc == L.OK, L._ERR.get(rc, rc)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_sentinel_past_rows(out, variant):
    F = DET[variant]
    for b in range(out.shape[0]):
        n = int(out[b, 0])
        tail = out[b, 1 + n * F:]
        assert (tail.view(np.uint32) == SENTINEL.view(np.uint32)).all(), (b, n, int((tail != SENTINEL).sum()))


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


CASES = gpu_cases()


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_decode_paths(case):
    variant, dtype, shape, B, values = case
    in_h, in_w = shape
    seed = zlib.crc32(case_id(case).encode())
    heads = make_heads(variant, in_h, in_w, B, values, seed, half=dtype == "f16")
    ref = reference(heads, variant, in_h, in_w)
    if values == "dense":
        assert (ref.counts == total_priors(in_h, in_w)).all()
    if values == "empty":
        assert (ref.counts == 0).all()

    out = decode(to_device(heads, dtype), variant, in_h, in_w, dtype)
    stats = assert_matches(out, ref, variant, case_id(case))
    assert_sentinel_past_rows(out, variant)
    print(f"MARGIN {case_id(case)} " + " ".join(f"{g}={r:.3g}:{e:.3g}/{t:.3g}" for g, (r, e, t) in stats.items()))

    off = decode(to_device(heads, dtype, offset=True), variant, in_h, in_w, dtype)
    assert same_bits(off, out), "heads one element off alignment decode differently"

    if dtype == "f16":
        wide = decode(to_device(heads, "f32"), variant, in_h, in_w, "f32")
        assert np.array_equal(canonical_bits(wide), canonical_bits(out)), "fp16 heads differ from the fp32 call on them"

    if B > 1:
        perm = np.random.default_rng(seed).permutation(B)
        got = decode(to_device([h[perm] for h in heads], dtype), variant, in_h, in_w, dtype)
        assert same_bits(got, out[perm]), "permuting the images does not permute the outputs"


@pytest.mark.parametrize("dtype", ["f32", "f16"])
@pytest.mark.parametrize("shape", [(64, 64), (32, 32), (488, 648)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_gate_boundary(shape, dtype):
    """RetinaFace: equal logits give p = 0.5 exactly, dropped at gate 0.5 and kept at nextafter(0.5, 0).  AntiCov keeps a
    face probability of exactly 0.5 and drops nextafter(0.5, 0) (its gate is the literal)."""
    half = dtype == "f16"
    g1 = float(np.nextafter(F32(0.5), F32(0)))
    heads = gate_heads(FACE, *shape, 3, seed=17, half=half)
    dev = to_device(heads, dtype)
    at, below = decode(dev, FACE, *shape, dtype, gate=0.5), decode(dev, FACE, *shape, dtype, gate=g1)
    ref_at, ref_below = reference(heads, FACE, *shape, gate=0.5), reference(heads, FACE, *shape, gate=g1)
    assert_matches(at, ref_at, FACE, "gate 0.5")
    assert_matches(below, ref_below, FACE, "gate nextafter(0.5, 0)")
    equal = sum(int((h[:, 8:12:2] == h[:, 9:12:2]).sum()) for h in heads)
    assert equal > 0 and below[:, 0].sum() - at[:, 0].sum() == equal

    heads = gate_heads(ANTICOV, *shape, 3, seed=19, half=half)
    out = decode(to_device(heads, dtype), ANTICOV, *shape, dtype)
    ref = reference(heads, ANTICOV, *shape)
    assert_matches(out, ref, ANTICOV, "anticov 0.5")
    assert out[:, 0].sum() == sum(int((h[:, 2:4] >= F32(0.5)).sum()) for h in heads)


def traced_scans(run, windows=4, repeat=10):
    """the names of the scan kernels recorded in a profiler window of `repeat` calls of run(): the first of up to `windows`
    windows that recorded any, or an empty set.  CUPTI on a shared machine can drop a window's records, all of them or
    some, so a name that is missing proves nothing; a name that is recorded ran."""
    for _ in range(windows):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            rcs = [run() for _ in range(repeat)]
            torch.cuda.synchronize()
        assert set(rcs) == {L.OK}, rcs
        names = {e.name.replace(" ", "") for e in prof.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA and "scan_kernel" in e.name}
        if names:
            return names
    return set()


@pytest.mark.parametrize("variant", [FACE, ANTICOV], ids=VARIANTS.get)
@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_the_mirrored_scan_runs(variant, dtype):
    """aligned 64x64 heads run the four-cells-per-load scan and heads one element off it the one-cell scan, as dispatch()
    says, and no other scan.  Each window holds the enqueues of one of the two alone: their buffers are made before it."""
    heads = make_heads(variant, 64, 64, 2, "sparse", seed=23, half=dtype == "f16")
    es = DTYPE_SIZE[dtype]
    unseen = []
    for offset in (False, True):
        _, run = prepare(to_device(heads, dtype, offset), variant, 64, 64, dtype)
        assert run() == L.OK                            # first launch outside the trace
        torch.cuda.synchronize()
        want = dispatch(variant, dtype, 64, 64, 2, addr_mod=(es,) * 3 if offset else (0, 0, 0))["kernel"]
        assert DTYPE_T[dtype] in want and (want.endswith(", 1>") if offset else want.endswith(", 4>"))
        scans = traced_scans(run)
        assert all(want.replace(" ", "") in n for n in scans), (want, scans)
        if not scans:
            unseen.append(want)
    if unseen:
        pytest.skip(f"torch.profiler recorded no scan in 4 windows for {unseen}: the outputs were checked, the kernel "
                    "choice was not")
