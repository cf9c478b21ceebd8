"""RoIAlign on every kernel path of trtx_roi_align_typed (tensorrtx_b200/csrc/roi_align.cu) and every shape class.

Each case runs its proposals through the library in fp32 and checks:
  * against the float64 reference of tests/test_roi_align_paths_cpu.py, every bin that is pinned (see there) within its
    tolerance, and NaN bins (0 / 0) where the reference has them;
  * that the kernel it names ran (torch.profiler), and that nothing outside the output was written -- features and bins
    live one element past an aligned base inside larger buffers, the features' slack is NaN (a tap outside the map shows
    up as a NaN bin) and the output's slack is poisoned;
  * window kernel cases: the same proposals again with one more channel appended to the features -- an odd channel count,
    so the direct kernel -- give the same first C channels bit for bit, NaNs included.  A bin of channel c depends on
    channel c only, so this pins the window kernel to the direct one on every proposal, unpinned bins included;
  * fp16: half features give half(fp32 result on the widened halves) bit for bit, the definition of the half mode, and the
    window and direct kernels agree in fp16 as well;
  * where oracle/_ref/libref_rcnn.so was built, the reference's own roiAlign gives the same fp32 bits.
Adaptive sampling (sampling_ratio 0) gets finite proposals of at most 60 * P cells a side only: grid = ceil(side / P), so a
huge or non-finite proposal makes the work per bin unbounded, in the reference as here."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L

from test_roi_align_paths_cpu import (F32, assert_close_to_reference, cpass_boundaries, hull_proposal, kernel_for, proposals,
                                      regimes, window_hull)

pytestmark = pytest.mark.gpu
DEV = "cuda"
ES = {L.F32: 4, L.F16: 2}
TORCH = {L.F32: torch.float32, L.F16: torch.float16}
POISON = 0x5A


@dataclass
class Case:
    P: int
    C: int
    H: int
    W: int
    scale: float
    sampling: int
    B: int = 1
    n_each: int = 2
    offset: bool = False
    hulls: list = field(default_factory=list)   # (rows, cols) of extra proposals sized to a window of exactly that many cells
    naninf: bool = False
    tag: str = ""

    def build(self, seed):
        """(rois [B, N, 4], features [B, C, H, W]) fp32"""
        rng = np.random.default_rng(seed)
        rois = []
        for _ in range(self.B):
            r = proposals(rng, self.H, self.W, self.P, self.scale, self.n_each, max_cells=60 * self.P if self.sampling == 0 else None)
            extra = [hull_proposal(wh, ww, self.H, self.W, self.P, self.scale, self.sampling) for wh, ww in self.hulls]
            rois.append(np.concatenate([r, np.array(extra, F32).reshape(-1, 4)]))
        feat = rng.standard_normal((self.B, self.C, self.H, self.W)).astype(F32)
        if self.naninf:
            feat[:, 1, 0, 0] = np.inf
            feat[:, 2, -1, -1] = -np.inf
            feat[:, 3, self.H // 2, self.W // 2] = np.nan
            feat[:, 5, 0, :] = np.inf            # a whole row: the first row of channel 5 follows the last of channel 4
        return np.stack(rois), feat

    @property
    def id(self):
        k = kernel_for(self.P, self.C, self.H, self.W, 4)
        s = {0.25: "1_4", 0.125: "1_8", 0.0625: "1_16", 0.03125: "1_32", 1.0: "1"}.get(self.scale, f"{self.scale:g}")
        parts = [k, f"P{self.P}", f"c{self.C}", f"{self.H}x{self.W}", f"s{s}", f"sr{self.sampling}", f"b{self.B}"]
        return "-".join(parts + ([self.tag] if self.tag else []) + (["off1"] if self.offset else []))


# fp32 boundaries of the channels-per-pass regimes (240 / 1365 cells) and the fp16 ones (455 / 1365), each from both sides
B32, B16 = cpass_boundaries(4), cpass_boundaries(2)
WIDE_HULLS = [(1, c) for b in (B32, B16) for c in (b[0], b[0] + 1, b[1], b[1] + 1)]
CASES = [
    # window kernel (pooler 14, channels % 4 == 0, at most 4096 cells); fp16 takes it for channels % 8 == 0
    Case(14, 4, 1, 1, 1 / 8, 0, B=3, offset=True),
    Case(14, 8, 1, 67, 1 / 4, 2),
    Case(14, 20, 50, 1, 1 / 32, 3, offset=True, tag="cta20"),
    Case(14, 64, 7, 9, 1.0, 0, B=3),
    Case(14, 68, 50, 67, 0.3, 0, offset=True, tag="tail4"),
    Case(14, 84, 64, 64, 1 / 16, 4, hulls=[(15, 16), (35, 39), (35, 13), (19, 24)], tag="cta20-hulls"),
    Case(14, 1024, 50, 67, 1 / 16, 0, n_each=1, tag="cta16"),
    Case(14, 64, 1, 4096, 1 / 8, 2, n_each=1, hulls=WIDE_HULLS, tag="cpass-bounds-divfill"),
    Case(14, 20, 4096, 1, 1 / 4, 1, offset=True, tag="mulfill"),
    Case(14, 8, 64, 64, 1 / 16, 19, tag="untabled"),
    Case(14, 8, 7, 9, 1 / 8, 1, B=70, n_each=1),
    Case(14, 8, 50, 67, 1 / 16, 0, naninf=True, tag="naninf"),
    # direct kernel: other poolers, channel counts, maps of more than 4096 cells
    Case(1, 1, 50, 67, 1 / 16, 0, B=3, offset=True),
    Case(2, 3, 7, 9, 1 / 4, 2),
    Case(7, 5, 65, 64, 1 / 8, 0, offset=True),
    Case(7, 63, 50, 67, 1 / 32, 37, tag="untabled"),
    Case(16, 5, 200, 272, 0.3, 0),
    Case(16, 65, 64, 64, 1.0, 17, offset=True, tag="untabled"),
    Case(14, 78, 200, 272, 1 / 16, 2),
    Case(14, 64, 65, 64, 1 / 4, 3),
    Case(7, 3, 1, 4096, 1 / 8, 4, n_each=1, offset=True),
    Case(2, 1, 4096, 1, 1 / 32, 1, n_each=1),
    Case(7, 3, 7, 9, 0.3, 0, B=70, n_each=1),
    Case(14, 65, 1, 1, 1.0, 0, offset=True),
    Case(16, 1, 1, 67, 1 / 4, 3),
    Case(1, 78, 50, 1, 1.0, 4, offset=True),
]
UNSUPPORTED = Case(17, 8, 7, 9, 1 / 8, 2)      # 17 x 17 = 289 bins: more than the 256 threads of a CTA
DATA = {c.id: c.build(seed) for seed, c in enumerate(CASES + [UNSUPPORTED])}
assert len(DATA) == len(CASES) + 1


def _coverage():
    hit, cells = set(), {4: set(), 2: set()}
    for c in CASES + [UNSUPPORTED]:
        rois, _ = DATA[c.id]
        for es in (4, 2):
            for b in range(c.B):
                hit |= regimes(rois[b], c.P, c.C, c.H, c.W, c.scale, c.sampling, es)
                if kernel_for(c.P, c.C, c.H, c.W, es) == "window":
                    for h in window_hull(rois[b], c.P, c.scale, c.sampling, c.H, c.W):
                        if h:
                            cells[es].add((h[1] - h[0] + 1) * (h[3] - h[2] + 1))
    return hit, cells


REQUIRED = {f"{dt}:{r}" for dt in ("f32", "f16") for r in (
    "direct:tabled", "direct:untabled", "window:untabled", "window:outside", "window:cpass64", "window:cpass_mid", "window:kmin",
    "window:round_full@cpass64", "window:round_partial@cpass64", "window:round_full@cpass_mid", "window:round_partial@kmin",
    "window:pow2", "window:div", "window:fill_mul", "window:fill_div", "unsupported")} | {"f32:window:round_partial@cpass_mid"}
HIT, HULL_CELLS = _coverage()
assert REQUIRED <= HIT, f"dispatch regimes the case matrix misses: {sorted(REQUIRED - HIT)}"
for _es, _b in ((4, B32), (2, B16)):
    assert {_b[0], _b[0] + 1, _b[1], _b[1] + 1} <= HULL_CELLS[_es], (_es, _b)


def _launch(dtype, B, rois, feat, out, P, scale, sampling, N, Cc, H, W):
    return L.load().trtx_roi_align_typed(dtype, B, rois.data_ptr(), feat.data_ptr(), out.data_ptr(), P, scale, sampling, N, Cc, H,
                                         W, None)


def _kernels_run(fn):
    """(fn(), names of the device kernels it ran), the names None where the profiler reports no kernel"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc = fn()
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages() if "roi_align" in e.key}
    return rc, names or None


def _features(feat, dtype, offset, slack):
    """features as a view `offset` elements into a NaN-filled buffer with `slack` elements after them"""
    buf = torch.full((offset + feat.size + slack,), float("nan"), dtype=TORCH[dtype], device=DEV)
    view = buf[offset:offset + feat.size].view(feat.shape)
    view.copy_(torch.from_numpy(feat).to(DEV).to(TORCH[dtype]))
    return buf, view


def _output(shape, dtype, offset, slack):
    buf = torch.empty((offset + int(np.prod(shape)) + slack,), dtype=TORCH[dtype], device=DEV)
    buf.view(torch.uint8).fill_(POISON)
    return buf, buf[offset:offset + int(np.prod(shape))].view(shape)


def _run(case, dtype, rois_d, feat, expect=None):
    """one call on `feat` (host, [B, C', H, W] fp32, rounded to dtype on the device) -> bins [B, N, C', P, P] (device)"""
    B, N = rois_d.shape[:2]
    Cc = feat.shape[1]
    off = 1 if case.offset else 0
    fbuf, fview = _features(feat, dtype, off, 64 * case.H * case.W + 4096)
    shape = (B, N, Cc, case.P, case.P)
    obuf, oview = _output(shape, dtype, off, 64 * case.P * case.P)
    rc, names = _kernels_run(lambda: _launch(dtype, B, rois_d, fview, oview, case.P, case.scale, case.sampling, N, Cc, case.H, case.W))
    assert rc == 0, rc
    want = kernel_for(case.P, Cc, case.H, case.W, ES[dtype])
    if names is not None:
        ran = {"window" if "roi_align_window_kernel" in n else "direct" for n in names}
        assert ran == {want}, (names, want)
    assert expect is None or want == expect, (want, expect)
    raw = obuf.view(torch.uint8)
    es = ES[dtype]
    assert (raw[:off * es] == POISON).all() and (raw[(off + oview.numel()) * es:] == POISON).all(), "a bin written outside the output"
    return oview


def _same_bits(a, b, msg):
    """equal bit for bit, NaNs at the same places (of any payload)"""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), (msg, "NaN bins differ", int((na != nb).sum()))
    ia = a.view(torch.int32 if a.dtype == torch.float32 else torch.int16)[~na]
    ib = b.view(torch.int32 if b.dtype == torch.float32 else torch.int16)[~nb]
    assert torch.equal(ia, ib), (msg, int((ia != ib).sum()), "of", ia.numel())


def _widened(feat, extra):
    """feat with one more channel (other values) appended"""
    return np.concatenate([feat, extra[:, :1]], 1)


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_roi_align_path(case):
    rois, feat = DATA[case.id]
    rois_d = torch.from_numpy(rois).to(DEV)
    B, N = rois.shape[:2]
    extra = np.random.default_rng(7).standard_normal((B, 1, case.H, case.W)).astype(F32)
    # fp32 against the float64 reference
    got = _run(case, L.F32, rois_d, feat)
    g = got.cpu().numpy()
    finite = [c for c in range(case.C) if np.isfinite(feat[:, c]).all()]
    compared = 0
    for b in range(B):
        compared += assert_close_to_reference(g[b][:, finite], rois[b], feat[b][finite], case.P, case.scale, case.sampling,
                                              msg=f"{case.id} image {b}")
    assert compared > 0.3 * g.size * len(finite) / case.C
    # window kernel == direct kernel, bit for bit
    for dtype in (L.F32, L.F16):
        if kernel_for(case.P, case.C, case.H, case.W, ES[dtype]) != "window":
            continue
        main = got if dtype == L.F32 else _run(case, L.F16, rois_d, feat)
        plus = _run(case, dtype, rois_d, _widened(feat, extra), expect="direct")
        _same_bits(plus[:, :, :case.C].contiguous(), main, (case.id, dtype, "window vs direct"))
    # fp16 == half(fp32 on the widened halves)
    halves = feat.astype(np.float16).astype(F32)
    exp = _run(case, L.F32, rois_d, halves).half()
    _same_bits(_run(case, L.F16, rois_d, feat), exp, (case.id, "half mode"))
    # the reference's own kernel
    ref_lib = RefOutputs.lib("libref_rcnn.so")
    if ref_lib is None:
        pytest.skip("oracle/_ref/libref_rcnn.so was not built: no comparison with the reference's roiAlign")
    fd = torch.from_numpy(feat).to(DEV)
    ref = torch.zeros_like(got)
    assert ref_lib.ref_roi_align(B, C.c_void_p(rois_d.data_ptr()), C.c_void_p(fd.data_ptr()), C.c_void_p(ref.data_ptr()), case.P,
                             C.c_float(case.scale), case.sampling, N, case.C, case.H, case.W) == 0
    _same_bits(got, ref, (case.id, "reference kernel"))


@pytest.mark.parametrize("dtype", [L.F32, L.F16], ids=["f32", "f16"])
def test_pooler_17_is_unsupported_and_writes_nothing(dtype):
    """TRTX_ERR_UNSUPPORTED before any launch"""
    assert kernel_for(17, 8, 7, 9, ES[dtype]) == "unsupported"
    rois, feat = DATA[UNSUPPORTED.id]
    _, fview = _features(feat, dtype, 0, 0)
    obuf, oview = _output((1, rois.shape[1], 8, 17, 17), dtype, 0, 0)
    rc, names = _kernels_run(lambda: _launch(dtype, 1, torch.from_numpy(rois).to(DEV), fview, oview, 17, 1 / 8, 2, rois.shape[1], 8, 7,
                                             9))
    assert rc == L.ERR_UNSUPPORTED and not names
    assert (obuf.view(torch.uint8) == POISON).all()
