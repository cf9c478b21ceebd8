"""Every path and edge of the RefineDet post-process (refinedet.cu) at the shapes its contract accepts, against the
reference's own float64 arithmetic bit for bit.

The expected output is the line-by-line transcription of the reference's libtorch post-process (oracle/refinedet.py) run on
CUDA: the same ATen ops and CUDA's double exp as the kernel, so there is no tolerance.  Where scores tie, torch::sort leaves
the order open and the CPU oracle (oracle/refinedet_oracle.c), which applies the library's rule (the lower prior first),
is the expected output instead; those heads have zero offsets, so its boxes are exact too.  The cases are built by
oracle/refinedet_cases.py, and tests/test_refinedet_paths_cpu.py pins what each one claims before it runs here.

| path or edge | cases |
|---|---|
| every accepted side, P = 255 .. 65280, the `rd_prior` level search at levels 1, 3, 9 and 15 cells wide (S = 64, 192, 576, 960) and each level's first and last priors | `side[64]` .. `side[1024]` |
| the float-sqrt prior table where `sqrt(2.0)` and `sqrtf(2.f)` differ (S = 192, 384, 448, 704 .. 960) | `side[192]`, `side[384]`, `side[448]`, `side[704]` .. `side[960]` |
| uint16 keep lists near their limit: kept priors >= 65024 at S = 1024 | `side[1024]` |
| top_k 1, 2, 63, 64, 65, 128, 129, 1000, 1023, 1024: the mask at 1 .. 16 words (176 KB of shared memory at 1024) | `cut[K]`, also cycled over `side[*]` |
| 0, 1, top_k - 1, top_k, top_k + 1 and top_k + 8000 candidates: no select, and the select's cut | `cut[K]` (one class each) |
| every prior a candidate (conf_thresh < 0), the cut inside a +-0 tie across all P | `negative_conf` |
| C = 2, 21, 25, 81 | `side[*]`, `frames[*]` (C = 2) |
| C = 1024: 1023 class CTAs per frame, the rows kernel's largest prefix and class search | `many_classes[*]` |
| B = 1, 3, 64, 65, 130 of distinct frame sizes; frames 63 / 64 and 127 / 128 straddle rows launches | `frames[*]` |
| max_det 1, cut inside a class and at a class boundary, n = 511, 512, 513, 1024, 1025 rows, the default (C - 1) * top_k | `many_classes[64-*]`, `many_classes[128-default]` |
| `score < TH` failures in every pass of 512 rows | `many_classes[*]` |
| sweep keeps exactly one box (nms_thresh 0, -0.5; identical boxes) or all m (disjoint boxes) | `edges[*]`, `cut[*]` |
| suppression chains across mask words 64 .. 320 | `edges[0.45]`, `edges[1]` |
| NaN corners (a NaN IoU suppresses) and zero-area boxes (0 / 0) | `edges[*]` |
| nms_thresh one float ulp above and below a pair's IoU | `pair[above]`, `pair[below]` |
| rounding box i's corners to float decides the pair | `pair[rounding]` |
| an empty frame (every objectness <= obj_thresh) between two others; scores at score_thresh, +inf, NaN | `frames[3]`, `frames[*]` |
| the atomicAdd compaction order does not reach the output | `test_repeat_is_bit_identical` |

Every call writes into outputs filled with a NaN sentinel with a guard element on either side, and into a workspace of
exactly trtx_refinedet_workspace_size bytes followed by guard bytes: every element up to 1 + max_det * 6 must be written,
and no guard touched.  dets must equal the expected rows bit for bit (signed zeros included; NaN at the same places) and
rows must equal the driver loop over them (`RO.rows`)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import refinedet as RO
from oracle import refinedet_cases as RC
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
SENTINEL = 0x7FBADBAD  # a quiet NaN with a payload the device never writes
GUARD = 0xA5
DEFAULTS = {"obj_thresh": 0.01, "conf_thresh": 0.01, "nms_thresh": 0.45, "score_thresh": 0.2}


@functools.lru_cache(maxsize=None)
def _prior(net):
    return RO.prior_box(net, "cuda")


def _params(case, max_det):
    kw = {**DEFAULTS, **case.kw}
    return L.RefinedetParams(kw["net"], case.h[3].shape[2], kw["obj_thresh"], kw["conf_thresh"], kw["nms_thresh"],
                             kw["top_k"], max_det, kw["score_thresh"])


def _max_det(case, max_det):
    return (case.h[3].shape[2] - 1) * case.kw["top_k"] if max_det is None else max_det


def _call(case, dev, max_det=None, rows=True):
    """The post-process into sentinel-filled outputs and an exact workspace with guards -> host (dets, rows or None)."""
    B = case.h[0].shape[0]
    md = _max_det(case, max_det)
    n = B * (1 + 6 * md)
    big = torch.full((2, n + 2), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)
    out, rws = big[0, 1:1 + n].view(B, -1), big[1, 1:1 + n].view(B, -1)
    ws_bytes = int(L.load().trtx_refinedet_workspace_size(C.byref(_params(case, md)), B))
    assert ws_bytes > 0 and ws_bytes % 256 == 0
    wbuf = torch.full((256 + ws_bytes + 256,), GUARD, dtype=torch.uint8, device=dev)
    heads = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in case.h]
    sizes = case.sizes if rows else None
    P.refinedet_postprocess(*heads, sizes, max_det=md, workspace=wbuf[256:256 + ws_bytes], out=out,
                            rows_out=rws if sizes else None, **case.kw)
    wb = wbuf.cpu().numpy()
    assert (wb[:256] == GUARD).all() and (wb[256 + ws_bytes:] == GUARD).all(), "workspace guard written"
    bits = big.view(torch.int32).cpu().numpy()
    assert (bits[:, 0] == SENTINEL).all() and (bits[:, -1] == SENTINEL).all(), "output guard written"
    assert not (bits[0, 1:1 + n] == SENTINEL).any(), "dets element left unwritten"
    if sizes:
        assert not (bits[1, 1:1 + n] == SENTINEL).any(), "rows element left unwritten"
    got = big.cpu().numpy()
    return got[0, 1:1 + n].reshape(B, -1), (got[1, 1:1 + n].reshape(B, -1) if sizes else None)


def _reference(case, b):
    """The expected rows [N, 6] of frame b: the CUDA transcription, or the oracle's tie rule where scores tie."""
    if case.ties:
        d = RO.postprocess(*[x[b] for x in case.h], **case.kw, max_det=_max_det(case, None))
        return d[1:1 + 6 * int(d[0])].reshape(-1, 6)
    return RO.reference_postprocess(*[x[b] for x in case.h], device="cuda", prior=_prior(case.kw["net"]), **case.kw)


def _same_bits(got, want):
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got.view(np.int32)[~nan], want.view(np.int32)[~nan])


def _check(case, dets, rows, refs, max_det=None):
    md = _max_det(case, max_det)
    th = {**DEFAULTS, **case.kw}["score_thresh"]
    for b in range(len(dets)):
        want = RO.as_dets(refs[b], md)
        assert _same_bits(dets[b], want), (b, int(dets[b, 0]), int(want[0]))
        if rows is not None:
            assert _same_bits(rows[b], RO.rows(want, *case.sizes[b], th)), b


def _kept_per_class(ref):
    labels = ref[:, 5].astype(int)
    return {c: int((labels == c).sum()) for c in np.unique(labels)}


def _run(case, dev, **kw):
    refs = [_reference(case, b) for b in range(case.h[0].shape[0])]
    dets, rows = _call(case, dev, **kw)
    _check(case, dets, rows, refs, kw.get("max_det"))
    return refs


# ------------------------------------------------------------------ sides, top_k and the cut -----------------------------
@pytest.mark.parametrize("net", RC.SIDES)
def test_side(dev, net):
    refs = _run(RC.side(net), dev)
    assert all(len(r) > 0 for r in refs)


@pytest.mark.parametrize("K", RC.TOP_KS)
def test_cut(dev, K):
    case = RC.cut(K)
    refs = _run(case, dev)
    got = _kept_per_class(refs[0])
    assert {c: got.get(c, 0) for c in case.claims} == case.claims


def test_negative_conf_thresh_ties_over_all_priors(dev):
    case = RC.negative_conf()
    refs = _run(case, dev)
    assert _kept_per_class(refs[0]).keys() == {1, 2}


def test_repeat_is_bit_identical(dev):
    """A dense large-P case run twice gives the same bits: the order of the atomicAdd compaction is sorted away."""
    case = RC.cut(1024)
    a = _call(case, dev)
    b = _call(case, dev)
    assert np.array_equal(a[0].view(np.int32), b[0].view(np.int32))
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32))


# ------------------------------------------------------------------ sweep and IoU edges --------------------------------
@pytest.mark.parametrize("nms", [0.45, 0.0, -0.5, 1.0], ids=["0.45", "0", "-0.5", "1"])
def test_edges(dev, nms):
    case = RC.edges(nms)
    refs = _run(case, dev)
    got = _kept_per_class(refs[0])
    if nms <= 0:
        assert got == {1: 1, 2: 1, 3: 1, 4: 1}
    elif nms == 0.45:
        assert {c: got[c] for c in case.claims} == case.claims
    else:
        assert got[2] == 1  # identical boxes: IoU exactly 1, not below 1


@functools.lru_cache(maxsize=None)
def _pairs():
    return RC.pair_search()


@pytest.mark.parametrize("which", ["above", "below", "rounding"])
def test_pair_decision(dev, which):
    (i, j, v), (ri, rj, t) = _pairs()
    if which == "rounding":
        b = RC.boxes(320)
        case, kept = RC.pair(ri, rj, t), 2 if RC.iou(b[ri], b[rj])[0] < t else 1
    else:
        t = float(np.nextafter(np.float32(v), np.float32(1 if which == "above" else 0)))
        case, kept = RC.pair(i, j, t), 2 if which == "above" else 1
    refs = _run(case, dev)
    assert len(refs[0]) == kept


# ------------------------------------------------------------------ frames and rows ------------------------------------
@pytest.mark.parametrize("B", [1, 3, 64, 65, 130])
def test_frames(dev, B):
    case = RC.frames(B)
    refs = _run(case, dev)
    if B >= 3:
        assert len(refs[0]) > 0 and len(refs[1]) == 0 and len(refs[2]) > 0
    if B == 1:  # the frame rows are optional: dets alone
        dets, rows = _call(case, dev, rows=False)
        assert rows is None
        _check(case, dets, None, refs)


@functools.lru_cache(maxsize=None)
def _many(net):
    case = RC.many_classes(net)
    return case, [_reference(case, b) for b in range(2)]


def _cuts(ref):
    """max_det inside a class (one past its first row) and at a class boundary, for a class of frame 0 with >= 2 rows."""
    labels = ref[:, 5]
    starts = np.flatnonzero(np.r_[True, labels[1:] != labels[:-1]])
    ends = np.r_[starts[1:], len(labels)]
    s, e = next((s, e) for s, e in zip(starts, ends) if e - s >= 2 and s > 600)
    return {"inside": int(s) + 1, "boundary": int(e)}


@pytest.mark.parametrize("net,max_det", [(64, 1), (64, 511), (64, 512), (64, 513), (64, 1024), (64, 1025),
                                         (64, "inside"), (64, "boundary"), (64, None), (128, None), (128, 512)])
def test_many_classes(dev, net, max_det):
    case, refs = _many(net)
    assert all(len(r) > 1025 for r in refs)
    md = _cuts(refs[0])[max_det] if isinstance(max_det, str) else max_det
    dets, rows = _call(case, dev, max_det=md)
    _check(case, dets, rows, refs, md)
