"""Half-precision scores and deltas through RpnDecode and PredictorDecode (include/trtx_hot.h: trtx_rpn_decode_typed,
trtx_predictor_decode_typed), the mode an FP16 Mask R-CNN engine uses so that no reformat copy sits in front of either plugin.
The half result is DEFINED as the fp32 call on the device-widened tensors (torch's .float() on CUDA is __half2float), so
every half call here is compared byte for byte with that fp32 call, and the widened fp32 run is checked against the CPU
oracle (itself pinned to the reference's kernels by tests/test_vs_reference_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth
from tensorrtx_b200.pipeline import RcnnHeadChain

pytestmark = pytest.mark.gpu
ATOL = 1e-4
RTOL_EXP = 2e-6  # columns that pass through expf (CUDA expf vs glibc expf), as tests/test_others_gpu.py
W4 = (10.0, 10.0, 5.0, 5.0)
IMG_H, IMG_W = 800, 1067

# half bit patterns at the edges: +-0, +-inf, NaNs with several payloads and both signs, subnormals, +-65504
EDGE_SCORES = np.array([0x0000, 0x8000, 0x7c00, 0xfc00, 0x7e00, 0xfe00, 0x7c01, 0xfc01, 0x7fff, 0xffff, 0x0001, 0x8001, 0x03ff,
                        0x83ff, 0x0400, 0x7bff, 0xfbff], np.uint16)
# deltas: the same, plus values whose expf overflows (100, 65504) or underflows (-100)
EDGE_DELTAS = np.concatenate([EDGE_SCORES, np.array([100.0, -100.0, 89.0, 20.0], np.float16).view(np.uint16)])


def _ws(dev):
    return torch.empty(4096, dtype=torch.uint8, device=dev)


def _poisoned(shape, dev):
    t = torch.empty(shape, dtype=torch.float32, device=dev)
    t.view(torch.uint8).fill_(0x5a)
    return t


def _bits(t):
    return t.contiguous().view(torch.int32)


def _sprinkle(x16: np.ndarray, edges: np.ndarray, rng, frac: float) -> np.ndarray:
    """x16 (float16) with a fraction `frac` of its elements replaced by edge bit patterns"""
    flat = x16.reshape(-1).view(np.uint16).copy()
    pos = rng.choice(flat.size, int(flat.size * frac), replace=False)
    flat[pos] = edges[rng.integers(0, len(edges), len(pos))]
    return flat.view(np.float16).reshape(x16.shape)


def _rpn(dev, scores, deltas, top_n, anchors, H, W, image=(IMG_H, IMG_W)):
    B = scores.shape[0]
    plug = P.RpnDecodePlugin(top_n, anchors, 16.0, image[0], image[1], H, W)
    os_, ob = _poisoned((B, top_n), dev), _poisoned((B, top_n, 4), dev)
    assert plug.enqueue(B, [scores, deltas], [os_, ob], _ws(dev)) == 0
    torch.cuda.synchronize()
    return os_, ob


def _pred(dev, scores, deltas, props):
    B, N, Cc = scores.shape
    plug = P.PredictorDecodePlugin(N, IMG_H, IMG_W, W4, Cc)
    outs = [_poisoned((B, N), dev), _poisoned((B, N, 4), dev), _poisoned((B, N), dev)]
    assert plug.enqueue(B, [scores, deltas, props], outs, _ws(dev)) == 0
    torch.cuda.synchronize()
    return outs


def _assert_same(got, exp, msg=""):
    for g, e in zip(got, exp):
        assert torch.equal(_bits(g), _bits(e)), (msg, int((_bits(g) != _bits(e)).sum()))


# ------------------------------------------------------------------ RpnDecode -------------------------------------------
RPN_CASES = {"b8.top6000": (8, 15, 50, 67, 6000),     # the reference's shape (rcnn.cpp: pre_nms_topk 6000)
             "b2.top8192": (2, 15, 50, 67, 8192),     # the largest top_n, sort_cap 8192
             "b2.unsorted": (2, 15, 8, 9, 2000)}      # 1080 scores < top_n: no select, -FLT_MAX fill


@pytest.mark.parametrize("case", list(RPN_CASES))
def test_rpn_decode_half_equals_the_widened_fp32_call(dev, oracle, case):
    B, A, H, W, top_n = RPN_CASES[case]
    anchors = synth.rcnn_anchors()
    image = (IMG_H, IMG_W) if H == 50 else (128, 144)
    rng = np.random.default_rng(500 + top_n)
    s32, d32 = synth.rpn_inputs(B, seed=top_n, A=A, H=H, W=W)
    s16, d16 = s32.astype(np.float16), d32.astype(np.float16)
    # clean inputs: half == widened fp32, and the widened fp32 run == the oracle on the same floats
    sd, dd = torch.from_numpy(s16).to(dev), torch.from_numpy(d16).to(dev)
    got = _rpn(dev, sd, dd, top_n, anchors, H, W, image)
    exp = _rpn(dev, sd.float(), dd.float(), top_n, anchors, H, W, image)
    _assert_same(got, exp, case)
    ref_s, ref_b = oracle.rpn_decode(s16.astype(np.float32), d16.astype(np.float32), image[0], image[1], 16.0, anchors, top_n)
    n = min(top_n, A * H * W)
    assert np.array_equal(exp[0].cpu().numpy(), ref_s)
    np.testing.assert_allclose(exp[1].cpu().numpy()[:, :n], ref_b[:, :n], atol=ATOL, rtol=RTOL_EXP)
    if A * H * W > top_n:  # half-quantized logits tie: many equal neighbours in the sorted output
        top = exp[0][:, :n]
        assert (top[:, 1:] == top[:, :-1]).sum() > n // 4
    # edge values in scores and deltas
    s16e = _sprinkle(s16, EDGE_SCORES, rng, 0.05)
    d16e = _sprinkle(d16, EDGE_DELTAS, rng, 0.05)
    sd, dd = torch.from_numpy(s16e).to(dev), torch.from_numpy(d16e).to(dev)
    got = _rpn(dev, sd, dd, top_n, anchors, H, W, image)
    exp = _rpn(dev, sd.float(), dd.float(), top_n, anchors, H, W, image)
    _assert_same(got, exp, case + " edges")
    os_ = exp[0]
    assert torch.isnan(os_).any() and torch.isinf(os_).any() and (os_ == -torch.finfo(torch.float32).max).any()


# ------------------------------------------------------------------ PredictorDecode -------------------------------------
def _half_softmax(rng, B, N, Cc):
    """class probabilities as a half head delivers them: a softmax over 80 classes + background, rounded to half.  Most
    proposals are background, so most class probabilities are 0 or half subnormals, a few hundred distinct values in all,
    and the cut of the top N lands inside a run of equal scores"""
    logits = rng.standard_normal((B, N, Cc + 1)).astype(np.float32) * 3.0
    logits[..., Cc] = np.where(rng.random((B, N)) < 0.005, 0.0, 22.0)
    p = np.exp(logits - logits.max(-1, keepdims=True))
    p = p / p.sum(-1, keepdims=True)
    return np.ascontiguousarray(p[..., :Cc]).astype(np.float16)


@pytest.mark.parametrize("N", [1000, 8192])
def test_predictor_decode_half_equals_the_widened_fp32_call(dev, oracle, N):
    B, Cc = 2, 80
    rng = np.random.default_rng(510 + N)
    s32, d32, props = synth.predictor_inputs(B, seed=N, N=N, Ccls=Cc)
    s16, d16 = s32.astype(np.float16), d32.astype(np.float16)
    pd = torch.from_numpy(props).to(dev)
    sd, dd = torch.from_numpy(s16).to(dev), torch.from_numpy(d16).to(dev)
    got = _pred(dev, sd, dd, pd)
    exp = _pred(dev, sd.float(), dd.float(), pd)
    _assert_same(got, exp, N)
    rs, rb, rc_ = oracle.predictor_decode(s16.astype(np.float32), d16.astype(np.float32), props, IMG_H, IMG_W, W4)
    assert np.array_equal(exp[0].cpu().numpy(), rs) and np.array_equal(exp[2].cpu().numpy(), rc_)
    np.testing.assert_allclose(exp[1].cpu().numpy(), rb, atol=ATOL, rtol=RTOL_EXP)
    # half softmax scores: ties straddle the cut
    sm = torch.from_numpy(_half_softmax(rng, B, N, Cc)).to(dev)
    got = _pred(dev, sm, dd, pd)
    exp = _pred(dev, sm.float(), dd.float(), pd)
    _assert_same(got, exp, f"{N} softmax")
    for b in range(B):
        cut = exp[0][b].min()
        flat = sm[b].flatten().float()
        assert 0 < cut < 6.1e-5 and 1 < (exp[0][b] == cut).sum() < (flat == cut).sum()   # some of the tied scores are cut
        assert (flat == 0).float().mean() > 0.9 and len(torch.unique(flat)) < 4000
    # edge values (1 %: the NaNs, which rank above +inf, leave room for the infs in the top N)
    sde = torch.from_numpy(_sprinkle(s16, EDGE_SCORES, rng, 0.01)).to(dev)
    dde = torch.from_numpy(_sprinkle(d16, EDGE_DELTAS, rng, 0.05)).to(dev)
    got = _pred(dev, sde, dde, pd)
    exp = _pred(dev, sde.float(), dde.float(), pd)
    _assert_same(got, exp, f"{N} edges")
    assert torch.isnan(exp[0]).any() and torch.isinf(exp[0]).any()


# ------------------------------------------------------------------ all 65536 half patterns -----------------------------
def _float_key(widened: torch.Tensor) -> torch.Tensor:
    """float_key of the device-widened values (common.cuh) as int64: the order both select modes must reproduce"""
    b = widened.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = torch.where(b == 0x80000000, torch.zeros_like(b), b)
    return torch.where(b >= 0x80000000, (~b) & 0xFFFFFFFF, b | 0x80000000)


def test_every_half_pattern_is_ranked_through_the_half_select(dev):
    """All 65536 half bit patterns, ranked by float_key of their device widening into 8 groups of 8192.  Image g holds group g
    and every lower-ranked pattern (padded with copies of the lowest one to 65536 scores, in a seeded random order), so the
    top 8192 of image g is group g: every pattern's rank shows in the output of one image.  Further calls put the cut at
    other ranks.  RpnDecode ([8, 16, 64, 64]) and PredictorDecode ([8, 8192, 8]) read the same images."""
    pats = torch.arange(-32768, 32768, dtype=torch.int16, device=dev).view(torch.float16)
    key = _float_key(pats.float())
    order = torch.sort(key, descending=True, stable=True).indices               # rank -> pattern
    rng = np.random.default_rng(520)
    imgs = torch.empty((8, 65536), dtype=torch.float16, device=dev)
    for g in range(8):
        mine = pats[order[8192 * g:]]
        pad = pats[order[-1:]].expand(65536 - mine.numel())
        row = torch.cat([mine, pad])
        imgs[g] = row[torch.from_numpy(rng.permutation(65536)).to(dev)]
    deltas_r = torch.zeros((8, 64, 64, 64), dtype=torch.float16, device=dev)
    deltas_p = torch.zeros((8, 65536, 4), dtype=torch.float16, device=dev)
    anchors = [v for a in range(16) for v in (-8.0 - a, -8.0, 8.0 + a, 8.0)]        # 16 anchors, every box inside the image
    props = torch.tensor([[0.0, 0.0, 64.0, 48.0]], device=dev).expand(8, 8192, 4).contiguous()
    seen = torch.zeros(65536, dtype=torch.bool, device=dev)
    for top_n in (8192, 8191, 4097, 1000, 1):
        got = _rpn(dev, imgs.view(8, 16, 64, 64), deltas_r, top_n, anchors, 64, 64, (1100, 1100))
        exp = _rpn(dev, imgs.view(8, 16, 64, 64).float(), deltas_r.float(), top_n, anchors, 64, 64, (1100, 1100))
        _assert_same(got, exp, top_n)
        if top_n == 8192:
            # the output of image g is group g: in rank order (-0.0 and +0.0 tie, so they are compared as values), and as a
            # set of half bit patterns every pattern of the group once
            for g in range(8):
                mine = pats[order[8192 * g:8192 * (g + 1)]]
                out, nan = got[0][g], torch.isnan(got[0][g])
                assert torch.equal(nan, torch.isnan(mine)) and torch.equal(out[~nan], mine.float()[~nan])
                out_bits = out[~nan].half().view(torch.int16).sort().values
                assert torch.equal(out_bits, mine[~nan].view(torch.int16).sort().values)
                seen[order[8192 * g:8192 * (g + 1)]] = True
    assert bool(seen.all())
    got = _pred(dev, imgs.view(8, 8192, 8), deltas_p, props)
    exp = _pred(dev, imgs.view(8, 8192, 8).float(), deltas_p.float(), props)
    _assert_same(got, exp, "predictor")


# ------------------------------------------------------------------ the chain, the ABI ----------------------------------
def test_rcnn_head_chain_half_heads_equal_the_widened_heads(dev):
    B = 8
    chain = RcnnHeadChain(B, synth.rcnn_anchors(), dev)
    s, d = synth.rpn_inputs(B, seed=530)
    cs, cd, _ = synth.predictor_inputs(B, seed=531, N=1000, Ccls=80)
    h = [torch.from_numpy(x.astype(np.float16)).to(dev) for x in (s, d, cs, cd)]
    a = [t.clone() for t in chain.run_device(*h)]
    b = [t.clone() for t in chain.run_device(*[t.float() for t in h])]
    torch.cuda.synchronize()
    assert (a[0][:, 0] > 0).all()
    _assert_same(a, b, "chain")


def test_typed_fp32_calls_equal_the_untyped_ones_byte_for_byte(dev):
    lib = L.load()
    B, A, H, W, top_n = 2, 15, 50, 67, 6000
    s, d = (torch.from_numpy(x).to(dev) for x in synth.rpn_inputs(B, seed=540))
    anchors = synth.rcnn_anchors()
    anc = (C.c_float * len(anchors))(*anchors.tolist())
    ws = _ws(dev)
    outs = [[_poisoned((B, top_n), dev), _poisoned((B, top_n, 4), dev)] for _ in range(2)]
    args = lambda o: (B, s.data_ptr(), d.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), H, W, IMG_H, IMG_W, 16.0, anc, A, top_n,  # noqa: E731
                      ws.data_ptr(), ws.numel(), None)
    assert lib.trtx_rpn_decode(*args(outs[0])) == 0 and lib.trtx_rpn_decode_typed(L.F32, *args(outs[1])) == 0
    torch.cuda.synchronize()
    _assert_same(outs[0], outs[1], "rpn")
    N, Cc = 1000, 80
    cs, cd, pr = (torch.from_numpy(x).to(dev) for x in synth.predictor_inputs(B, seed=541, N=N, Ccls=Cc))
    w4 = (C.c_float * 4)(*W4)
    outs = [[_poisoned((B, N), dev), _poisoned((B, N, 4), dev), _poisoned((B, N), dev)] for _ in range(2)]
    pargs = lambda o: (B, cs.data_ptr(), cd.data_ptr(), pr.data_ptr(), *(t.data_ptr() for t in o), N, Cc, IMG_H, IMG_W, w4,  # noqa: E731
                       ws.data_ptr(), ws.numel(), None)
    assert lib.trtx_predictor_decode(*pargs(outs[0])) == 0 and lib.trtx_predictor_decode_typed(L.F32, *pargs(outs[1])) == 0
    torch.cuda.synchronize()
    _assert_same(outs[0], outs[1], "predictor")


def test_rejections_leave_poisoned_outputs_untouched(dev):
    """Unknown dtype and misaligned half pointers through the C ABI -> -TRTX_ERR_INVALID; other or mixed dtypes through the
    Python wrappers -> TrtxError before the library is called.  The poisoned outputs stay as they were."""
    lib = L.load()
    INV = -L.ERR_INVALID
    B, A, H, W, top_n = 1, 15, 8, 9, 500
    s16 = torch.zeros(A * H * W + 8, dtype=torch.float16, device=dev)
    d16 = torch.zeros(4 * A * H * W + 8, dtype=torch.float16, device=dev)
    os_, ob = _poisoned((B, top_n), dev), _poisoned((B, top_n, 4), dev)
    anchors = synth.rcnn_anchors()
    anc = (C.c_float * len(anchors))(*anchors.tolist())
    ws = _ws(dev)

    def rpn(dtype, sp, dp):
        return lib.trtx_rpn_decode_typed(dtype, B, sp, dp, os_.data_ptr(), ob.data_ptr(), H, W, 128, 144, 16.0, anc, A, top_n,
                                         ws.data_ptr(), ws.numel(), None)

    assert rpn(2, s16.data_ptr(), d16.data_ptr()) == rpn(-1, s16.data_ptr(), d16.data_ptr()) == INV
    assert rpn(L.F16, s16.data_ptr() + 1, d16.data_ptr()) == rpn(L.F16, s16.data_ptr(), d16.data_ptr() + 1) == INV
    N, Cc = 50, 8
    ps = torch.zeros(N * Cc + 8, dtype=torch.float16, device=dev)
    pdl = torch.zeros(N * Cc * 4 + 8, dtype=torch.float16, device=dev)
    props = torch.zeros((B, N, 4), device=dev)
    po = [_poisoned((B, N), dev), _poisoned((B, N, 4), dev), _poisoned((B, N), dev)]
    w4 = (C.c_float * 4)(*W4)

    def pred(dtype, sp, dp):
        return lib.trtx_predictor_decode_typed(dtype, B, sp, dp, props.data_ptr(), *(t.data_ptr() for t in po), N, Cc, IMG_H, IMG_W,
                                               w4, ws.data_ptr(), ws.numel(), None)

    assert pred(7, ps.data_ptr(), pdl.data_ptr()) == INV
    assert pred(L.F16, ps.data_ptr() + 1, pdl.data_ptr()) == INV
    for off in (1, 2, 4, 6):                                                    # half deltas need 8 bytes
        assert pred(L.F16, ps.data_ptr(), pdl.data_ptr() + off) == INV
    # the Python wrappers
    rp = P.RpnDecodePlugin(top_n, anchors, 16.0, 128, 144, H, W)
    sv, dv = s16[:A * H * W].view(B, A, H, W), d16[:4 * A * H * W].view(B, 4 * A, H, W)
    for ins, outs in (([sv, dv.float()], [os_, ob]), ([sv.bfloat16(), dv.bfloat16()], [os_, ob]), ([sv, dv], [os_.half(), ob])):
        with pytest.raises(L.TrtxError):
            rp.enqueue(B, ins, outs, ws)
    pp = P.PredictorDecodePlugin(N, IMG_H, IMG_W, W4, Cc)
    psv, pdv = ps[:N * Cc].view(B, N, Cc), pdl[:N * Cc * 4].view(B, N * Cc, 4)
    for ins, outs in (([psv, pdv.float(), props], po), ([psv, pdv, props.half()], po), ([psv.double(), pdv.double(), props], po),
                      ([psv, pdv, props], [po[0], po[1], po[2].half()])):
        with pytest.raises(L.TrtxError):
            pp.enqueue(B, ins, outs, ws)
    torch.cuda.synchronize()
    for t in (os_, ob, *po):
        assert (t.view(torch.uint8) == 0x5a).all()
