"""YOLO classification pre- and post-process on the GPU (trtx_cls_preprocess_enqueue, trtx_cls_postprocess_enqueue) against the
CPU oracle (oracle/cls_oracle.c, pinned to cv2 and to the drivers' compiled code in tests/test_cls_cpu.py).  The pre-process is
compared bit for bit on outputs pre-filled with a sentinel, so an equal result also proves that every element was written.  The
post-process's probabilities come from CUDA's expf (within 2 ulp of the host's): they are compared within rtol 2e-6, the
indices exactly where no two probabilities of a row are that close, and always against the oracle's order of the device's own
probabilities."""
import numpy as np
import pytest
import torch

from oracle import cls as CO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
SENTINEL = -7.0
RTOL = 2e-6


def _frames(rng, sizes, dev, pitch_pad=0, offset=0):
    """u8 HWC frames on the device (rows padded to an odd pitch when pitch_pad > 0, base `offset` bytes into an allocation)
    and their host copies."""
    host, devs = [], []
    for (w, h) in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        pitch = 3 * w + pitch_pad
        pitch += pitch_pad > 0 and pitch % 2 == 0
        buf = torch.zeros(offset + pitch * h, dtype=torch.uint8, device=dev)
        view = buf[offset:].as_strided((h, w, 3), (pitch, 3, 1))
        view.copy_(torch.from_numpy(img))
        host.append(img)
        devs.append(view)
    return host, devs


def _check_pre(host, devs, variant, net_w, net_h, dev, out=None):
    if out is None:
        out = torch.full((len(devs), 3, net_h, net_w), SENTINEL, dtype=torch.float32, device=dev)
    got = P.cls_preprocess(devs, variant, net_w, net_h, out=out)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    for b, img in enumerate(host):
        exp = CO.cls_preprocess(img, variant, net_w, net_h)
        assert exp is not None
        assert np.array_equal(got[b], exp[0]), (variant, b, img.shape, int((got[b] != exp[0]).sum()))


MIXED = [(640, 480), (480, 640), (224, 224), (300, 224), (224, 301), (448, 448), (896, 600), (100, 80), (1, 1), (1, 9),
         (7, 1), (1920, 1080), (641, 480), (333, 517)]


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_cls_preprocess_mixed_batch(dev, variant):
    """Landscape, portrait, square; m == net (a plain copy), m == 2 net (the 2x fast path), upscales, 1 x 1, 1 x N, odd w - m;
    odd pitches and a 1-byte-offset base, in one call."""
    rng = np.random.default_rng(70 + variant)
    h1, d1 = _frames(rng, MIXED[:8], dev)
    h2, d2 = _frames(rng, MIXED[8:11], dev, pitch_pad=5)
    h3, d3 = _frames(rng, MIXED[11:], dev, pitch_pad=1, offset=1)
    assert all(d.stride(0) % 2 == 1 for d in d2 + d3) and d3[0].data_ptr() % 2 == 1
    _check_pre(h1 + h2 + h3, d1 + d2 + d3, variant, 224, 224, dev)


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_cls_preprocess_rectangular_net_and_dst_offset(dev, variant):
    """A non-square engine input, written 4 bytes off a 16-byte boundary, with sentinels on both sides."""
    rng = np.random.default_rng(72 + variant)
    host, devs = _frames(rng, [(640, 480), (480, 640), (333, 517)], dev)
    net_w, net_h = 161, 97
    n = 3 * 3 * net_h * net_w
    buf = torch.full((n + 2,), SENTINEL, dtype=torch.float32, device=dev)
    out = buf[1:n + 1].view(3, 3, net_h, net_w)
    assert out.data_ptr() % 16 == 4
    _check_pre(host, devs, variant, net_w, net_h, dev, out=out)
    assert buf[0].item() == SENTINEL and buf[-1].item() == SENTINEL


@pytest.mark.parametrize("variant", [L.YOLO_V8, L.YOLO_V5])
def test_cls_preprocess_70_frames_and_graph(dev, variant):
    """70 frames (two launches) of mixed sizes, then the same call captured in a CUDA graph and replayed on new pixels."""
    rng = np.random.default_rng(74 + variant)
    sizes = [(int(w), int(h)) for w, h in rng.integers(1, 700, (70, 2))]
    host, devs = _frames(rng, sizes, dev)
    _check_pre(host, devs, variant, 224, 224, dev)
    out = torch.full((70, 3, 224, 224), SENTINEL, dtype=torch.float32, device=dev)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        P.cls_preprocess(devs, variant, 224, 224, out=out)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            P.cls_preprocess(devs, variant, 224, 224, out=out)
    for b, d in enumerate(devs):
        host[b] = rng.integers(0, 256, host[b].shape, dtype=np.uint8)
        d.copy_(torch.from_numpy(host[b]))
    out.fill_(SENTINEL)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    _check_pre(host, devs, variant, 224, 224, dev, out=out)


def test_cls_preprocess_rejected_call_writes_nothing(dev):
    rng = np.random.default_rng(76)
    _, devs = _frames(rng, [(640, 480), (1, 5000)], dev)
    out = torch.full((2, 3, 224, 224), SENTINEL, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.cls_preprocess(devs, L.YOLO_V5, 224, 224, out=out)
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())


# ------------------------------------------------------------------ post-process ---------------------------------
def _post(logits, k, softmax, dev, probs=True):
    x = torch.from_numpy(logits).to(dev)
    b, c = logits.shape
    idx = torch.full((b, k), -5, dtype=torch.int32, device=dev)
    val = torch.full((b, k), SENTINEL, dtype=torch.float32, device=dev)
    p = torch.full((b, c), SENTINEL, dtype=torch.float32, device=dev) if probs else None
    L.check(L.load().trtx_cls_postprocess_enqueue(int(softmax), b, c, x.data_ptr(), k, idx.data_ptr(), val.data_ptr(),
                                                  p.data_ptr() if probs else None, torch.cuda.current_stream().cuda_stream),
            "trtx_cls_postprocess_enqueue")
    torch.cuda.synchronize()
    return idx.cpu().numpy(), val.cpu().numpy(), (p.cpu().numpy() if probs else None)


def _check_post(logits, k, softmax, dev):
    idx, val, probs = _post(logits, k, softmax, dev)
    b, c = logits.shape
    kk = min(k, c)
    exp_res = CO.softmax(logits) if softmax else logits
    nan = np.isnan(exp_res)
    assert np.array_equal(np.isnan(probs), nan)
    np.testing.assert_allclose(probs[~nan], exp_res[~nan], rtol=RTOL, atol=0)
    if not softmax:
        assert np.array_equal(probs.view(np.uint32), logits.view(np.uint32))       # raw: the bits, NaN signs included
    # the selection and order, exact, of the device's own probabilities
    assert np.array_equal(idx[:, :kk], CO.topk(probs, k))
    assert np.array_equal(val[:, :kk].view(np.uint32), np.take_along_axis(probs, idx[:, :kk].astype(np.int64), 1).view(np.uint32))
    # past min(k, C): untouched
    assert (idx[:, kk:] == -5).all() and (val[:, kk:] == SENTINEL).all()
    # and the oracle's indices, on rows where no two probabilities are within the tolerance
    exp_idx = CO.topk(exp_res, k)
    for r in range(b):
        s = np.sort(exp_res[r][~nan[r]])
        if s.size < 2 or np.all(np.diff(s) > RTOL * np.abs(s[1:]) * 2):
            assert np.array_equal(idx[r, :kk], exp_idx[r]), r
    # probs NULL gives the same indices and values
    idx2, val2, _ = _post(logits, k, softmax, dev, probs=False)
    assert np.array_equal(idx2, idx) and np.array_equal(val2.view(np.uint32), val.view(np.uint32))


@pytest.mark.parametrize("softmax", [1, 0])
@pytest.mark.parametrize("c", [1, 2, 1000, 1001])
def test_cls_postprocess_matches_oracle(dev, softmax, c):
    rng = np.random.default_rng(80 + c + softmax)
    x = (rng.standard_normal((6, c)) * 4).astype(np.float32)
    for k in sorted({1, 3, 5, c}):
        _check_post(x, k, softmax, dev)


def test_cls_postprocess_ties_signed_zero_inf_nan_raw(dev):
    """Raw mode: equal values in ascending index, -0.0 == +0.0, +NaN above +inf, -NaN below -inf."""
    x = np.zeros((3, 16), np.float32)
    x[0] = [1, 2, 2, 1, 2, 0, -0.0, 0, -0.0, 3, 3, -1, -1, 3, 0, 2]
    x[1] = [np.inf, -np.inf, np.nan, 1, 0, -0.0, np.inf, np.nan, -np.inf, 5, -5, 0, 1, 1, np.nan, -1]
    x[1, 7] = -np.abs(np.float32(np.nan))
    x[2] = 0.5
    for k in (1, 3, 5, 16, 20):
        _check_post(x, k, 0, dev)
    idx, _, _ = _post(x, 16, 0, dev)
    assert idx[0].tolist() == [9, 10, 13, 1, 2, 4, 15, 0, 3, 5, 6, 7, 8, 14, 11, 12]
    assert idx[1][:3].tolist() == [2, 14, 0] and idx[1][-2:].tolist() == [8, 7]
    assert idx[2].tolist() == list(range(16))


def test_cls_postprocess_overflow_and_underflow_rows(dev):
    """A logit above 88.72 makes expf inf and its probability inf / inf = NaN; an all-underflow row makes every one 0 / 0."""
    rng = np.random.default_rng(90)
    x = (rng.standard_normal((3, 1000)) * 2).astype(np.float32)
    x[0, 17] = 95.0
    x[1, :] = -200.0
    x[2, [5, 500]] = 100.0
    for k in (1, 3, 1000):
        _check_post(x, k, 1, dev)
    idx, _, probs = _post(x, 3, 1, dev)
    assert np.isnan(probs[0, 17]) and idx[0, 0] == 17
    assert np.isnan(probs[1]).all() and idx[1].tolist() == [0, 1, 2]
    assert idx[2, :2].tolist() == [5, 500]


def test_cls_postprocess_70_images_and_graph(dev):
    rng = np.random.default_rng(91)
    x = (rng.standard_normal((70, 1000)) * 3).astype(np.float32)
    _check_post(x, 5, 1, dev)
    d = torch.from_numpy(x).to(dev)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        P.cls_postprocess(d, 5, True)
        torch.cuda.synchronize()
        idx = torch.zeros((70, 5), dtype=torch.int32, device=dev)
        val = torch.zeros((70, 5), dtype=torch.float32, device=dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            L.check(L.load().trtx_cls_postprocess_enqueue(1, 70, 1000, d.data_ptr(), 5, idx.data_ptr(), val.data_ptr(), None,
                                                          torch.cuda.current_stream().cuda_stream),
                    "trtx_cls_postprocess_enqueue")
    x2 = (rng.standard_normal((70, 1000)) * 3).astype(np.float32)
    d.copy_(torch.from_numpy(x2))
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    ref_idx, ref_val, _ = _post(x2, 5, 1, dev, probs=False)
    assert np.array_equal(idx.cpu().numpy(), ref_idx) and np.array_equal(val.cpu().numpy(), ref_val)
    assert np.array_equal(ref_idx, CO.topk(CO.softmax(x2), 5))


def test_cls_plugins_wrappers(dev):
    rng = np.random.default_rng(92)
    x = (rng.standard_normal((4, 1000)) * 3).astype(np.float32)
    idx, val, probs = P.cls_postprocess(torch.from_numpy(x).to(dev), 3, True, probs=True)
    torch.cuda.synchronize()
    assert idx.shape == (4, 3) and val.shape == (4, 3) and probs.shape == (4, 1000)
    np.testing.assert_allclose(probs.cpu().numpy(), CO.softmax(x), rtol=RTOL, atol=0)
    host, devs = _frames(rng, [(640, 480)], dev)
    out = P.cls_preprocess(devs, L.YOLO_V8, 224, 224)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy()[0], CO.cls_preprocess(host[0], 0, 224, 224)[0])
