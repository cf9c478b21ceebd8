"""The bicubic letterbox pre-process on the device: trtx_cubic_preprocess_enqueue against the CPU oracle (oracle/cubic_oracle.c,
pinned to cv2's 8-bit INTER_CUBIC without IPP by tests/test_cubic_pre_cpu.py), bit for bit, for yolov3-tiny and
retinafaceAntiCov."""

import numpy as np
import pytest
import torch

from oracle import cubic as CO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
VARIANTS = [(L.CUBIC_YOLOV3_TINY, 608), (L.CUBIC_ANTICOV, 640)]
# up- and downscales, the identity at both nets, 1-pixel-wide and -tall frames, odd sizes, portrait, a 4x vertical shrink
MIXED = [(1920, 1080), (1280, 720), (608, 608), (640, 640), (640, 480), (480, 640), (300, 200), (2, 2), (1, 3), (3, 1),
         (97, 301), (731, 1299), (3840, 2160), (2432, 600), (53, 77)]


def _frame(rng, w, h, dev, extra):
    """A random u8 BGR frame [h, w, 3] on the device, read through a pitch of 3 * w + extra + 1 bytes from an odd base."""
    buf = torch.from_numpy(rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)).to(dev)
    return buf[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def _expect(frames, variant, net_w, net_h):
    return np.stack([CO.preprocess(_host(f), variant, net_w, net_h)[0] for f in frames])


@pytest.mark.parametrize("variant,net", VARIANTS)
def test_mixed_sizes_pitched_odd_bases_equal_oracle(dev, variant, net):
    """One call over frames of mixed sizes (enlarged and shrunk), pitch > 3 * width at odd bases, into a dst that is only
    4-byte aligned, equals the oracle bit for bit; nothing around the output is written, and the frames are not."""
    rng = np.random.default_rng(1 + variant)
    frames = [_frame(rng, w, h, dev, 5 + 3 * (i % 4)) for i, (w, h) in enumerate(MIXED)]
    before = [_host(f) for f in frames]
    n = len(frames) * 3 * net * net
    big = torch.full((n + 8,), -7.0, dtype=torch.float32, device=dev)
    P.cubic_preprocess(frames, variant, out=big[1:1 + n].view(len(frames), 3, net, net), net_w=net, net_h=net)
    got = big.cpu().numpy()
    exp = _expect(frames, variant, net, net)
    for i in range(len(frames)):
        assert np.array_equal(got[1:1 + n].reshape(-1, 3, net, net)[i], exp[i]), MIXED[i]
        assert np.array_equal(_host(frames[i]), before[i])
    assert got[0] == -7.0 and (got[1 + n:] == -7.0).all()


@pytest.mark.parametrize("variant,net", VARIANTS)
def test_saturating_frames_and_rectangular_net(dev, variant, net):
    """Frames of only 0 and 255 (the cubic overshoot saturates on both sides) into a rectangular net."""
    rng = np.random.default_rng(5)
    frames = [(_frame(rng, w, h, dev, 2) >> 7) * 255 for w, h in ((1920, 1080), (333, 517), (64, 48))]
    out = P.cubic_preprocess(frames, variant, net_w=net, net_h=net // 2 + 3)
    assert np.array_equal(out.cpu().numpy(), _expect(frames, variant, net, net // 2 + 3))


@pytest.mark.parametrize("variant,net", VARIANTS)
def test_70_frames_two_launches_and_graph_replay(dev, variant, net):
    """70 frames take two launches; a graph-captured call replayed on overwritten frames gives the oracle's bytes for them."""
    rng = np.random.default_rng(9 + variant)
    sizes = [MIXED[i % len(MIXED)] if i % 5 else (1280, 720) for i in range(70)]
    sizes = [(w, h) if w * h <= 1280 * 720 else (w // 3, h // 3) for w, h in sizes]
    frames = [_frame(rng, w, h, dev, i % 7) for i, (w, h) in enumerate(sizes)]
    out = torch.empty((70, 3, net, net), dtype=torch.float32, device=dev)
    P.cubic_preprocess(frames, variant, out=out, net_w=net, net_h=net)
    assert np.array_equal(out.cpu().numpy(), _expect(frames, variant, net, net))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.cubic_preprocess(frames, variant, out=out, net_w=net, net_h=net)
    for f in frames:
        f.copy_(torch.from_numpy(rng.integers(0, 256, tuple(f.shape), dtype=np.uint8)))
    out.fill_(5.0)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), _expect(frames, variant, net, net))


def test_rejected_calls_write_nothing(dev):
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 320, 180, dev, 5) for _ in range(69)] + [_frame(rng, 1, 700, dev, 0)]
    out = torch.full((70, 3, 608, 608), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):  # frame 69's rectangle is empty: no launch for frames 0..63 either
        P.cubic_preprocess(frames, L.CUBIC_YOLOV3_TINY, out=out)
    descs = P._image_descs(frames[:2])
    lib = L.load()
    assert lib.trtx_cubic_preprocess_enqueue(7, descs, 2, 608, 608, out.data_ptr(), None) == L.ERR_INVALID
    assert lib.trtx_cubic_preprocess_enqueue(0, descs, 2, 608, 608, out.data_ptr() + 2, None) == L.ERR_INVALID
    descs[1].pitch = 3 * 320 - 1
    assert lib.trtx_cubic_preprocess_enqueue(1, descs, 2, 608, 608, out.data_ptr(), None) == L.ERR_INVALID
    wide = torch.full((1, 3, 1200, 1200), 3.0, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):  # 16 staged rows of a 1200-wide rectangle exceed shared memory
        P.cubic_preprocess([_frame(rng, 4800, 100, dev, 0)], L.CUBIC_ANTICOV, out=wide, net_w=1200, net_h=1200)
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (wide == 3.0).all()
