"""Mask R-CNN pre-process on the GPU (trtx_rcnn_preprocess_enqueue, the device form of preprocessImg + the float widening of
rcnn/rcnn.cpp:497-506) against the CPU oracle, bit for bit.  Every output is pre-filled with a sentinel, so an equal result
also proves that every element was written.  The oracle itself is pinned to cv2 in tests/test_rcnn_pre_cpu.py."""
import numpy as np
import pytest
import torch

from oracle import rcnn_pre as RP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
SENTINEL = -7.0


def _frames(rng, sizes, dev, pitch_pad=0, offset=0):
    """u8 HWC frames on the device (rows padded by `pitch_pad` or `pitch_pad` + 1 bytes to an odd pitch, base `offset` bytes
    into an allocation) and their host copies."""
    host, devs = [], []
    for (w, h) in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        pitch = 3 * w + pitch_pad
        pitch += pitch_pad > 0 and pitch % 2 == 0        # padded rows get an odd pitch
        buf = torch.zeros(offset + pitch * h, dtype=torch.uint8, device=dev)
        view = buf[offset:].as_strided((h, w, 3), (pitch, 3, 1))
        view.copy_(torch.from_numpy(img))
        host.append(img)
        devs.append(view)
    return host, devs


def _check(host, devs, net_w, net_h, dev, out=None):
    if out is None:
        out = torch.full((len(devs), net_h, net_w, 3), SENTINEL, dtype=torch.float32, device=dev)
    got = P.rcnn_preprocess(devs, net_w, net_h, out=out)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    for b, img in enumerate(host):
        exp = RP.rcnn_preprocess(img, net_w, net_h)
        assert exp is not None
        assert np.array_equal(got[b], exp[0]), (b, img.shape, int((got[b] != exp[0]).sum()))
    return got


@pytest.mark.parametrize("img_w,img_h,net_w,net_h", [(640, 480, 1067, 800), (1920, 1080, 1333, 750)])
def test_rcnn_preprocess_b8_matches_oracle(dev, img_w, img_h, net_w, net_h):
    host, devs = _frames(np.random.default_rng(img_w), [(img_w, img_h)] * 8, dev)
    _check(host, devs, net_w, net_h, dev)


def test_rcnn_preprocess_mixed_batch_one_call(dev):
    """Landscape, portrait, exact 2x down, 2x up, scale 1, 1 x 1, top/bottom padding, an odd pitch and a 1-byte-offset base."""
    rng = np.random.default_rng(7)
    sizes = [(640, 480), (480, 640), (2134, 1600), (533, 400), (1067, 800), (1, 1), (3, 2), (1920, 1080), (641, 479)]
    h1, d1 = _frames(rng, sizes[:5], dev)
    h2, d2 = _frames(rng, sizes[5:7], dev, pitch_pad=5)                 # odd pitch
    h3, d3 = _frames(rng, sizes[7:], dev, pitch_pad=1, offset=1)        # odd pitch, base 1 byte into the allocation
    assert all(d.stride(0) % 2 == 1 for d in d2 + d3) and d3[0].data_ptr() % 2 == 1
    _check(h1 + h2 + h3, d1 + d2 + d3, 1067, 800, dev)


def test_rcnn_preprocess_more_images_than_one_launch(dev):
    """70 images: more than the 64 descriptors of one launch; mixed sizes so that every chunk differs."""
    rng = np.random.default_rng(8)
    sizes = [(int(w), int(h)) for w, h in rng.integers(8, 200, (70, 2))]
    host, devs = _frames(rng, sizes, dev)
    _check(host, devs, 96, 72, dev)


def test_rcnn_preprocess_dst_offset_by_4_bytes(dev):
    rng = np.random.default_rng(9)
    host, devs = _frames(rng, [(640, 480), (480, 640), (333, 517)], dev)
    net_w, net_h = 1067, 800
    n = 3 * net_h * net_w * 3
    buf = torch.full((n + 1,), SENTINEL, dtype=torch.float32, device=dev)
    out = buf[1:].view(3, net_h, net_w, 3)
    assert out.data_ptr() % 16 == 4
    _check(host, devs, net_w, net_h, dev, out=out)
    assert buf[0].item() == SENTINEL


def test_rcnn_preprocess_rejected_call_writes_nothing(dev):
    rng = np.random.default_rng(10)
    _, devs = _frames(rng, [(640, 480), (1, 5000)], dev)
    out = torch.full((2, 800, 1067, 3), SENTINEL, dtype=torch.float32, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        P.rcnn_preprocess(devs, 1067, 800, out=out)
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
