"""CenterNet on the GPU: trtx_centernet_preprocess_enqueue and trtx_centernet_decode_enqueue against the CPU oracle
(oracle/centernet_oracle.c) and, where oracle/_ref holds it, the sample's own ctdet_decode."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import centernet as CO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

from test_centernet_cpu import assert_dets, special_heads, tie_free_heads

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _frames(rng, sizes, pitch_pad=0, offset=0):
    """u8 BGR frames on the device, as views into larger buffers when pitch_pad / offset are set (pitched rows, odd bases)"""
    hosts, devs = [], []
    for w, h in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        buf = torch.zeros((h, w + pitch_pad, 3), dtype=torch.uint8, device=DEV).view(-1)
        flat = torch.zeros(buf.numel() + offset, dtype=torch.uint8, device=DEV)
        view = flat[offset:].view(h, w + pitch_pad, 3)[:, :w]
        view.copy_(torch.from_numpy(img))
        hosts.append(img)
        devs.append(view)
    return hosts, devs


MIXED = [(1920, 1080), (1280, 720), (512, 512), (640, 480), (333, 201), (1, 1), (1, 9), (3000, 2000), (2, 2), (480, 640),
         (720, 1280), (7, 300), (1023, 1024)]  # (w, h): portrait frames, w == 1 and 2 x 2 among them


@pytest.mark.parametrize("pitch_pad,offset", [(0, 0), (5, 3), (17, 1)])
def test_preprocess_matches_oracle(pitch_pad, offset):
    rng = np.random.default_rng(3 + pitch_pad)
    hosts, devs = _frames(rng, MIXED, pitch_pad, offset)
    out = P.centernet_preprocess(devs)
    got = out.cpu().numpy()
    for i, img in enumerate(hosts):
        assert np.array_equal(got[i], CO.preprocess(img)), (i, img.shape)


def test_preprocess_70_frames_into_a_4_byte_aligned_dst():
    rng = np.random.default_rng(70)
    sizes = [(int(w), int(h)) for w, h in rng.integers(1, 900, (70, 2))]
    hosts, devs = _frames(rng, sizes)
    n = 70 * 3 * 512 * 512
    buf = torch.full((n + 1,), 7.0, dtype=torch.float32, device=DEV)
    out = buf[1:].view(70, 3, 512, 512)  # base 4 bytes past a 256-byte boundary
    P.centernet_preprocess(devs, out=out)
    got = out.cpu().numpy()
    assert buf[0].item() == 7.0
    for i, img in enumerate(hosts):
        assert np.array_equal(got[i], CO.preprocess(img)), (i, img.shape)


def _decode(heat, wh, reg, k, sizes=None):
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (heat, wh, reg)]
    return P.centernet_decode(*t, k, image_sizes=sizes)


@pytest.mark.parametrize("B", [1, 8, 32])
def test_decode_sample_shape_matches_oracle(B):
    heat, wh, reg = tie_free_heads(B, B, 80, 128, 128)
    sizes = [(640 + 37 * b, 480 + 11 * b) for b in range(B)]
    dets, rows = _decode(heat, wh, reg, 100, sizes)
    dets, rows = dets.cpu().numpy(), rows.cpu().numpy()
    for b in range(B):
        want = CO.decode(heat[b], wh[b], reg[b], 100)
        assert_dets(dets[b], want, b)
        # the rows follow from the device's own dets bit for bit
        assert np.array_equal(rows[b], CO.rows(dets[b], *sizes[b])), b


@pytest.mark.parametrize("shape", [(3, 16, 20, 1), (2, 8, 8, 64), (5, 33, 17, 40), (1, 7, 300, 50), (12, 64, 48, 200),
                                   (1, 3, 1000, 1024), (4, 256, 256, 1024), (1000, 8, 8, 3), (2, 1, 1, 1)],
                         ids=lambda s: "x".join(map(str, s)))
def test_decode_other_shapes_match_oracle(shape):
    Cn, H, W, k = shape
    B = 2
    heat, wh, reg = tie_free_heads(sum(shape), B, Cn, H, W)
    dets = _decode(heat, wh, reg, k).cpu().numpy()
    for b in range(B):
        assert_dets(dets[b], CO.decode(heat[b], wh[b], reg[b], k), (shape, b))


@pytest.mark.parametrize("case", ["ties", "empty", "nan", "plateau", "sparse"])
@pytest.mark.parametrize("k", [1, 37, 120])
def test_decode_edge_cases_match_oracle(case, k):
    heat, wh, reg = special_heads(case)
    dets = _decode(heat[None], wh[None], reg[None], k).cpu().numpy()
    assert_dets(dets[0], CO.decode(heat, wh, reg, k), case)


def test_decode_saturated_maps_cut_the_candidate_list():
    """Every cell of a saturated 256 x 256 map is a peak of value 1.0f, so the shared candidate list overflows and is cut
    to K again and again; the K kept are the first cells in flat order, with a NaN and a few larger-ranked cells mixed in."""
    rng = np.random.default_rng(9)
    Cn, H, W, k = 3, 256, 256, 1000
    heat = np.full((1, Cn, H, W), 30.0, np.float32)
    heat[0, 2, 200, 100] = np.nan
    heat[0, 1, 255, 255] = 30.0
    heat[0, 0, :2] = rng.uniform(-2, 2, (2, W))
    wh = rng.uniform(0, 30, (1, 2, H, W)).astype(np.float32)
    reg = rng.uniform(0, 1, (1, 2, H, W)).astype(np.float32)
    dets = _decode(heat, wh, reg, k).cpu().numpy()
    assert_dets(dets[0], CO.decode(heat[0], wh[0], reg[0], k))


def test_decode_matches_the_sample():
    ref = CO.reference()
    if ref is None:
        pytest.skip("oracle/_ref/ref_centernet.pyc not built")
    heat, wh, reg = tie_free_heads(11, 4, 80, 128, 128)
    want = ref.ctdet_decode(torch.from_numpy(heat), torch.from_numpy(wh), torch.from_numpy(reg), K=100).numpy()
    assert_dets(_decode(heat, wh, reg, 100).cpu().numpy(), want)


def test_rejected_calls_write_nothing():
    lib = L.load()
    heat, wh, reg = (torch.zeros((2, c, 16, 16), device=DEV) for c in (4, 2, 2))
    q = L.CenternetParams(4, 16, 16, 10, 512, 4, 0.5)
    ws = torch.empty(lib.trtx_centernet_workspace_size(C.byref(q), 2), dtype=torch.uint8, device=DEV)
    dets = torch.full((2, 10, 6), -7.0, device=DEV)
    rows = torch.full((2, 61), -7.0, device=DEV)
    fw = (C.c_int32 * 4)(640, 480, 0, 480)  # frame 1 has width 0
    args = [heat.data_ptr(), wh.data_ptr(), reg.data_ptr(), ws.data_ptr(), ws.numel(), dets.data_ptr()]
    assert lib.trtx_centernet_decode_enqueue(C.byref(q), 2, *args, fw, rows.data_ptr(), None) == L.ERR_INVALID
    assert lib.trtx_centernet_decode_enqueue(C.byref(q), 2, *args[:4], ws.numel() - 1, args[5], None, None, None) == \
        L.ERR_WORKSPACE
    big = L.CenternetParams(4, 16, 16, 1025, 512, 4, 0.5)
    assert lib.trtx_centernet_decode_enqueue(C.byref(big), 2, *args, None, None, None) == L.ERR_INVALID  # K > H * W
    imgs = [torch.zeros((10, 10, 3), dtype=torch.uint8, device=DEV), torch.zeros((10, 10, 3), dtype=torch.uint8, device=DEV)]
    descs = (L.ImageDesc * 2)(L.ImageDesc(imgs[0].data_ptr(), 10, 10, 30, 0), L.ImageDesc(imgs[1].data_ptr(), 10, 10, 29, 0))
    pre = torch.full((2, 3, 64, 64), -7.0, device=DEV)
    assert lib.trtx_centernet_preprocess_enqueue(descs, 2, 64, pre.data_ptr(), None) == L.ERR_INVALID
    torch.cuda.synchronize()
    for t in (dets, rows, pre):
        assert (t == -7.0).all()


def test_graph_replay_of_the_whole_chain():
    """pre_process of a batch and the decode with frame rows, captured in one CUDA graph and replayed on new inputs."""
    rng = np.random.default_rng(21)
    sizes = [(1920, 1080), (640, 480), (1280, 720)]
    hosts, devs = _frames(rng, sizes)
    B = len(sizes)
    heat, wh, reg = tie_free_heads(5, B, 80, 128, 128)
    t = [torch.from_numpy(a).to(DEV) for a in (heat, wh, reg)]
    pre = torch.empty((B, 3, 512, 512), device=DEV)
    dets = torch.empty((B, 100, 6), device=DEV)
    rows = torch.empty((B, 601), device=DEV)
    q = L.CenternetParams(80, 128, 128, 100, 512, 4, 0.5)
    ws = torch.empty(L.load().trtx_centernet_workspace_size(C.byref(q), B), dtype=torch.uint8, device=DEV)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            P.centernet_preprocess(devs, out=pre)
            P.centernet_decode(*t, 100, image_sizes=sizes, workspace=ws, out=dets, rows_out=rows)
    hosts2, devs2 = _frames(rng, sizes)
    for d, d2 in zip(devs, devs2):
        d.copy_(d2)
    heat2, wh2, reg2 = tie_free_heads(6, B, 80, 128, 128)
    for x, a in zip(t, (heat2, wh2, reg2)):
        x.copy_(torch.from_numpy(a))
    g.replay()
    torch.cuda.synchronize()
    p, dd, rr = pre.cpu().numpy(), dets.cpu().numpy(), rows.cpu().numpy()
    for b in range(B):
        assert np.array_equal(p[b], CO.preprocess(hosts2[b]))
        assert_dets(dd[b], CO.decode(heat2[b], wh2[b], reg2[b], 100))
        assert np.array_equal(rr[b], CO.rows(dd[b], *sizes[b]))
