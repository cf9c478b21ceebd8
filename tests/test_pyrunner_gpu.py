"""The Python runners' pre- and post-process on the device, bit for bit with the runners' own numpy: the digests of
preprocess_image and post_process in tests/golden/ref_pyrunner_host.npz (recorded from the reference runners by
tests/test_pyrunner_cpu.py on the same seeded inputs), and the oracle's tie and termination rules where the runners leave
the result open."""

import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import pyrunner as PR
from tensorrtx_b200 import plugins as P

pytestmark = pytest.mark.gpu
R = G.RefOutputs("ref_pyrunner_host")


def _pitched(f, dev, extra):
    """Frame f [h, w, 3] on the device behind a pitch of 3 * w + extra + 1 bytes from an odd base."""
    h, w, _ = f.shape
    buf = torch.zeros((h, 3 * w + extra + 1), dtype=torch.uint8)
    buf[:, 1:1 + 3 * w] = torch.from_numpy(f.reshape(h, 3 * w))
    return buf.to(dev)[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


@pytest.mark.parametrize("net", PR.PRE_NETS)
def test_preprocess_equals_runner(dev, net):
    """One call over pitched frames of mixed sizes (592 x 333, 1920 x 1080, 1-pixel sides) equals preprocess_image; nothing
    around the output is written."""
    net_w, net_h = net
    frames = [_pitched(f, dev, e) for f, (_, _, e) in zip(PR.pre_frames(net), PR.PRE_FRAMES)]
    n = len(frames) * 3 * net_w * net_h
    big = torch.full((n + 2,), -7.0, dtype=torch.float32, device=dev)
    plan = P.PyRunnerPreprocessPlan(frames, out=big[1:1 + n].view(len(frames), 3, net_h, net_w), net_w=net_w, net_h=net_h)
    plan.enqueue()
    got = big.cpu().numpy()
    assert got[0] == -7.0 and got[-1] == -7.0
    for i, img in enumerate(got[1:1 + n].reshape(-1, 3, net_h, net_w)):
        R.equal(f"pre-{net_w}x{net_h}-{i}", img)


@pytest.mark.parametrize("key,runner,dets,sizes", PR.post_cases(P.PYRUNNER_PRESETS), ids=lambda v: v if isinstance(v, str) else "")
def test_postprocess_equals_runner(dev, key, runner, dets, sizes):
    """Every preset at b32 with mixed frame sizes equals post_process bit for bit; floats past each count are zero."""
    post = P.PyRunnerPostprocess(runner, max_rows=1000)
    out = torch.full((len(sizes), 1 + 1000 * 6), -3.0, dtype=torch.float32, device=dev)
    post(torch.from_numpy(dets).to(dev), sizes, rows_out=out)
    rows = out.cpu().numpy()
    R.equal(key, PR.canonical(PR.device_rows(rows)))
    for r in rows:
        assert (r[1 + 6 * int(r[0]):] == 0).all()
    exp = PR.canonical([PR.postprocess(d, w, h, P.PYRUNNER_PRESETS[runner]) for d, (w, h) in zip(dets, sizes)])
    assert np.array_equal(PR.canonical(PR.device_rows(rows)), exp, equal_nan=True)


def _crafted(rng, max_rows):
    """Rows the runners leave open: ties in confidence that interact, NaN labels, NaN corners, inverted boxes, and many
    rows on one spot (every row passes conf and suppresses the next)."""
    F = 6
    bufs = []
    for kind in range(4):
        t = np.zeros((max_rows, F), np.float32)
        k = max_rows if kind == 3 else 300
        c = rng.uniform(0, 640, (k, 2))
        wh = rng.uniform(5, 120, (k, 2))
        t[:k, :4] = np.concatenate([c - wh / 2, c + wh / 2], 1)
        t[:k, 4] = rng.choice(np.float32([0.5, 0.6, 0.75, 0.9]), k)  # ties everywhere
        t[:k, 5] = rng.integers(0, 3, k)
        if kind == 1:
            t[rng.choice(k, 40, replace=False), 5] = np.nan
            t[rng.choice(k, 20, replace=False), rng.integers(0, 4)] = np.nan
        if kind == 2:
            inv = rng.choice(k, 60, replace=False)
            t[inv, :4] = t[inv][:, [2, 3, 0, 1]]
        if kind == 3:
            t[:k, :4] = [100, 100, 200, 200]
            t[:k, 4] = rng.uniform(0.5, 1.0, k)
            t[::7, 4] = 0.75
        b = np.zeros(1 + max_rows * F, np.float32)
        b[0] = k
        b[1:] = t.reshape(-1)
        bufs.append(b)
    return np.stack(bufs)


@pytest.mark.parametrize("max_rows", [300, 2048])
def test_ties_and_termination_equal_oracle(dev, max_rows):
    """Equal confidences in ascending row order, and front rows consumed once, as the oracle states them."""
    rng = np.random.default_rng(max_rows)
    dets = _crafted(rng, max_rows)
    sizes = [(1920, 1080), (640, 640), (333, 592), (1280, 720)]
    post = P.PyRunnerPostprocess("yolov10_det_trt", max_rows=max_rows)
    rows = post(torch.from_numpy(dets).to(dev), sizes).cpu().numpy()
    for b, (w, h) in enumerate(sizes):
        exp = PR.postprocess(dets[b], w, h, P.PYRUNNER_PRESETS["yolov10_det_trt"])
        got = PR.device_rows(rows[b:b + 1])[0]
        assert got.shape == exp.shape and np.array_equal(got, exp, equal_nan=True), b


def test_graph_replay_and_many_frames(dev):
    """70 frames (two launches) captured in a CUDA graph and replayed on new rows give the eager result."""
    cases = PR.post_cases({"yolov8_det_trt": P.PYRUNNER_PRESETS["yolov8_det_trt"]}, batch=35)
    dets = np.concatenate([c[2] for c in cases])
    sizes = cases[0][3] + cases[1][3]
    post = P.PyRunnerPostprocess("yolov8_det_trt")
    src = torch.zeros(dets.shape, dtype=torch.float32, device=dev)
    out = torch.zeros((len(sizes), 1 + 6000), dtype=torch.float32, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        post(src, sizes, rows_out=out, stream=s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        post(src, sizes, rows_out=out, stream=s)
    src.copy_(torch.from_numpy(dets))
    g.replay()
    torch.cuda.synchronize()
    eager = post(src, sizes).cpu().numpy()
    assert np.array_equal(out.cpu().numpy(), eager)
    exp = PR.canonical([PR.postprocess(d, w, h, P.PYRUNNER_PRESETS["yolov8_det_trt"]) for d, (w, h) in zip(dets, sizes)])
    assert np.array_equal(PR.canonical(PR.device_rows(eager)), exp)
