"""Unit-scale letterbox over a whole batch of frames held in one [B, h, w, 3] tensor.

The frames are equally sized and equally spaced, so the launch reads them through ONE 3-D tensor map -- the path
bench.py's step takes.  A batch whose frames are not equally spaced reads them through one map per frame.  At scale 1
the letterbox is exact, so the result must equal the oracle bit for bit."""
import numpy as np
import pytest
import torch

from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu

SHAPES = [(640, 640), (480, 640), (640, 480), (416, 640)]  # (h, w): all scale 1 into 640 x 640


def _check(oracle, frames_host, views, odt, dev):
    B = len(views)
    dst = torch.full((B, 3, 640, 640), float("nan"), dtype=odt, device=dev)
    P.PreprocessPlan(views, dst, 640, 640).enqueue()
    got = dst.float().cpu().numpy()
    for b in range(B):
        ref = oracle.warpaffine(frames_host[b], 640, 640)
        if odt == torch.float16:
            ref = ref.astype(np.float16).astype(np.float32)
        assert np.array_equal(got[b], ref), (b, int(np.sum(got[b] != ref)))


@pytest.mark.parametrize("h,w", SHAPES)
@pytest.mark.parametrize("odt", [torch.float32, torch.float16])
def test_unit_letterbox_one_batch_tensor(oracle, dev, h, w, odt):
    fr = synth.frames(32, seed=7 * h + w, h=h, w=w)
    batch = torch.from_numpy(fr).to(dev)
    _check(oracle, fr, list(batch.unbind(0)), odt, dev)


@pytest.mark.parametrize("h,w", SHAPES)
def test_unit_letterbox_unequal_spacing(oracle, dev, h, w):
    B, n = 32, h * w * 3
    fr = synth.frames(B, seed=11 * h + w, h=h, w=w)
    offs = [i * (n + 256) + (i % 3) * 64 for i in range(B)]  # 16-byte aligned, spacing varies
    buf = torch.zeros(offs[-1] + n, dtype=torch.uint8, device=dev)
    views = []
    for i, o in enumerate(offs):
        v = buf[o:o + n].view(h, w, 3)
        v.copy_(torch.from_numpy(fr[i]))
        views.append(v)
    _check(oracle, fr, views, torch.float32, dev)
