"""Timing of the RefineDet pre-process (trtx_refinedet_preprocess_enqueue) and post-process
(trtx_refinedet_postprocess_enqueue), and of the reference's libtorch post-process restated in torch on CUDA
(oracle/refinedet.py: the same ATen ops, with nms()'s per-box .item() synchronisations).

  python tools/refinedet_probe.py OUTDIR      -> OUTDIR/refinedet_probe.json (and the card line on stdout)

Workloads: b1 and b32.  Pre-process: 1920x1080 frames into the 320x320 input (1.23 MB of fp32 written per frame).  The call
is timed as 20 launches captured in one CUDA graph, replayed 20 times between two events (probe_timing.graph_us); the
medians over 3 rounds are reported.  Post-process: the four heads of seeded frames with 50 planted objects per class
(0.89 MB per frame, 28.6 MB at b32) and frame rows for 1920x1080, timed the same way.  The torch restatement runs frame
after frame, as the reference does at its batch 1; it is timed with a host clock around a synchronised run of the whole
batch (median of 3).  The NMS is latency-bound, so times are reported in microseconds, not as a share of a roofline."""
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, probe_main  # noqa: E402
from oracle import refinedet as RO  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
NET = RO.NET


def workload(B, rng):
    frames = [torch.from_numpy(rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)).to(dev) for _ in range(B)]
    inp = torch.empty((B, 3, NET, NET), dtype=torch.float32, device=dev)
    h = RO.heads(B, seed=B)
    hd = [torch.from_numpy(x).to(dev) for x in h]
    sizes = [(1920, 1080)] * B
    dets = torch.empty((B, 1 + 6 * 24000), dtype=torch.float32, device=dev)
    rows = torch.empty_like(dets)
    ws = torch.empty(B * 24 * (4 + 2 * 1000) + 512, dtype=torch.uint8, device=dev)
    t = alternating({"pre": lambda: P.refinedet_preprocess(frames, out=inp),
                     "post": lambda: P.refinedet_postprocess(*hd, sizes, workspace=ws, out=dets, rows_out=rows)})
    prior = RO.prior_box(NET, dev)
    ref = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in range(B):
            RO.reference_postprocess(*[x[b] for x in h], device=dev, prior=prior)
        torch.cuda.synchronize()
        ref.append((time.perf_counter() - t0) * 1e6)
    torch.cuda.synchronize()
    return {
        "workload": f"b{B}", "batch": B,
        "pre_us": round(t["pre"], 2), "pre_bytes_written": inp.numel() * 4, "pre_bytes_read": B * 1920 * 1080 * 3,
        "post_us": round(t["post"], 2), "head_bytes": sum(x.nbytes for x in h),
        "rows_per_frame": float(dets[:, 0].mean()),
        "torch_reference_us": round(statistics.median(ref), 1),
        "speedup_vs_torch_reference": round(statistics.median(ref) / t["post"], 1),
    }


def main(outdir):
    rng = np.random.default_rng(0)
    res = []
    for B in (1, 32):
        r = workload(B, rng)
        print(r, flush=True)
        res.append(r)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("refinedet_probe", main)
