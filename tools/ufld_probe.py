"""Timing of the UFLD pre-process (trtx_ufld_preprocess_enqueue) against its write floor, and of the post-process
(trtx_ufld_postprocess_enqueue) against the D2H copy of `prob` it removes.

  python tools/ufld_probe.py OUTDIR      -> OUTDIR/ufld_probe.json (and the card line on stdout)

Pre-process workloads: b8 and b32 of 1280x720 and of 1920x1080 frames into UFLD's 800x288 input (2.76 MB of fp32 per frame).
The call is timed as 20 launches captured in one CUDA graph, replayed 20 times between two events (probe_timing.graph_us); its
floor is a plain device fill (torch fill_) of the bytes it writes, timed the same way; call and floor alternate over 3 rounds
and the medians are reported, with the bytes the call reads and writes.
Post-process workloads: b1 and b32 of prob [101, 56, 4] (lane logits with points in two lanes), points for the 1280x720 `vis`.
The call is timed as above; the D2H copy of prob (90 496 B per frame) into pinned memory plus a synchronise is the median of
200 (probe_timing.d2h_sync_us)."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, d2h_sync_us, probe_main  # noqa: E402
from oracle import ufld as UO  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
NET_W, NET_H = UO.NET_W, UO.NET_H


def pre_workload(name, w, h, B, rng):
    frames = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).to(dev) for _ in range(B)]
    inp = torch.empty((B, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    floor = torch.empty(inp.numel(), dtype=torch.float32, device=dev)
    t = alternating({"call": lambda: P.ufld_preprocess(frames, out=inp), "floor": lambda: floor.fill_(1.0)})
    return {
        "workload": f"pre {name} b{B}", "batch": B,
        "pre_us": round(t["call"], 2), "pre_floor_us": round(t["floor"], 2), "pre_over_floor": round(t["call"] / t["floor"], 2),
        "pre_bytes_written": inp.numel() * 4, "pre_bytes_read": B * w * h * 3,
    }


def post_workload(B):
    prob = torch.from_numpy(np.stack([UO.lane_prob(seed=b, nan_cell=False) for b in range(B)])).to(dev)
    rows = torch.empty((B, 1 + 56 * 4 * 3), dtype=torch.float32, device=dev)
    sizes = [(1280, 720)] * B
    t = alternating({"call": lambda: P.ufld_postprocess(prob, sizes, out=rows)})
    d2h = d2h_sync_us(prob)
    return {
        "workload": f"post b{B}", "batch": B, "post_us": round(t["call"], 2), "d2h_bytes": prob.numel() * 4,
        "d2h_sync_us": round(d2h, 1), "post_over_d2h": round(t["call"] / d2h, 3),
        "points_per_frame": float(rows[:, 0].float().mean()),
    }


def main(outdir):
    rng = np.random.default_rng(0)
    res = []
    for B in (8, 32):
        for name, (w, h) in (("720p", (1280, 720)), ("1080p", (1920, 1080))):
            r = pre_workload(name, w, h, B, rng)
            print(r, flush=True)
            res.append(r)
    for B in (1, 32):
        r = post_workload(B)
        print(r, flush=True)
        res.append(r)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("ufld_probe", main)
