"""The timing method the pre- and post-process probes share, so that a figure from one probe means what a figure from
another means.

  graph_us        n calls captured in one CUDA graph on a side stream, 3 warm replays, then `reps` replays between two CUDA
                  events; microseconds per call.
  alternating     the median over `rounds` of each function's graph_us, the functions timed in turn within each round.
  d2h_sync_us     a copy into pinned host memory + torch.cuda.synchronize(), host wall clock, median of `reps`.
  card            the device name and nvidia-smi's name, power limit, max and current SM clock.
  probe_main      `python tools/<name>.py OUTDIR`: runs the probe and writes OUTDIR/<name>.json."""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch


def graph_us(fn, n=20, reps=20):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(n):
                fn()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (n * reps) * 1e3


def alternating(fns: dict, rounds=3, **kw) -> dict:
    """Median over `rounds` of each fn's graph time, the fns timed in turn within each round."""
    t = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            t[k].append(graph_us(fn, **kw))
    return {k: float(np.median(v)) for k, v in t.items()}


def d2h_sync_us(t, reps=200):
    host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host.copy_(t, non_blocking=True)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def card() -> dict:
    """The card a figure was measured on; "unavailable" where nvidia-smi is missing or does not answer."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        q = []
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable"}


def probe_main(name, main):
    """`python tools/<name>.py OUTDIR`: the card, then main(OUTDIR)'s result, to OUTDIR/<name>.json; the card line last."""
    if len(sys.argv) != 2:
        sys.exit(f"usage: python tools/{name}.py OUTDIR")
    outdir = Path(sys.argv[1])
    outdir.mkdir(parents=True, exist_ok=True)
    res = {**card(), **main(outdir)}
    (outdir / f"{name}.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps({"card": res["card"], "nvidia_smi": res["nvidia_smi"]}))
