"""Time the YOLOv8 scan's launch shapes where it runs: inside the benchmark step, next to the letterbox.

The step is bench.py's graph of 4 consecutive steps as two concurrent chains: chain A = the 4 letterbox launches, chain B
(high priority) = the 4 scan -> NMS launches, 4 rotating input sets.  For every candidate (class slices, rows in flight)
this captures that graph, then times the candidates in alternation (`--rounds` rounds of `--replays` replays each, the
median per step is reported), and the scan alone (20 launches in one graph).  0 in a candidate field = the library default.
With tools/lb_ceiling built next to this file, its byte-stream floors (stream c = the step's floor) are run in the same call.
`--trace` also records a few replays of the first candidate's step graph with torch.profiler and reports how long the
letterbox and the scan kernels ran at the same time, with every kernel's span.

    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/lb_ceiling tools/lb_ceiling.cu   (optional, first)
    python tools/step_sweep.py OUTDIR [--head-dtype f16] [--cands 0:0,4:10,...] [--trace]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import card  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import synth  # noqa: E402
from tensorrtx_b200.pipeline import DetectionPipeline  # noqa: E402

NET, NC, STRIDES, MAX_OUT, B, R = 640, 80, (8, 16, 32), 1000, 32, 4


def tune_all(pipes, cand) -> None:
    slices, rows = cand
    for p in pipes:
        p.plugin.tune(slices=slices, rows=rows)


def step_graph(pipes, heads, dev):
    """bench.py make_group(0, 4): chain B = scan -> NMS of each step on a high-priority stream, chain A = the letterboxes."""
    chain_b = torch.cuda.Stream(dev, priority=-1)

    def f():
        cur = torch.cuda.current_stream(dev)
        chain_b.wait_stream(cur)
        with torch.cuda.stream(chain_b):
            for j in range(R):
                pipes[j].decode_nms_gather(heads[j], None)
        for j in range(R):
            pipes[j].pre.enqueue()
        cur.wait_stream(chain_b)
    return pipes[0].capture(f)


def scan_graph(pipes, heads):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(20):
            pipes[0].fused.enqueue_scan(B, heads[i % R])
    return g


def time_graph(g, replays: int) -> float:
    """ms per replay"""
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / replays


def overlap_report(trace_file: Path) -> dict:
    """Kernel spans of the trace: busy time of each kernel family and the time letterbox and scan kernels ran together."""
    ev = json.loads(trace_file.read_text())["traceEvents"]
    spans = {"scan": [], "letterbox": [], "nms": []}
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        n = e["name"]
        k = "scan" if "scan_kernel" in n else ("letterbox" if "letterbox" in n else ("nms" if "nms_kernel" in n else None))
        if k:
            spans[k].append((float(e["ts"]), float(e["ts"]) + float(e["dur"])))

    def merged(s):
        out = []
        for a, b in sorted(s):
            if out and a <= out[-1][1]:
                out[-1][1] = max(out[-1][1], b)
            else:
                out.append([a, b])
        return out

    def inter(x, y):
        t, i, j = 0.0, 0, 0
        while i < len(x) and j < len(y):
            t += max(0.0, min(x[i][1], y[j][1]) - max(x[i][0], y[j][0]))
            if x[i][1] < y[j][1]:
                i += 1
            else:
                j += 1
        return t
    m = {k: merged(v) for k, v in spans.items()}
    allk = merged(spans["scan"] + spans["letterbox"] + spans["nms"])
    return {"launches": {k: len(v) for k, v in spans.items()},
            "busy_us": {k: round(sum(b - a for a, b in v), 1) for k, v in m.items()},
            "scan_with_letterbox_us": round(inter(m["scan"], m["letterbox"]), 1),
            "nms_with_letterbox_us": round(inter(m["nms"], m["letterbox"]), 1),
            "span_us": round(allk[-1][1] - allk[0][0], 1) if allk else 0.0,
            "scan_spans_us": [[round(a - allk[0][0], 1), round(b - allk[0][0], 1)] for a, b in spans["scan"]],
            "letterbox_spans_us": [[round(a - allk[0][0], 1), round(b - allk[0][0], 1)] for a, b in spans["letterbox"]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--head-dtype", default="f32", choices=["f32", "f16"])
    ap.add_argument("--cands", default="0:0", help="comma-separated slices:rows, 0 = default")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--replays", type=int, default=500)
    ap.add_argument("--trace", action="store_true")
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    log = open(out / f"step_sweep_{args.head_dtype}.jsonl", "w")

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        log.write(line + "\n")
        log.flush()
    emit({**card(), "head_dtype": args.head_dtype})
    ceiling = ROOT / "tools" / "lb_ceiling"
    if ceiling.exists():
        r = subprocess.run([str(ceiling)], capture_output=True, text=True, timeout=300)
        for line in r.stdout.splitlines():
            if line.startswith("{") and ("a_expand" in line or "b_read" in line or "c_a_parallel" in line):
                emit({"floor": json.loads(line)})

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    hd = L.F32 if args.head_dtype == "f32" else L.F16
    tdt = torch.float32 if hd == L.F32 else torch.float16
    pipes, heads = [], []
    for i in range(R):
        p = DetectionPipeline(B, NET, NET, NET, NET, NC, STRIDES, MAX_OUT, 0.5, 0.45, dev, head_dtype=hd)
        p.frames_dev.copy_(torch.from_numpy(synth.frames(B, seed=77 + i, h=NET, w=NET)))
        pipes.append(p)
        heads.append([torch.from_numpy(h).to(dev).to(tdt).contiguous()
                      for h in synth.yolov8_heads(B, seed=i, nc=NC, net_w=NET, net_h=NET, strides=STRIDES)])
    cands = [tuple(int(x) for x in c.split(":")) for c in args.cands.split(",")]
    st = torch.cuda.Stream(dev)
    with torch.cuda.stream(st):
        steps, scans = {}, {}
        for c in cands:
            tune_all(pipes, c)
            steps[c] = step_graph(pipes, heads, dev)
            scans[c] = scan_graph(pipes, heads)
        step_us = {c: [] for c in cands}
        scan_us = {c: [] for c in cands}
        for _ in range(args.rounds):
            for c in cands:
                step_us[c].append(time_graph(steps[c], args.replays) / R * 1e3)
                scan_us[c].append(time_graph(scans[c], 10) / 20 * 1e3)
        for c in cands:
            emit({"slices": c[0], "rows": c[1], "step_us": round(statistics.median(step_us[c]), 2),
                  "step_us_all": [round(x, 2) for x in step_us[c]], "scan_alone_us": round(statistics.median(scan_us[c]), 2)})
        if args.trace:
            from torch.profiler import ProfilerActivity, profile
            g = steps[cands[0]]
            time_graph(g, 20)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    g.replay()
                torch.cuda.synchronize()
            tf = out / f"step_{args.head_dtype}.pt.trace.json"
            prof.export_chrome_trace(str(tf))
            emit({"trace": tf.name, "candidate": list(cands[0]), **overlap_report(tf)})
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
