"""Timing of the Mask R-CNN post-process for frames of mixed sizes (trtx_rcnn_postprocess_frames_enqueue) against the
single-size entry (trtx_rcnn_postprocess_enqueue) and the write floor.

  python tools/rcnn_post_frames_probe.py OUTDIR      -> OUTDIR/rcnn_post_frames_probe.json (and the same JSON on stdout)

Workloads, b8 x D = 100 BatchedNms-like outputs with 14 x 14 masks, 20 kept per image, boxes log-uniform 32..256 px squares in
the network input:
  mixed   eight frame sizes, net 1067 x 800: one per-frame call against eight batch-1 calls of the single-size entry (what
          a caller had to do before), both captured in one graph;
  uniform eight frames of one size: the per-frame call against one call of the single-size entry.
Timing: 20 calls (or 20 groups of eight calls) captured in one CUDA graph, replayed 20 times between two events; each
variant is timed three times, alternating, and the median is reported.  The floor is a device fill (torch fill_) of the
canvas bytes the call writes, timed the same way in the same process.  Outputs of the compared variants are checked equal."""
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, graph_us, probe_main  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B, D, S, KEPT = 8, 100, 14, 20
MIXED = [(640, 480), (480, 640), (1280, 720), (1920, 1080), (1333, 750), (800, 800), (3000, 200), (64, 48)]


def inputs(seed, net_w, net_h):
    rng = np.random.default_rng(seed)
    s = np.exp(rng.uniform(np.log(32), np.log(256), (B, D)))
    x1, y1 = rng.uniform(0, net_w - s), rng.uniform(0, net_h - s)
    boxes = np.stack([x1, y1, x1 + s, y1 + s], -1).astype(np.float32)
    scores = np.where(np.arange(D)[None, :] < KEPT, 0.9, 0.3).astype(np.float32).repeat(B, 0)
    for b in range(B):
        rng.shuffle(scores[b])
    classes = rng.integers(0, 80, (B, D)).astype(np.float32)
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 2))).astype(np.float32)
    return [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]


def fill_floor_us(nbytes):
    fill = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    us = graph_us(lambda: fill.fill_(0))
    del fill
    return us


def mixed_workload():
    net_w, net_h = 1067, 800
    t = inputs(1, net_w, net_h)
    rows_f = torch.empty((B, 1 + D * 7), dtype=torch.float32, device=dev)
    canv_f = [torch.zeros((D, h, w), dtype=torch.uint8, device=dev) for w, h in MIXED]
    rows_s = torch.empty_like(rows_f)
    canv_s = [torch.zeros((1, D, h, w), dtype=torch.uint8, device=dev) for w, h in MIXED]

    def frames_call():
        P.rcnn_postprocess_frames(*t, frames=MIXED, net_w=net_w, net_h=net_h, rows=rows_f, canvases=canv_f)

    def eight_calls():
        for b, (w, h) in enumerate(MIXED):
            P.rcnn_postprocess(*(x[b:b + 1] for x in t), img_w=w, img_h=h, net_w=net_w, net_h=net_h,
                               out=(rows_s[b:b + 1], canv_s[b]))

    us = alternating({"frames_call": frames_call, "eight_single_calls": eight_calls})
    torch.cuda.synchronize()
    equal = torch.equal(rows_f, rows_s) and all(torch.equal(a, c[0]) for a, c in zip(canv_f, canv_s))
    counts = rows_f[:, 0].to(torch.int64).tolist()
    nbytes = sum(min(n, D) * w * h for n, (w, h) in zip(counts, MIXED))
    floor = fill_floor_us(nbytes)
    return {"name": "b8_mixed_8_sizes_kept20", "frames": MIXED, "net": [net_w, net_h], "canvases": sum(counts),
            "bytes_written": nbytes, "frames_call_us": round(us["frames_call"], 2),
            "eight_single_calls_us": round(us["eight_single_calls"], 2),
            "speedup": round(us["eight_single_calls"] / us["frames_call"], 3), "fill_floor_us": round(floor, 2),
            "frames_call_ratio_to_floor": round(us["frames_call"] / floor, 3), "outputs_equal": bool(equal)}


def uniform_workload(img_w, img_h, net_w, net_h):
    t = inputs(2, net_w, net_h)
    frames = [(img_w, img_h)] * B
    rows_f = torch.empty((B, 1 + D * 7), dtype=torch.float32, device=dev)
    canv_f = [torch.zeros((D, img_h, img_w), dtype=torch.uint8, device=dev) for _ in frames]
    rows_s = torch.empty_like(rows_f)
    canv_s = torch.zeros((B, D, img_h, img_w), dtype=torch.uint8, device=dev)

    def frames_call():
        P.rcnn_postprocess_frames(*t, frames=frames, net_w=net_w, net_h=net_h, rows=rows_f, canvases=canv_f)

    def single_call():
        P.rcnn_postprocess(*t, img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h, out=(rows_s, canv_s))

    us = alternating({"frames_call": frames_call, "single_size_call": single_call})
    torch.cuda.synchronize()
    equal = torch.equal(rows_f, rows_s) and all(torch.equal(canv_f[b], canv_s[b]) for b in range(B))
    n = int(rows_f[:, 0].sum().item())
    floor = fill_floor_us(n * img_w * img_h)
    return {"name": f"b8_{img_w}x{img_h}_kept20", "net": [net_w, net_h], "canvases": n, "bytes_written": n * img_w * img_h,
            "frames_call_us": round(us["frames_call"], 2), "single_size_call_us": round(us["single_size_call"], 2),
            "ratio": round(us["frames_call"] / us["single_size_call"], 3), "fill_floor_us": round(floor, 2),
            "outputs_equal": bool(equal)}


def main(outdir: Path):
    res = {"timing": "20 graph-captured calls x 20 replays between CUDA events, median of 3 alternating", "workloads": []}
    for w in (mixed_workload(), uniform_workload(640, 480, 1067, 800), uniform_workload(1920, 1080, 1333, 750)):
        res["workloads"].append(w)
        print(json.dumps(w), flush=True)
    return res


if __name__ == "__main__":
    probe_main("rcnn_post_frames_probe", main)
