"""Sweep the (class slices, rows in flight) variants of the YoloLayer scan at b32, fp32 and fp16, dense / background heads.
Timing: 20 launches captured in ONE CUDA graph, replayed 10 times between two events (stream launches from Python are
quantised to ~2 us ticks of the launch path and cannot separate the variants; the step runs the kernel from a graph too).
Run on the GPU box:  python tools/sweep_scan.py"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402
from tensorrtx_b200 import synth  # noqa: E402

dev = torch.device("cuda", 0)
B, R = 32, 4


def graph_us(fn, n=20, reps=10):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn(0)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(n):
                fn(i)
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


for data, nobj in (("dense", 64), ("background", 0)):
    sets = [[torch.from_numpy(h).to(dev) for h in synth.yolov8_heads(B, seed=i, n_obj=nobj)] for i in range(R)]
    sets16 = [[h.half() for h in s] for s in sets]
    nbytes = sum(h.numel() * 4 for h in sets[0])
    for dt, ss, nb in ((L.F32, sets, nbytes), (L.F16, sets16, nbytes // 2)):
        plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32), in_dtype=dt)
        fused = P.FusedYoloDecodeNms(plug, B, device=dev)
        for slices, unroll in [(1, 8), (1, 16), (2, 4), (2, 5), (2, 8), (2, 10), (2, 20), (4, 4), (4, 5), (4, 10), (4, 20), (8, 5), (8, 10)]:
            for box in ((2, 3) if slices == 2 and unroll == 5 else (0,)):
                plug.tune(slices=slices, rows=unroll, box=box)
                us = graph_us(lambda i: fused.enqueue_scan(B, ss[i % R]))
                print(json.dumps({"data": data, "dtype": "f32" if dt == L.F32 else "f16", "slices": slices, "rows": unroll, "box": box,
                                  "us": round(us, 2), "GBps": round(nb / us / 1e3, 1)}), flush=True)
    del sets, sets16
# NMS alone, fused, letterbox (graph timing as well)
sets = [[torch.from_numpy(h).to(dev) for h in synth.yolov8_heads(B, seed=i)] for i in range(R)]
plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
fused = P.FusedYoloDecodeNms(plug, B, device=dev)
fused.enqueue_scan(B, sets[0])
print(json.dumps({"kernel": "nms", "us": round(graph_us(lambda i: fused.enqueue_nms(B, sets[0])), 2)}), flush=True)
print(json.dumps({"kernel": "scan+nms", "us": round(graph_us(lambda i: fused.enqueue(B, sets[i % R])), 2)}), flush=True)
for odt in (torch.float32, torch.float16):
    frames = [torch.from_numpy(synth.frames(B, seed=i)).to(dev) for i in range(R)]
    dst = torch.empty((B, 3, 640, 640), dtype=odt, device=dev)
    plans = [P.PreprocessPlan(list(f.unbind(0)), dst, 640, 640) for f in frames]
    us = graph_us(lambda i: plans[i % R].enqueue())
    nb = B * (640 * 640 * 3 + 3 * 640 * 640 * dst.element_size())
    print(json.dumps({"kernel": "letterbox", "out": str(odt), "us": round(us, 2), "GBps": round(nb / us / 1e3, 1)}), flush=True)
