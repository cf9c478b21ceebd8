"""Letterbox kernel timing at b32 into 640x640 for four source sizes (three unit-scale, one resampled) and both output types."""
import json, sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tensorrtx_b200 import _lib as L, plugins as P, synth
dev = torch.device("cuda", 0)
lib = L.load()
B, R, K = 32, 4, 200
for (h, w) in ((640, 640), (480, 640), (640, 480), (1080, 1920)):
    frames = [torch.from_numpy(synth.frames(B, seed=i, h=h, w=w)).to(dev) for i in range(R if h <= 640 else 2)]
    for odt in (torch.float32, torch.float16):
        dst = torch.empty((B, 3, 640, 640), dtype=odt, device=dev)
        plans = [P.PreprocessPlan(list(f.unbind(0)), dst, 640, 640) for f in frames]
        for i in range(10):
            plans[i % len(plans)].enqueue()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(K):
            plans[i % len(plans)].enqueue()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / K * 1e3
        print(json.dumps({"lib": L.LIB_PATH.name, "src": f"{w}x{h}", "out": str(odt), "us": round(us, 2)}), flush=True)
