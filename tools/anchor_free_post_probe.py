"""Timing of yolov9's NMS on converted boxes (TRTX_BOX_V9) and of yolov10's top-k rows (trtx_yolo_topk_postprocess_enqueue).

  python tools/anchor_free_post_probe.py OUTDIR      -> OUTDIR/anchor_free_post_probe.json (and the card line on stdout)

Workloads: yolov9's fused decode + NMS (YoloLayerPluginV9, 80 classes, maxOut 2000, conf 0.1, IoU 0.45) at b32 640x640 on
seeded heads (tensorrtx_b200/synth.py), once with TRTX_BOX_V9 and once with TRTX_BOX_CXCYWH on the same heads, to show what the
per-row conversion at load costs; and the top-k rows of b32 frames of mixed sizes with 1000 plugin rows of 6 floats each
(about half above kConfThresh 0.5).  Every figure is probe_timing.alternating: 20 launches in one CUDA graph, replayed 20
times between two events, the calls alternating over 3 rounds, medians in microseconds per call."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402
from tensorrtx_b200 import synth  # noqa: E402

dev = torch.device("cuda", 0)


def main(outdir):
    B = 32
    heads = [torch.from_numpy(h).to(dev) for h in synth.yolov8_heads(B, seed=5, nc=80)]
    plug = P.YoloLayerPluginV9(80, 640, 640, 2000, False)
    fused = {f: P.FusedYoloDecodeNms(plug, B, 0.1, 0.45, box_format=f, device=dev) for f in (L.BOX_V9, L.BOX_CXCYWH)}
    fns = {"v9 fused b32 BOX_V9": lambda: fused[L.BOX_V9].enqueue(B, heads),
           "v9 fused b32 BOX_CXCYWH": lambda: fused[L.BOX_CXCYWH].enqueue(B, heads)}
    kept = {k: fused[f].enqueue(B, heads)[0][:, 0].sum().item() for k, f in zip(fns, (L.BOX_V9, L.BOX_CXCYWH))}
    rng = np.random.default_rng(0)
    K = 1000
    dets = np.zeros((B, 1 + K * 6), np.float32)
    for b in range(B):
        xy = rng.uniform(-20, 640, (K, 2))
        r = np.concatenate([xy, xy + rng.uniform(1, 300, (K, 2)), rng.uniform(0, 1, (K, 1)), rng.integers(0, 80, (K, 1))], 1)
        dets[b, 0], dets[b, 1:] = K, r.reshape(-1)
    dets_d = torch.from_numpy(dets).to(dev)
    sizes = [(1920, 1080), (1280, 720), (640, 480), (720, 1280)] * (B // 4)
    rows = torch.empty((B, 1 + K * 6), dtype=torch.float32, device=dev)
    fns["v10 topk rows b32 x 1000"] = lambda: P.yolo_topk_postprocess(dets_d, sizes, max_rows=K, rows_out=rows)
    t = alternating(fns)
    res = [{"workload": k, "us": round(v, 2)} for k, v in t.items()]
    for r in res:
        if r["workload"] in kept:
            r["rows_kept_b32"] = int(kept[r["workload"]])
    nbytes = dets.nbytes + rows.numel() * 4
    res[-1].update(bytes=nbytes, GB_per_s=round(nbytes / t["v10 topk rows b32 x 1000"] / 1e3, 1))
    for r in res:
        print(r, flush=True)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("anchor_free_post_probe", main)
