"""Timing of the bilinear letterbox pre-process (trtx_linear_preprocess_enqueue) and of the truncating get_rect rows
(trtx_yolo_seg_postprocess_enqueue's rows-only mode with TRTX_YOLO_V3).

  python tools/linear_pre_probe.py OUTDIR      -> OUTDIR/linear_pre_probe.json (and the card line on stdout)

Workloads: b16 of 1920x1080 frames into yolov3's 608x608 input (TRTX_LINEAR_YOLOV3) and RetinaFace's 640x480 one
(TRTX_LINEAR_RETINA), b16 of 1920x1080 frames into yolov3-spp's 608x352 canvas (TRTX_LINEAR_YOLOV3_SPP), and the rows of b32
frames of 1000 compact NMS rows each.  Every figure is probe_timing.alternating: 20 launches in one CUDA graph, replayed 20
times between two events, the calls alternating over 3 rounds, medians in microseconds per call.  GB/s counts the u8 frame bytes
read once and the fp32 bytes written (the rows: the 7-float rows read and the 6-float rows written)."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)


def main(outdir):
    rng = np.random.default_rng(0)
    frames = [torch.from_numpy(rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)).to(dev) for _ in range(16)]
    read = 16 * 1920 * 1080 * 3
    spp_w, spp_h = P.yolov3spp_letterbox(1920, 1080)[0]
    cases = {"yolov3 608x608": (L.LINEAR_YOLOV3, 608, 608), "retinaface 640x480": (L.LINEAR_RETINA, 640, 480),
             f"yolov3-spp {spp_w}x{spp_h}": (L.LINEAR_YOLOV3_SPP, spp_w, spp_h)}
    outs = {k: torch.empty((16, 3, h, w), dtype=torch.float32, device=dev) for k, (_, w, h) in cases.items()}
    fns = {k: (lambda k=k, v=v, w=w, h=h: P.linear_preprocess(frames, v, out=outs[k], net_w=w, net_h=h))
           for k, (v, w, h) in cases.items()}
    # the rows: b32 frames of mixed sizes, 1000 rows of 7 floats each
    B, K = 32, 1000
    dets = np.zeros((B, 1 + K * 7), np.float32)
    for b in range(B):
        r = np.concatenate([rng.uniform(0, 608, (K, 2)), rng.uniform(1, 300, (K, 2)), rng.uniform(0, 1, (K, 1)),
                            rng.integers(0, 80, (K, 1)), np.ones((K, 1))], 1)
        dets[b, 0], dets[b, 1:] = K, r.reshape(-1)
    dets_d = torch.from_numpy(dets).to(dev)
    sizes = [(1920, 1080), (1280, 720), (640, 480), (720, 1280)] * (B // 4)
    rows = torch.empty((B, 1 + K * 6), dtype=torch.float32, device=dev)
    fns["rows b32"] = lambda: P.yolo_seg_postprocess(None, dets_d, sizes, variant=L.YOLO_V3, max_rows=K, row_floats=7,
                                                     max_masks=1, net_w=608, net_h=608, masks=False, rows_out=rows)
    t = alternating(fns)
    res = []
    for k, (_, w, h) in cases.items():
        nbytes = read + 16 * 3 * w * h * 4
        res.append({"workload": f"{k} b16 1920x1080", "us": round(t[k], 2), "bytes": nbytes,
                    "GB_per_s": round(nbytes / t[k] / 1e3, 1)})
    nbytes = dets.nbytes + rows.numel() * 4
    res.append({"workload": "rows b32 x 1000", "us": round(t["rows b32"], 2), "bytes": nbytes,
                "GB_per_s": round(nbytes / t["rows b32"] / 1e3, 1)})
    for r in res:
        print(r, flush=True)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("linear_pre_probe", main)
