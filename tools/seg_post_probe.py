"""Timing of the YOLO segmentation post-process (trtx_yolo_seg_postprocess_enqueue: rows kernel + fused canvas kernel) against
the composition it replaces and against the write floor.

  python tools/seg_post_probe.py OUTDIR      -> OUTDIR/seg_post_probe.json (and the same JSON on stdout)

Each workload is b8 x 20 detections per image (compact NMS rows, 39 floats, coefficients at 7; boxes log-uniform 32..256 px
inside the letterboxed frame) at one frame size.  Timed, each as 20 launches captured in one CUDA graph and replayed between
two events:
  call         the new call (u8 canvases [20, h, w] per image);
  composition  trtx_process_mask_enqueue (fp32 640 x 640 masks) + one trtx_scale_mask_enqueue per image (fp32 h x w) + a
               torch threshold / crop to the same u8 canvases (the crop is a precomputed get_rect window mask);
  fill_floor   a device fill (torch fill_) of the canvas bytes."""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import graph_us, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B, K, R, OFF = 8, 20, 39, 7


def inputs(seed, img_w, img_h):
    rng = np.random.default_rng(seed)
    arr = (C.c_int * 4)()
    L.load().trtx_scale_mask_rect(640, 640, img_w, img_h, arr)
    x, y, w, h = list(arr)   # the frame inside the network input
    proto = rng.standard_normal((B, 32, 160, 160)).astype(np.float32)
    dets = np.zeros((B, 1 + K * R), np.float32)
    for b in range(B):
        dets[b, 0] = K
        rows = dets[b, 1:].reshape(K, R)
        s = np.exp(rng.uniform(np.log(32), np.log(256), K))
        x1, y1 = rng.uniform(x, x + w - s), rng.uniform(y, y + h - np.minimum(s, h - 1))
        rows[:, :4] = np.stack([x1, y1, x1 + s, y1 + s], -1)
        rows[:, 4], rows[:, 5] = 0.9, rng.integers(0, 80, K)
        rows[:, OFF:OFF + 32] = rng.standard_normal((K, 32)) * 0.6
    return proto, dets


def main(outdir: Path):
    res = {"timing": "20 graph-captured launches x 20 replays between CUDA events", "workloads": []}
    for img_w, img_h in ((1920, 1080), (1280, 720), (640, 480)):
        proto, dets = inputs(3, img_w, img_h)
        proto_d, dets_d = torch.from_numpy(proto).to(dev), torch.from_numpy(dets).to(dev)
        sizes = [(img_w, img_h)] * B
        rows = torch.empty((B, 1 + K * 6), dtype=torch.float32, device=dev)
        canv = [torch.zeros((K, img_h, img_w), dtype=torch.uint8, device=dev) for _ in range(B)]
        call = lambda: P.yolo_seg_postprocess(proto_d, dets_d, sizes, variant=L.YOLO_V8, max_rows=K, max_masks=K,
                                              rows_out=rows, canvases_out=canv)
        us = graph_us(call)
        # the composition: fp32 intermediates, one scale_mask per image, threshold + crop in torch
        masks = torch.empty((B, K, 640, 640), dtype=torch.float32, device=dev)
        S = [torch.empty((K, img_h, img_w), dtype=torch.float32, device=dev) for _ in range(B)]
        win = []
        for b in range(B):
            m = torch.zeros((K, img_h, img_w), dtype=torch.bool)
            for k in range(K):
                x, y, w, h = P.get_rect(img_w, img_h, dets[b, 1 + k * R:1 + k * R + 4])
                m[k, max(y, 0):max(min(y + h, img_h), 0), max(x, 0):max(min(x + w, img_w), 0)] = True
            win.append(m.to(dev))
        ref = [torch.empty((K, img_h, img_w), dtype=torch.uint8, device=dev) for _ in range(B)]

        def composition():
            P.process_mask(proto_d, dets_d, K, R, OFF, K, 640, 640, variant=L.YOLO_V8, out=masks)
            for b in range(B):
                P.scale_mask(masks[b], img_w, img_h, out=S[b])
                torch.logical_and(S[b] > 0.5, win[b], out=ref[b].view(torch.bool))
                ref[b].mul_(255)

        comp_us = graph_us(composition)
        call()
        composition()
        torch.cuda.synchronize()
        same = all(torch.equal(canv[b], ref[b]) for b in range(B))
        nbytes = B * K * img_w * img_h
        fill = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        floor_us = graph_us(lambda: fill.fill_(0))
        del fill, masks, S, ref, win
        w = {"img": [img_w, img_h], "batch": B, "masks_per_image": K, "canvas_bytes": nbytes, "call_us": round(us, 2),
             "call_GBps": round(nbytes / us / 1e3, 1), "composition_us": round(comp_us, 2),
             "speedup_vs_composition": round(comp_us / us, 2), "fill_floor_us": round(floor_us, 2),
             "ratio_to_floor": round(us / floor_us, 3), "canvases_equal_composition": same}
        res["workloads"].append(w)
        print(json.dumps(w), flush=True)
        del canv
    return res


if __name__ == "__main__":
    probe_main("seg_post_probe", main)
