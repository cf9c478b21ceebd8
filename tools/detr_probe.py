"""Timing of the DETR pre-process (trtx_detr_preprocess_enqueue) and post-process (trtx_detr_postprocess_enqueue) against the
write floor, against the bare copies they remove and against the host code they replace.

  python tools/detr_probe.py OUTDIR      -> OUTDIR/detr_probe.json (and the card line on stdout)

Pre-process workloads: b8 of 1920x1080, of 1280x720 and of 8 mixed sizes, and b32 of 1920x1080, into DETR's 1066x800 input
(10.2 MB of fp32 per frame).  The call is timed as 20 launches captured in one CUDA graph, replayed 20 times between two events;
its floor is a plain device fill (torch fill_) of the bytes it writes, timed the same way; call and floor alternate over 3
rounds and the medians are reported.  End to end, host clock around a device synchronise, best of 3:
  host path:   per frame cv2 cvtColor, resize, astype * (1 / 255), subtract, divide, the plane copy into one pageable fp32
               batch, then its H2D copy (detr/common.hpp:81-89, detr/detr.cpp:754-767, :640);
  device path: the H2D copy of the u8 frames from pinned memory, then the call.
Post-process workloads: b8 and b32 of 100 queries x 92 classes, 12 planted objects per frame, frames of 1920x1080.  The call
is timed as above; the bare D2H copy of the scores and boxes into pinned memory plus a synchronise is the median of 200; the
host loop (detr/detr.cpp:777-806) is the oracle's line-by-line C restatement, compiled at -O2, over every frame, best of 5."""
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, probe_main  # noqa: E402
from oracle import detr as DO  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
NET_W, NET_H, Q, NC = 1066, 800, 100, 92
MEAN, STD = (0.485, 0.456, 0.406, 0.0), (0.229, 0.224, 0.225, 0.0)
MIXED = [(1920, 1080), (1280, 720), (640, 480), (3840, 2160), (1080, 1920), (800, 600), (1024, 576), (427, 240)]


def _best_us(fn, reps):
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1e6)
    return best


def host_pre_us(frames_h, reps=3):
    import cv2
    data = np.empty((len(frames_h), 3, NET_H, NET_W), np.float32)  # pageable, as the driver's std::vector<float>
    dst = torch.empty(data.shape, dtype=torch.float32, device=dev)

    def run():
        for b, f in enumerate(frames_h):
            t = cv2.resize(cv2.cvtColor(f, cv2.COLOR_BGR2RGB), (NET_W, NET_H)).astype(np.float32) * np.float32(1 / 255.0)
            t = cv2.divide(cv2.subtract(t, MEAN), STD)
            data[b] = t.transpose(2, 0, 1)
        dst.copy_(torch.from_numpy(data))
    return _best_us(run, reps)


def device_pre_us(frames_h, reps=3):
    pinned = [torch.from_numpy(f).pin_memory() for f in frames_h]
    frames = [torch.empty(f.shape, dtype=torch.uint8, device=dev) for f in frames_h]
    inp = torch.empty((len(frames_h), 3, NET_H, NET_W), dtype=torch.float32, device=dev)

    def run():
        for d, h in zip(frames, pinned):
            d.copy_(h, non_blocking=True)
        P.detr_preprocess(frames, out=inp)
    run()
    return _best_us(run, reps)


def pre_workload(name, sizes, rng):
    B = len(sizes)
    frames_h = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sizes]
    frames = [torch.from_numpy(f).to(dev) for f in frames_h]
    inp = torch.empty((B, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    floor = torch.empty(inp.numel(), dtype=torch.float32, device=dev)
    t = alternating({"call": lambda: P.detr_preprocess(frames, out=inp), "floor": lambda: floor.fill_(1.0)})
    hp, dp = host_pre_us(frames_h), device_pre_us(frames_h)
    return {
        "workload": f"pre {name} b{B}", "batch": B,
        "pre_us": round(t["call"], 2), "pre_floor_us": round(t["floor"], 2), "pre_over_floor": round(t["call"] / t["floor"], 2),
        "pre_bytes_written": inp.numel() * 4,
        "host_path_us": round(hp, 1), "device_path_us": round(dp, 1), "path_speedup": round(hp / dp, 1),
    }


def _outputs(B, rng):
    logits = rng.normal(0, 1, (B, Q, NC)).astype(np.float32)
    logits[:, :, NC - 1] += 3.0
    for b in range(B):
        qs = rng.choice(Q, 12, replace=False)
        logits[b, qs, rng.integers(0, NC - 1, 12)] += 8.0
    e = np.exp(logits - logits.max(-1, keepdims=True))
    boxes = (1 / (1 + np.exp(-rng.normal(0, 1.5, (B, Q, 4))))).astype(np.float32)
    return (e / e.sum(-1, keepdims=True)).astype(np.float32), boxes


def post_workload(B, rng):
    s_np, b_np = _outputs(B, rng)
    scores, boxes = torch.from_numpy(s_np).to(dev), torch.from_numpy(b_np).to(dev)
    sizes = [(1920, 1080)] * B
    rows = torch.empty((B, 1 + Q * 6), dtype=torch.float32, device=dev)
    t = alternating({"call": lambda: P.detr_postprocess(scores, boxes, sizes, out=rows)})
    hs, hb = torch.empty(scores.shape, pin_memory=True), torch.empty(boxes.shape, pin_memory=True)
    d2h = []
    for _ in range(200):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hs.copy_(scores, non_blocking=True)
        hb.copy_(boxes, non_blocking=True)
        torch.cuda.synchronize()
        d2h.append((time.perf_counter() - t0) * 1e6)
    d2h_us = float(np.median(d2h))
    s_h, b_h = hs.numpy(), hb.numpy()
    loop_us = _best_us(lambda: [DO.postprocess(s_h[b], b_h[b], 1920, 1080) for b in range(B)], 5)
    return {
        "workload": f"post b{B}", "batch": B,
        "post_us": round(t["call"], 2), "d2h_sync_us": round(d2h_us, 1), "host_loop_us": round(loop_us, 1),
        "host_path_us": round(d2h_us + loop_us, 1), "path_speedup": round((d2h_us + loop_us) / t["call"], 1),
        "post_over_d2h": round(t["call"] / d2h_us, 3), "kept_per_frame": float(rows[:, 0].float().mean()),
    }


def main(outdir):
    rng = np.random.default_rng(0)
    res = []
    for name, sizes in (("1080p", [(1920, 1080)] * 8), ("720p", [(1280, 720)] * 8), ("mixed", MIXED),
                        ("1080p", [(1920, 1080)] * 32)):
        r = pre_workload(name, sizes, rng)
        print(r, flush=True)
        res.append(r)
    for B in (8, 32):
        r = post_workload(B, rng)
        print(r, flush=True)
        res.append(r)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("detr_probe", main)
