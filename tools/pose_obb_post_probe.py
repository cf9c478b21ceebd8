"""Timing of the pose / oriented-box post-process (trtx_yolo_pose_obb_postprocess_enqueue) against what any host path pays
before its first row: the D2H copy of the same compact NMS rows and a synchronisation.

  python tools/pose_obb_post_probe.py OUTDIR      -> OUTDIR/pose_obb_post_probe.json (and the same JSON on stdout)

Workloads: b32 frames, 20 or 100 kept rows per frame (compact NMS rows: pose 58 floats with keypoints at 7, OBB 8 floats with
the angle at 7), all frames 1920 x 1080 or a mix of sizes.  Timed:
  call_us       the call, 20 launches captured in one CUDA graph, 20 replays between two CUDA events, per call;
  d2h_sync_us   torch copy of the compact rows into pinned host memory + torch.cuda.synchronize(), host wall clock, median
                of 200 (the least a host post-process pays before it starts);
  ref_host_us   where oracle/_ref/libref_pose_obb_host.so exists: the reference's compiled draw_bbox_keypoints_line /
                draw_bbox_obb (yolov8, net 640) over the 32 frames' rows on one host core, drawing calls recording only,
                median of 5.  Not a device number: the host's own clock and CPU.
The call is latency-bound (a few hundred KB at most), so the figures are microseconds, not a bandwidth share."""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import pose_obb as PO  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B = 32
MIXED = [(1920, 1080), (1280, 720), (640, 480), (1080, 1920), (3840, 2160), (333, 1001), (720, 1280), (1024, 1024)]


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


def inputs(task, K, seed=3):
    rng = np.random.default_rng(seed)
    R = 58 if task == L.TASK_POSE else 8
    d = np.zeros((B, 1 + K * R), np.float32)
    for b in range(B):
        d[b, 0] = K
        r = d[b, 1:].reshape(K, R)
        s = np.exp(rng.uniform(np.log(32), np.log(256), K))
        x, y = rng.uniform(0, 640 - s), rng.uniform(80, 560 - np.minimum(s, 400))
        if task == L.TASK_POSE:
            r[:, :4] = np.stack([x, y, x + s, y + s], -1)
            r[:, 7:] = rng.uniform(0, 640, (K, 51))
            r[:, 9::3] = rng.uniform(0, 1, (K, 17))
        else:
            r[:, :4] = np.stack([x + s / 2, y + s / 2, s, s * rng.uniform(0.3, 1.5, K)], -1)
            r[:, 7] = rng.uniform(-np.pi / 4, 3 * np.pi / 4, K)
        r[:, 4], r[:, 5], r[:, 6] = 0.9, 0, 1
    return d, R


def d2h_us(dets_d):
    host = torch.empty(dets_d.shape, dtype=torch.float32, pin_memory=True)
    ts = []
    for _ in range(200):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host.copy_(dets_d, non_blocking=True)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def ref_us(task, dets, R, K, sizes):
    if PO.load_ref() is None:
        return None
    rows = dets[:, 1:].reshape(B, K, R)
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        for b, (w, h) in enumerate(sizes):
            if task == L.TASK_POSE:
                PO.ref_draw_bbox_keypoints_line("v8", w, h, rows[b, :, :4], rows[b, :, 7:58])
            else:
                PO.ref_draw_bbox_obb("v8", w, h, np.concatenate([rows[b, :, :4], rows[b, :, 7:8]], 1))
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def main(outdir: Path):
    outdir.mkdir(parents=True, exist_ok=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable",
           "timing": "call: 20 graph-captured launches x 20 replays between CUDA events; d2h: median of 200 host-timed",
           "workloads": []}
    for task, name in ((L.TASK_POSE, "pose"), (L.TASK_OBB, "obb")):
        for K in (20, 100):
            dets, R = inputs(task, K)
            dets_d = torch.from_numpy(dets).to(dev)
            Fo = 57 if task == L.TASK_POSE else 10
            rows = torch.empty((B, 1 + K * Fo), dtype=torch.float32, device=dev)
            for label, sizes in (("1080p", [(1920, 1080)] * B), ("mixed", [MIXED[b % len(MIXED)] for b in range(B)])):
                us = graph_us(lambda: P.yolo_pose_obb_postprocess(dets_d, sizes, task=task, max_rows=K, row_floats=R,
                                                                   rows_out=rows))
                w = {"task": name, "frames": label, "batch": B, "rows_per_frame": K, "in_bytes": dets.nbytes,
                     "out_bytes": rows.numel() * 4, "call_us": round(us, 2), "d2h_sync_us": round(d2h_us(dets_d), 2)}
                r = ref_us(task, dets, R, K, sizes)
                if r is not None:
                    w["ref_host_us"] = round(r, 1)
                res["workloads"].append(w)
                print(json.dumps(w), flush=True)
    (outdir / "pose_obb_post_probe.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps({"card": res["card"], "nvidia_smi": res["nvidia_smi"]}))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tools/pose_obb_post_probe.py OUTDIR")
    main(Path(sys.argv[1]))
