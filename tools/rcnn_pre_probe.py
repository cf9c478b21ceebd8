"""Timing of the Mask R-CNN pre-process (trtx_rcnn_preprocess_enqueue) against the write floor, and of the two ways to feed the
engine input end to end.

  python tools/rcnn_pre_probe.py OUTDIR      -> OUTDIR/rcnn_pre_probe.json (and the same JSON on stdout)

Each workload is a batch of 8 random u8 BGR frames of one size.  The call is timed as 20 launches captured in one CUDA graph,
replayed 20 times between two events.  The floor is a plain device fill (torch fill_) of the bytes the call writes, timed the
same way in the same process.  End to end, per batch:
  device path: H2D copy of the u8 frames from pinned host memory + the call (graph-captured like the call);
  host path:   what rcnn.cpp:497-506 + :330 do, in one process: cv2.resize, the 128 canvas, astype(float32), then the H2D
               copy of the fp32 batch from pageable memory, timed with a host clock around a device synchronise."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B = 8


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


def host_path_us(frames, net_w, net_h, reps=5):
    """preprocessImg + the widening loop with cv2 / numpy, then the fp32 H2D copy (pageable, as from the std::vector)."""
    import cv2
    pads = [P.rcnn_letterbox_pads(f.shape[1], f.shape[0], net_w, net_h) for f in frames]
    data = np.empty((len(frames), net_h, net_w, 3), np.float32)
    dst = torch.empty(data.shape, dtype=torch.float32, device=dev)
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b, f in enumerate(frames):
            l, r, t, bt = pads[b]
            w, h = net_w - l - r, net_h - t - bt
            re = cv2.resize(f, (w, h), interpolation=cv2.INTER_LINEAR)
            out = np.full((net_h, net_w, 3), 128, np.uint8)
            out[t:t + h, l:l + w] = re
            data[b] = out.astype(np.float32)
        dst.copy_(torch.from_numpy(data))
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1e6)
    return best


def main(outdir: Path):
    outdir.mkdir(parents=True, exist_ok=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable",
           "timing": "20 graph-captured calls x 20 replays between CUDA events", "workloads": []}
    rng = np.random.default_rng(1)
    for name, img_w, img_h, net_w, net_h in (("b8_640x480_to_1067x800", 640, 480, 1067, 800),
                                             ("b8_1920x1080_to_1333x750", 1920, 1080, 1333, 750),
                                             ("b8_1920x1080_to_1067x800", 1920, 1080, 1067, 800)):
        frames = [rng.integers(0, 256, (img_h, img_w, 3), dtype=np.uint8) for _ in range(B)]
        pinned = torch.from_numpy(np.stack(frames)).pin_memory()
        d_frames = torch.empty(pinned.shape, dtype=torch.uint8, device=dev)
        d_frames.copy_(pinned)
        imgs = list(d_frames.unbind(0))
        out = torch.empty((B, net_h, net_w, 3), dtype=torch.float32, device=dev)
        us = graph_us(lambda: P.rcnn_preprocess(imgs, net_w, net_h, out=out))
        nbytes = out.numel() * 4
        fill = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        floor_us = graph_us(lambda: fill.fill_(128.0))
        del fill

        def device_path():
            d_frames.copy_(pinned, non_blocking=True)
            P.rcnn_preprocess(imgs, net_w, net_h, out=out)
        dev_us = graph_us(device_path, n=5, reps=20)
        host_us = host_path_us(frames, net_w, net_h)
        w = {"name": name, "img": [img_w, img_h], "net": [net_w, net_h], "bytes_written": nbytes,
             "bytes_read_u8": int(pinned.numel()), "us": round(us, 2), "GBps": round(nbytes / us / 1e3, 1),
             "fill_floor_us": round(floor_us, 2), "fill_GBps": round(nbytes / floor_us / 1e3, 1),
             "ratio_to_floor": round(us / floor_us, 3), "device_path_us_per_batch": round(dev_us, 1),
             "host_path_us_per_batch": round(host_us, 1)}
        res["workloads"].append(w)
        print(json.dumps(w), flush=True)
    (outdir / "rcnn_pre_probe.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps({"card": res["card"], "nvidia_smi": res["nvidia_smi"]}))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tools/rcnn_pre_probe.py OUTDIR")
    main(Path(sys.argv[1]))
