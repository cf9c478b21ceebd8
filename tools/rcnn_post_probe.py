"""Timing of the Mask R-CNN post-process (trtx_rcnn_postprocess_enqueue: rows kernel + paste kernel) against the write floor.

  python tools/rcnn_post_probe.py OUTDIR      -> OUTDIR/rcnn_post_probe.json (and the same JSON on stdout)

Each workload is b8 x D = 100 BatchedNms-like outputs with 14 x 14 masks; boxes are log-uniform 32..256 px squares in the
network input.  Timing: 20 launches captured in one CUDA graph, replayed between two events.  The write floor is a plain
device fill (torch fill_) of the same byte count, timed the same way in the same process.  The host path's time per batch
(cv2 per kept detection, one process, as rcnn.cpp:543-550 does it) is given for context and is a CPU number."""
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
B, D, S = 8, 100, 14


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


def inputs(seed, kept, net_w, net_h):
    rng = np.random.default_rng(seed)
    s = np.exp(rng.uniform(np.log(32), np.log(256), (B, D)))
    x1, y1 = rng.uniform(0, net_w - s), rng.uniform(0, net_h - s)
    boxes = np.stack([x1, y1, x1 + s, y1 + s], -1).astype(np.float32)
    scores = np.where(np.arange(D)[None, :] < kept, 0.9, 0.3).astype(np.float32).repeat(B, 0)
    for b in range(B):
        rng.shuffle(scores[b])
    classes = rng.integers(0, 80, (B, D)).astype(np.float32)
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 2))).astype(np.float32)
    return scores, boxes, classes, masks


def host_us_per_batch(scores, boxes, masks, img_w, img_h, net_w, net_h):
    """rcnn.cpp:516-550 on the host with cv2 (rescale, rectangle, resize, threshold, add into a zero canvas), one process."""
    import cv2
    pl, pr, pt, pb = P.rcnn_letterbox_pads(img_w, img_h, net_w, net_h)
    h_ratio = np.float32(img_h) / np.float32(net_h - (pt + pb))
    w_ratio = np.float32(img_w) / np.float32(net_w - (pl + pr))
    t0 = time.perf_counter()
    for b in range(B):
        for i in range(D):
            if not scores[b, i] > np.float32(0.6):
                continue
            x1, y1, x2, y2 = ((boxes[b, i] - np.float32([pl, pt, pl, pt])) * np.float32([w_ratio, h_ratio, w_ratio, h_ratio]))
            p0 = (int(max(np.floor(x1) - 1, 0)), int(max(np.floor(y1) - 1, 0)))
            p1 = (int(min(np.ceil(x2) + 1, img_w)), int(min(np.ceil(y2) + 1, img_h)))
            x, y, w, h = min(p0[0], p1[0]), min(p0[1], p1[1]), abs(p1[0] - p0[0]), abs(p1[1] - p0[1])
            part = cv2.resize(masks[b, i], (w, h))
            cur = np.zeros((img_h, img_w), np.uint8)
            _, part = cv2.threshold(part, 0.5, 255, cv2.THRESH_BINARY)
            cur[y:y + h, x:x + w] = cv2.add(cur[y:y + h, x:x + w], part, dtype=cv2.CV_8U)
    return (time.perf_counter() - t0) * 1e6


def main(outdir: Path):
    outdir.mkdir(parents=True, exist_ok=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    res = {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable",
           "timing": "20 graph-captured launches x 20 replays between CUDA events", "workloads": []}
    for name, img_w, img_h, net_w, net_h, kept, with_masks in (
            ("b8_640x480_kept20", 640, 480, 1067, 800, 20, True),
            ("b8_640x480_kept100", 640, 480, 1067, 800, 100, True),
            ("b8_1920x1080_kept20", 1920, 1080, 1333, 750, 20, True),
            ("b8_640x480_rows_only", 640, 480, 1067, 800, 20, False)):
        sc, bx, cl, mk = inputs(1, kept, net_w, net_h)
        t = [torch.from_numpy(a).to(dev) for a in (sc, bx, cl, mk)]
        rows = torch.empty((B, 1 + D * 7), dtype=torch.float32, device=dev)
        kw = dict(img_w=img_w, img_h=img_h, net_w=net_w, net_h=net_h)
        w = {"name": name, "img": [img_w, img_h], "net": [net_w, net_h], "kept_per_image": kept}
        if with_masks:
            canv = torch.zeros((B, D, img_h, img_w), dtype=torch.uint8, device=dev)
            us = graph_us(lambda: P.rcnn_postprocess(*t, **kw, out=(rows, canv)))
            P.rcnn_postprocess(*t, **kw, out=(rows, canv))
            torch.cuda.synchronize()
            n = int(rows[:, 0].sum().item())
            nbytes = n * img_w * img_h
            fill = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            floor_us = graph_us(lambda: fill.fill_(0))
            del fill
            host = host_us_per_batch(sc, bx, mk, img_w, img_h, net_w, net_h)
            w.update({"canvases": n, "bytes_written": nbytes, "us": round(us, 2), "GBps": round(nbytes / us / 1e3, 1),
                      "fill_floor_us": round(floor_us, 2), "fill_GBps": round(nbytes / floor_us / 1e3, 1),
                      "ratio_to_floor": round(us / floor_us, 3), "cpu_host_path_us_per_batch": round(host, 1)})
            del canv
        else:
            us = graph_us(lambda: P.rcnn_postprocess(*t[:3], **kw, out=(rows, None)))
            w.update({"us": round(us, 2), "bytes_written": rows.numel() * 4})
        res["workloads"].append(w)
        print(json.dumps(w), flush=True)
    # the call is two launches; the rows kernel alone is the rows-only workload, the rest is the paste
    rows_us = res["workloads"][-1]["us"]
    for w in res["workloads"][:-1]:
        w["paste_us_est"] = round(w["us"] - rows_us, 2)
        w["paste_ratio_to_floor_est"] = round(w["paste_us_est"] / w["fill_floor_us"], 3)
    (outdir / "rcnn_post_probe.json").write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps({"card": res["card"], "nvidia_smi": res["nvidia_smi"]}))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tools/rcnn_post_probe.py OUTDIR")
    main(Path(sys.argv[1]))
