"""Timing of the Mask R-CNN instance outlines (trtx_rcnn_contours_enqueue) against the post-process call that made the
canvases and against the host path the call replaces.

  python tools/rcnn_contours_probe.py OUTDIR      -> OUTDIR/rcnn_contours_probe.json (and the same JSON on stdout)

Workloads, b8 x D = 100 BatchedNms-like outputs with 14 x 14 masks, boxes log-uniform 32..256 px squares in the network
input (the rcnn probes' inputs): 20 kept per image at 640 x 480 and at 1920 x 1080, all 100 kept at 640 x 480, and the batch
of eight mixed sizes with 20 kept.
Device timings: 20 calls captured in one CUDA graph, replayed 20 times between two events; the contour call and the
post-process call (trtx_rcnn_postprocess_frames_enqueue) are timed in turn, three rounds, median reported.
Host path: the D2H copy of the kept canvases to pinned memory plus a synchronize, then cv2.findContours(RETR_EXTERNAL,
CHAIN_APPROX_NONE) per kept canvas on one host thread; median of three.
Every canvas's counts, lengths and points are checked against the CPU oracle (oracle_find_contours_external)."""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import contours as CO  # noqa: E402
from probe_timing import alternating, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B, D, S = 8, 100, 14
MAX_CONTOURS, MAX_POINTS = 64, 16384
MIXED = [(640, 480), (480, 640), (1280, 720), (1920, 1080), (1333, 750), (800, 800), (3000, 200), (64, 48)]


def inputs(seed, net_w, net_h, kept):
    rng = np.random.default_rng(seed)
    s = np.exp(rng.uniform(np.log(32), np.log(256), (B, D)))
    x1, y1 = rng.uniform(0, net_w - s), rng.uniform(0, net_h - s)
    boxes = np.stack([x1, y1, x1 + s, y1 + s], -1).astype(np.float32)
    scores = np.where(np.arange(D)[None, :] < kept, 0.9, 0.3).astype(np.float32).repeat(B, 0)
    for b in range(B):
        rng.shuffle(scores[b])
    classes = rng.integers(0, 80, (B, D)).astype(np.float32)
    masks = (1 / (1 + np.exp(-rng.standard_normal((B, D, S, S)) * 2))).astype(np.float32)
    return [torch.from_numpy(a).to(dev) for a in (scores, boxes, classes, masks)]


def host_path_ms(canv, counts):
    """D2H of the kept canvases into pinned buffers + sync, then cv2.findContours per kept canvas on one thread."""
    pinned = [torch.empty((n,) + tuple(c.shape[1:]), dtype=torch.uint8, pin_memory=True) for c, n in zip(canv, counts)]
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c, p, n in zip(canv, pinned, counts):
            p.copy_(c[:n], non_blocking=True)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        for p in pinned:
            a = p.numpy()
            for k in range(a.shape[0]):
                cv2.findContours(a[k], cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)
        t2 = time.perf_counter()
        times.append((t1 - t0, t2 - t1))
    copy, find = (float(np.median([t[i] for t in times])) * 1e3 for i in range(2))
    return copy, find


def workload(name, frames, net_w, net_h, kept, seed):
    t = inputs(seed, net_w, net_h, kept)
    rows = torch.empty((B, 1 + D * 7), dtype=torch.float32, device=dev)
    canv = [torch.zeros((D, h, w), dtype=torch.uint8, device=dev) for w, h in frames]
    out = (torch.zeros((B, D, 2), dtype=torch.int32, device=dev), torch.zeros((B, D, MAX_CONTOURS), dtype=torch.int32,
           device=dev), torch.zeros((B, D, MAX_POINTS, 2), dtype=torch.int32, device=dev))
    lib = L.load()
    q = L.RcnnPostParams(net_w, net_h, 0, 0, D, S, D, 0.6)
    descs, _ = P._frames(frames, canv, D, dev, True)
    nbytes = lib.trtx_rcnn_contours_workspace_size(C.byref(q), descs, B)
    work = torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def post_call():
        P.rcnn_postprocess_frames(*t, frames=frames, net_w=net_w, net_h=net_h, rows=rows, canvases=canv)

    def contour_call():
        L.check(lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, B, rows.data_ptr(), MAX_CONTOURS, MAX_POINTS,
                                               out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), work.data_ptr(),
                                               nbytes, torch.cuda.current_stream().cuda_stream), "contours")

    post_call()
    contour_call()
    torch.cuda.synchronize()
    us = alternating({"contours": contour_call, "post": post_call})
    counts = [min(int(v), D) for v in rows[:, 0].tolist()]
    # every canvas against the oracle
    cnt, ln, pt = (x.cpu().numpy() for x in out)
    ok, n_contours, n_points = True, 0, 0
    for b, c in enumerate(canv):
        a = c.cpu().numpy()
        for k in range(counts[b]):
            n, tot, l2, p2 = CO.find_contours_external(np.ascontiguousarray(a[k]))
            n_contours, n_points = n_contours + n, n_points + tot
            nl, npt = min(n, MAX_CONTOURS), min(tot, MAX_POINTS)
            ok &= tuple(cnt[b, k]) == (n, tot) and np.array_equal(ln[b, k, :nl], l2[:nl]) and \
                np.array_equal(pt[b, k, :npt], p2[:npt])
    copy_ms, find_ms = host_path_ms(canv, counts)
    host_us = (copy_ms + find_ms) * 1e3
    return {"name": name, "frames": frames, "net": [net_w, net_h], "canvases": sum(counts), "contours": n_contours,
            "points": n_points, "canvas_bytes": sum(n * w * h for n, (w, h) in zip(counts, frames)),
            "workspace_bytes": int(nbytes), "contours_call_us": round(us["contours"], 2),
            "postprocess_call_us": round(us["post"], 2), "contours_over_postprocess": round(us["contours"] / us["post"], 3),
            "host_d2h_sync_ms": round(copy_ms, 3), "host_findcontours_ms": round(find_ms, 3),
            "host_path_over_contours_call": round(host_us / us["contours"], 2), "equal_to_oracle": bool(ok)}


def main(outdir: Path):
    cv2.setNumThreads(1)
    res = {"cv2": cv2.__version__,
           "timing": "20 graph-captured calls x 20 replays between CUDA events, median of 3 alternating rounds",
           "workloads": []}
    for args in (("b8_640x480_kept20", [(640, 480)] * B, 1067, 800, 20, 2),
                 ("b8_1920x1080_kept20", [(1920, 1080)] * B, 1333, 750, 20, 2),
                 ("b8_640x480_kept100", [(640, 480)] * B, 1067, 800, 100, 2),
                 ("b8_mixed_8_sizes_kept20", MIXED, 1067, 800, 20, 1)):
        w = workload(*args)
        res["workloads"].append(w)
        print(json.dumps(w), flush=True)
    return res


if __name__ == "__main__":
    probe_main("rcnn_contours_probe", main)
