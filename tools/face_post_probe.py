"""Timing of the RetinaFace post-process (trtx_retina_postprocess_enqueue) and of yolo26-obb's NMS-free rows
(TASK_OBB_NMS_FREE of trtx_yolo_pose_obb_postprocess_enqueue) against what any host path pays before its first row: the D2H
copy of the same compact rows and a synchronisation.

  python tools/face_post_probe.py OUTDIR      -> OUTDIR/face_post_probe.json (and the same JSON on stdout)

Workloads: b16 (BASELINE config 3, retina_b16) and b32 frames; retinaface (17-float NMS rows, CONF_THRESH 0.75, 3 in 4 faces
above it, 640x640 input) and retinafaceAntiCov (18-float rows, no threshold) at 20, 100 and 1000 faces per frame; yolo26-obb
plugin rows (90 floats, net 1024) at 300 rows per frame; all frames 1920 x 1080 or a mix of sizes.  Timed:
  call_us       the call, 20 launches captured in one CUDA graph, 20 replays between two CUDA events, per call;
  d2h_sync_us   torch copy of the compact rows into pinned host memory + torch.cuda.synchronize(), host wall clock, median
                of 200 (the least a host post-process pays before it starts);
  ref_host_us   where oracle/_ref was built: the reference's compiled loop over the frames' rows on one host core --
                retina_r50.cpp:373-388's threshold + get_rect_adapt_landmark (libref_retina_rows_host.so; AntiCov's copy is the
                same statements), or yolo26's draw_bbox_obb with its debug prints and recording drawing calls
                (libref_obb26_host.so) -- median of 5.  Not a device number: the host's own clock and CPU.
The calls are latency-bound (a few MB at most), so the figures are microseconds, not a bandwidth share."""
import ctypes as C
import json
import math
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import face_obb26 as FO  # noqa: E402
from probe_timing import d2h_sync_us, graph_us, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
MIXED = [(1920, 1080), (1280, 720), (640, 480), (1080, 1920), (3840, 2160), (333, 1001), (720, 1280), (1024, 1024)]
OBB26 = "obb26"


def inputs(kind, B, K, seed=3):
    rng = np.random.default_rng(seed)
    R = {L.RETINA_FACE: 17, L.RETINA_ANTICOV: 18, OBB26: 90}[kind]
    net = 1024 if kind == OBB26 else 640
    d = np.zeros((B, 1 + K * R), np.float32)
    for b in range(B):
        d[b, 0] = K
        r = d[b, 1:].reshape(K, R)
        s = np.exp(rng.uniform(np.log(16), np.log(256), K))
        x, y = rng.uniform(0, net - s), rng.uniform(0, net - s)
        if kind == OBB26:
            r[:, :4] = np.stack([x + s / 2, y + s / 2, s, s * rng.uniform(0.3, 1.5, K)], -1)
            r[:, 4], r[:, 5] = rng.uniform(0.3, 1, K), rng.integers(0, 15, K)
            r[:, 89] = rng.uniform(-np.pi / 4, 3 * np.pi / 4, K)
        else:
            r[:, :4] = np.stack([x, y, x + s, y + s], -1)
            r[:, 4] = np.where(rng.uniform(0, 1, K) < 0.75, 0.9, 0.5)
            r[:, 6] = 1
            r[:, 7:17] = (np.stack([x, y] * 5, -1) + rng.uniform(0, 1, (K, 10)) * np.repeat(s, 10).reshape(K, 10))
            if kind == L.RETINA_ANTICOV:
                r[:, 17] = rng.uniform(0, 1, K)
    return d, R


def ref_us(kind, dets, R, K, sizes):
    B = len(sizes)
    rows = np.ascontiguousarray(dets[:, 1:].reshape(B, K, R))
    if kind == OBB26:
        if FO.load_obb26() is None:
            return None
        boxes5 = [np.concatenate([rows[b, :, :4], rows[b, :, 89:90]], 1) for b in range(B)]

        def run():
            for b, (w, h) in enumerate(sizes):
                FO.ref_draw_bbox_obb_v26(w, h, boxes5[b])
    else:
        lib = FO.load_retina_rows()
        if lib is None:
            return None
        thr = 0.75 if kind == L.RETINA_FACE else -math.inf
        rect, lmk = np.zeros((K, 4), np.int32), np.zeros((K, 10), np.float32)
        ptrs = [rows[b].ctypes.data_as(C.c_void_p) for b in range(B)]
        pr, pl = rect.ctypes.data_as(C.c_void_p), lmk.ctypes.data_as(C.c_void_p)

        def run():
            for b, (w, h) in enumerate(sizes):
                lib.ref_retina_rows(w, h, 640, 640, ptrs[b], K, R, thr, pr, pl)
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        run()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def call(kind, dets_d, sizes, K, rows):
    if kind == OBB26:
        return lambda: P.yolo_pose_obb_postprocess(dets_d, sizes, task=L.TASK_OBB_NMS_FREE, max_rows=K, net_w=1024,
                                                   net_h=1024, rows_out=rows)
    thr = 0.75 if kind == L.RETINA_FACE else -math.inf
    return lambda: P.retina_postprocess(dets_d, sizes, variant=kind, max_rows=K, conf_thresh=thr, in_w=640, in_h=640,
                                        rows_out=rows)


def main(outdir: Path):
    res = {"timing": "call: 20 graph-captured launches x 20 replays between CUDA events; d2h: median of 200 host-timed",
           "workloads": []}
    plan = [(kind, K) for kind in (L.RETINA_FACE, L.RETINA_ANTICOV) for K in (20, 100, 1000)] + [(OBB26, 300)]
    names = {L.RETINA_FACE: "retinaface", L.RETINA_ANTICOV: "anticov", OBB26: OBB26}
    for B in (16, 32):
        for kind, K in plan:
            dets, R = inputs(kind, B, K)
            dets_d = torch.from_numpy(dets).to(dev)
            Fo = {L.RETINA_FACE: 15, L.RETINA_ANTICOV: 16, OBB26: 10}[kind]
            rows = torch.empty((B, 1 + K * Fo), dtype=torch.float32, device=dev)
            for label, sizes in (("1080p", [(1920, 1080)] * B), ("mixed", [MIXED[b % len(MIXED)] for b in range(B)])):
                us = graph_us(call(kind, dets_d, sizes, K, rows))
                w = {"kind": names[kind], "frames": label, "batch": B, "rows_per_frame": K, "in_bytes": dets.nbytes,
                     "out_bytes": rows.numel() * 4, "call_us": round(us, 2), "d2h_sync_us": round(d2h_sync_us(dets_d), 2)}
                r = ref_us(kind, dets, R, K, sizes)
                if r is not None:
                    w["ref_host_us"] = round(r, 1)
                res["workloads"].append(w)
                print(json.dumps(w), flush=True)
    return res


if __name__ == "__main__":
    probe_main("face_post_probe", main)
