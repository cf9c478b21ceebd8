"""Timing of the YOLOP pre-process (trtx_yolop_preprocess_enqueue) and post-process with labels (trtx_yolop_postprocess_enqueue)
against the write floor and against the host code they replace.

  python tools/yolop_probe.py OUTDIR      -> OUTDIR/yolop_probe.json (and the card line on stdout)

Workloads: b8 and b32 of 1920x1080, of 1280x720 and of 8 mixed sizes (repeated), into YOLOP's 640x384 input; the post-process
takes 20 NMS rows per frame and writes one label canvas per frame from two 640x360 int32 maps.  Each call is timed as 20 launches
captured in one CUDA graph, replayed 20 times between two events; its floor is a plain device fill (torch fill_) of the bytes
the call writes, timed the same way; call and floor alternate over 3 rounds and the medians are reported.  Host paths, in one
process, host clock around a device synchronise:
  pre-process: per frame cv2 resize into the letterbox on a 114 canvas, convertTo / subtract / divide, the plane split, then the
               H2D copy of the fp32 batch from pageable memory (yolop/utils.h:11-36, yolop/yolop.cpp:110-127, yolop.hpp:217);
  labels:      the D2H copy of both int32 maps, then per frame two cv2.resize(INTER_NEAREST) and the lane / drivable-area
               selection in numpy (yolop.cpp:148-169 without the colour blend)."""
import ctypes as C
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
NET_W, NET_H, MAP_W, MAP_H, ROWS = 640, 384, 640, 360, 20
MEAN, STD = (0.485, 0.456, 0.406, 0.0), (0.229, 0.224, 0.225, 1.0)
MIXED = [(1920, 1080), (1280, 720), (640, 480), (3840, 2160), (1080, 1920), (800, 600), (1024, 576), (427, 240)]


def _letterbox_rect(w, h):
    r = (C.c_int * 4)()
    L.load().trtx_calib_letterbox_rect(w, h, NET_W, NET_H, r)
    return tuple(r)


def host_pre_us(frames, reps=3):
    import cv2
    data = np.empty((len(frames), 3, NET_H, NET_W), np.float32)
    dst = torch.empty(data.shape, dtype=torch.float32, device=dev)
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b, f in enumerate(frames):
            h, w = f.shape[:2]
            x, y, rw, rh = _letterbox_rect(w, h)
            out = np.full((NET_H, NET_W, 3), 114, np.uint8)
            out[y:y + rh, x:x + rw] = cv2.resize(f, (rw, rh), interpolation=cv2.INTER_LINEAR)
            t = out.astype(np.float32) * np.float32(1.0 / 255.0)
            t = cv2.divide(cv2.subtract(t, MEAN), STD, scale=1)
            data[b] = t.transpose(2, 0, 1)
        dst.copy_(torch.from_numpy(data))
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1e6)
    return best


def host_labels_us(seg, lane, sizes, reps=3):
    import cv2
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s, ln = seg.cpu().numpy(), lane.cpu().numpy()
        for b, (w, h) in enumerate(sizes):
            rs = cv2.resize(s[b], (w, h), interpolation=cv2.INTER_NEAREST)
            rl = cv2.resize(ln[b], (w, h), interpolation=cv2.INTER_NEAREST)
            np.where(rl != 0, 2, np.where(rs != 0, 1, 0)).astype(np.uint8)
        best = min(best, (time.perf_counter() - t0) * 1e6)
    return best


def workload(name, sizes, rng):
    B = len(sizes)
    frames_h = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sizes]
    frames = [torch.from_numpy(f).to(dev) for f in frames_h]
    inp = torch.empty((B, 3, NET_H, NET_W), dtype=torch.float32, device=dev)
    pre_floor = torch.empty(inp.numel(), dtype=torch.float32, device=dev)
    pre = alternating({"call": lambda: P.yolop_preprocess(frames, out=inp), "floor": lambda: pre_floor.fill_(1.0)})
    dets = torch.zeros((B, 1 + ROWS * 7), dtype=torch.float32, device=dev)
    d = dets[:, 1:].view(B, ROWS, 7)
    d[:, :, 0:2] = torch.rand((B, ROWS, 2), device=dev) * 600
    d[:, :, 2:4] = torch.rand((B, ROWS, 2), device=dev) * 100 + 4
    d[:, :, 4], d[:, :, 6] = 0.5, 1.0
    dets[:, 0] = ROWS
    seg = (torch.rand((B, MAP_H, MAP_W), device=dev) < 0.5).to(torch.int32)
    lane = (torch.rand((B, MAP_H, MAP_W), device=dev) < 0.1).to(torch.int32)
    rows = torch.empty((B, 1 + ROWS * 6), dtype=torch.float32, device=dev)
    canv = [torch.empty((h, w), dtype=torch.uint8, device=dev) for w, h in sizes]
    label_bytes = sum(w * h for w, h in sizes)
    lab_floor = torch.empty(label_bytes, dtype=torch.uint8, device=dev)
    post = alternating({"call": lambda: P.yolop_postprocess(dets, sizes, max_rows=ROWS, seg=seg, lane=lane, rows_out=rows,
                                                            canvases_out=canv),
                        "floor": lambda: lab_floor.fill_(1)})
    hp, hl = host_pre_us(frames_h), host_labels_us(seg, lane, sizes)
    return {
        "workload": name, "batch": B,
        "pre_us": round(pre["call"], 2), "pre_floor_us": round(pre["floor"], 2), "pre_bytes_written": inp.numel() * 4,
        "pre_host_us": round(hp, 1), "pre_speedup": round(hp / pre["call"], 1),
        "labels_us": round(post["call"], 2), "labels_floor_us": round(post["floor"], 2), "labels_bytes_written": label_bytes,
        "labels_over_floor": round(post["call"] / post["floor"], 2),
        "labels_host_us": round(hl, 1), "labels_speedup": round(hl / post["call"], 1),
    }


def main(outdir):
    rng = np.random.default_rng(0)
    res = []
    for B in (8, 32):
        for name, sizes in (("1080p", [(1920, 1080)] * B), ("720p", [(1280, 720)] * B), ("mixed", (MIXED * 4)[:B])):
            r = workload(f"{name} b{B}", sizes, rng)
            print(r, flush=True)
            res.append(r)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("yolop_probe", main)
