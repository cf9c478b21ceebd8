"""Timing of the bicubic letterbox pre-process (trtx_cubic_preprocess_enqueue) against its write floor, the bilinear letterbox
of the same shapes, and the host path it replaces.

  python tools/cubic_pre_probe.py OUTDIR      -> OUTDIR/cubic_pre_probe.json (and the card line on stdout)

Workloads: b8 and b32 of 1920x1080 frames and b8 of mixed sizes (1920x1080, 1280x720, 640x480, 480x640, 300x200, 3840x2160,
608x608, 97x301), into yolov3-tiny's 608x608 input (TRTX_CUBIC_YOLOV3_TINY) and retinafaceAntiCov's 640x640 one
(TRTX_CUBIC_ANTICOV).  Every device figure is probe_timing.alternating: 20 launches in one CUDA graph, replayed 20 times between
two events, call and references alternating over 3 rounds, medians in microseconds per call:
  floor    a plain device fill (torch fill_) of the bytes the call writes;
  linear   trtx_cls_preprocess_enqueue's TRTX_YOLO_V5 letterbox (OpenCV's INTER_LINEAR into the same rectangle, 128 canvas,
           planar fp32) of the same frames;
  host     the path the call replaces, once per batch on the host clock (median of 5): cv2.resize INTER_CUBIC (cv2's default
           threads, IPP as installed) into the letterbox on a 128 canvas, the plane loop in numpy, and a pageable H2D copy of
           the fp32 batch followed by a synchronise."""
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
MIXED = [(1920, 1080), (1280, 720), (640, 480), (480, 640), (300, 200), (3840, 2160), (608, 608), (97, 301)]
MODELS = (("yolov3-tiny", L.CUBIC_YOLOV3_TINY, 608), ("anticov", L.CUBIC_ANTICOV, 640))


def _host_path(host_frames, variant, net):
    import cv2

    lut = (np.arange(256) / 255.0).astype(np.float32) if variant == L.CUBIC_YOLOV3_TINY else \
        ((np.arange(256).astype(np.float32).astype(np.float64) - 127.5) * 0.0078125).astype(np.float32)
    out = np.empty((len(host_frames), 3, net, net), np.float32)
    for b, img in enumerate(host_frames):
        x, y, w, h = _rect(img.shape[1], img.shape[0], net)
        canvas = np.full((net, net, 3), 128, np.uint8)
        canvas[y:y + h, x:x + w] = cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC)
        for c in range(3):
            out[b, c] = lut[canvas[:, :, 2 - c]]
    torch.from_numpy(out).to(dev)
    torch.cuda.synchronize()


def _rect(w, h, net):
    import ctypes as C

    r = (C.c_int * 4)()
    L.check(L.load().trtx_calib_letterbox_rect(w, h, net, net, r), "trtx_calib_letterbox_rect")
    return tuple(r)


def workload(name, sizes, model, variant, net, rng):
    host_frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sizes]
    frames = [torch.from_numpy(f).to(dev) for f in host_frames]
    B = len(frames)
    out = torch.empty((B, 3, net, net), dtype=torch.float32, device=dev)
    lin = torch.empty_like(out)
    floor = torch.empty(out.numel(), dtype=torch.float32, device=dev)
    t = alternating({"call": lambda: P.cubic_preprocess(frames, variant, out=out, net_w=net, net_h=net),
                     "linear": lambda: P.cls_preprocess(frames, L.YOLO_V5, net, net, out=lin),
                     "floor": lambda: floor.fill_(1.0)})
    host = []
    for _ in range(5):
        t0 = time.perf_counter()
        _host_path(host_frames, variant, net)
        host.append((time.perf_counter() - t0) * 1e6)
    host_us = float(np.median(host))
    return {
        "workload": f"{model} {name} b{B}", "net": net, "batch": B,
        "cubic_us": round(t["call"], 2), "floor_us": round(t["floor"], 2), "linear_us": round(t["linear"], 2),
        "cubic_over_floor": round(t["call"] / t["floor"], 2), "cubic_over_linear": round(t["call"] / t["linear"], 2),
        "host_us": round(host_us, 1), "host_over_cubic": round(host_us / t["call"], 1),
        "bytes_written": out.numel() * 4, "bytes_read": sum(w * h * 3 for w, h in sizes),
    }


def main(outdir):
    rng = np.random.default_rng(0)
    res = []
    for model, variant, net in MODELS:
        for name, sizes in (("1080p", [(1920, 1080)] * 8), ("1080p", [(1920, 1080)] * 32), ("mixed", MIXED)):
            r = workload(name, sizes, model, variant, net, rng)
            print(r, flush=True)
            res.append(r)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("cubic_pre_probe", main)
