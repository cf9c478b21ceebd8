"""Timing of the YOLO classification pre- and post-process (trtx_cls_preprocess_enqueue, trtx_cls_postprocess_enqueue) against
the write floor and against the host code they replace.

  python tools/cls_probe.py OUTDIR      -> OUTDIR/cls_probe.json (and the same JSON on stdout)

Pre-process workloads: b32 of 1920x1080, of 640x480 and of 8 mixed sizes (each 4 times), into 224x224, for V8 and V5.  The call
is timed as 20 launches captured in one CUDA graph, replayed 20 times between two events; the floor is a plain device fill
(torch fill_) of the bytes the call writes, timed the same way; call and floor alternate over 3 rounds and the medians are
reported.  End to end, per batch:
  device path: H2D copy from pinned host memory of what the call reads (for V8 only the rows of each centre crop) + the call;
  host path:   what batch_preprocess + infer's H2D do (yolov8_cls.cpp:19-46, :149-150), in one process: cv2 crop, resize,
               cvtColor, the convertTo product (V5: the mean / std arithmetic), CHW, then the H2D copy of the fp32 batch from
               pageable memory, timed with a host clock around a device synchronise.
Post-process: b32 x 1 000 classes, k = 3 and 5, softmax.  The call is timed like the pre-process; the host path is the D2H copy
of the logits and a synchronise, then softmax + topk per image on one core: the drivers' own compiled functions
(oracle/_ref/libref_cls_yolov8.so) where they were built, else the C oracle, which restates them."""
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import cls as CO  # noqa: E402
from probe_timing import alternating, graph_us, probe_main  # noqa: E402
from tensorrtx_b200 import _lib as L  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
B, NET = 32, 224
MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
V5_LUT = ((np.arange(256.0)[:, None] / 255.0 - MEAN[None, :]) / STD[None, :]).astype(np.float32)   # [byte, R/G/B]


def host_pre_us(frames, variant, reps=3):
    import cv2
    data = np.empty((len(frames), 3, NET, NET), np.float32)
    dst = torch.empty(data.shape, dtype=torch.float32, device=dev)
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b, f in enumerate(frames):
            h, w = f.shape[:2]
            if variant == L.YOLO_V8:
                m = min(h, w)
                top, left = (h - m) // 2, (w - m) // 2
                re = cv2.resize(f[top:top + m, left:left + m], (NET, NET), interpolation=cv2.INTER_LINEAR)
                rgb = cv2.cvtColor(re, cv2.COLOR_BGR2RGB).astype(np.float32) * np.float32(1 / 255.0)
                data[b] = rgb.transpose(2, 0, 1)
            else:
                x, y, rw, rh = _v5_rect(w, h)
                re = cv2.resize(f, (rw, rh), interpolation=cv2.INTER_LINEAR)
                out = np.full((NET, NET, 3), 128, np.uint8)
                out[y:y + rh, x:x + rw] = re
                rgb = out[:, :, ::-1]
                data[b] = V5_LUT[rgb, np.arange(3)].transpose(2, 0, 1)
        dst.copy_(torch.from_numpy(data))
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) * 1e6)
    return best


def _v5_rect(w, h):
    r = (C.c_int * 4)()
    L.check(L.load().trtx_calib_letterbox_rect(w, h, NET, NET, r), "trtx_calib_letterbox_rect")
    return tuple(r)


def pre_workloads():
    mixed = [(1920, 1080), (1080, 1920), (640, 480), (480, 640), (1280, 720), (224, 224), (333, 517), (4000, 3000)]
    return (("b32_1920x1080", [(1920, 1080)] * B), ("b32_640x480", [(640, 480)] * B), ("b32_mixed8", mixed * (B // 8)))


def main(outdir: Path):
    res = {"timing": "20 graph-captured calls x 20 replays between CUDA events, median of 3 alternating rounds",
           "pre": [], "post": []}
    rng = np.random.default_rng(1)
    for name, sizes in pre_workloads():
        frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (w, h) in sizes]
        d_frames = [torch.from_numpy(f).to(dev) for f in frames]
        for variant, vname in ((L.YOLO_V8, "V8"), (L.YOLO_V5, "V5")):
            # the bytes the call reads: V8 the crop's rows, V5 the whole frame
            if variant == L.YOLO_V8:
                views = []
                for f in frames:
                    h, w = f.shape[:2]
                    m = min(h, w)
                    views.append(((h - m) // 2, m))
            else:
                views = [(0, f.shape[0]) for f in frames]
            pinned = [torch.from_numpy(np.ascontiguousarray(f[t:t + n])).pin_memory() for f, (t, n) in zip(frames, views)]
            targets = [d[t:t + n] for d, (t, n) in zip(d_frames, views)]
            read_bytes = int(sum(p.numel() for p in pinned))
            out = torch.empty((B, 3, NET, NET), dtype=torch.float32, device=dev)
            nbytes = out.numel() * 4
            fill = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
            tm = alternating({"call": lambda: P.cls_preprocess(d_frames, variant, NET, NET, out=out),
                              "floor": lambda: fill.fill_(0.5)})
            us, floor_us = tm["call"], tm["floor"]
            del fill

            def device_path():
                for p, t in zip(pinned, targets):
                    t.copy_(p, non_blocking=True)
                P.cls_preprocess(d_frames, variant, NET, NET, out=out)
            dev_us = graph_us(device_path, n=3, reps=10)
            host_us = host_pre_us(frames, variant)
            w = {"name": name, "variant": vname, "bytes_written": nbytes, "bytes_h2d_device_path": read_bytes,
                 "bytes_h2d_host_path": nbytes, "us": round(us, 2), "fill_floor_us": round(floor_us, 2),
                 "ratio_to_floor": round(us / floor_us, 3), "device_path_us_per_batch": round(dev_us, 1),
                 "host_path_us_per_batch": round(host_us, 1), "host_over_device": round(host_us / dev_us, 2)}
            res["pre"].append(w)
            print(json.dumps(w), flush=True)

    ref = ROOT / "oracle" / "_ref" / "libref_cls_yolov8.so"
    x = (rng.standard_normal((B, 1000)) * 3).astype(np.float32)
    d_x = torch.from_numpy(x).to(dev)
    host_x = torch.empty((B, 1000), dtype=torch.float32).pin_memory()
    if ref.exists():
        lib = C.CDLL(str(ref))
        res["host_post_code"] = "the driver's compiled softmax + topk (oracle/_ref/libref_cls_yolov8.so)"
    else:
        lib = None
        res["host_post_code"] = "the C oracle's softmax + topk (the drivers' functions were not built here)"
    for k in (3, 5):
        idx = torch.empty((B, k), dtype=torch.int32, device=dev)
        val = torch.empty((B, k), dtype=torch.float32, device=dev)

        def call():
            L.check(L.load().trtx_cls_postprocess_enqueue(1, B, 1000, d_x.data_ptr(), k, idx.data_ptr(), val.data_ptr(), None,
                                                          torch.cuda.current_stream().cuda_stream), "cls_post")
        us = float(np.median([graph_us(call) for _ in range(3)]))
        res_buf = np.empty(1000, np.float32)
        idx_buf = np.empty(k, np.int32)
        best = float("inf")
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_x.copy_(d_x, non_blocking=True)
            torch.cuda.synchronize()
            hx = host_x.numpy()
            for b in range(B):
                row = hx[b]
                if lib is not None:
                    lib.ref_cls_softmax(C.c_void_p(row.ctypes.data), 1000, C.c_void_p(res_buf.ctypes.data))
                    lib.ref_cls_topk(C.c_void_p(res_buf.ctypes.data), 1000, k, C.c_void_p(idx_buf.ctypes.data))
                else:
                    CO.topk(CO.softmax(row[None]), k)
            best = min(best, (time.perf_counter() - t0) * 1e6)
        w = {"name": f"b32_1000cls_k{k}", "us": round(us, 2), "host_path_us_per_batch": round(best, 1),
             "host_over_device": round(best / us, 1)}
        res["post"].append(w)
        print(json.dumps(w), flush=True)
    return res


if __name__ == "__main__":
    probe_main("cls_probe", main)
