"""Timing of the CenterNet decode (trtx_centernet_decode_enqueue) and pre-process (trtx_centernet_preprocess_enqueue) against
their HBM floors, against the D2H copy the device decode removes and against the sample's own host functions.

  python tools/centernet_probe.py OUTDIR      -> OUTDIR/centernet_probe.json (and the card line on stdout)

Decode workloads: b1, b8 and b32 of 80 x 128 x 128 heads of uniform logits in [-15, 15], and b32 of a N(-6, 2) background,
K = 100, with frame rows.  The floor is heat.amax() of the same tensor, a plain read of every logit.  Pre-process workloads: b8 of 1280x720, of 1920x1080 and of 8 mixed sizes, and b32 of
1920x1080, into the 512 x 512 input; the floor is a torch fill_ of the bytes it writes.  Each call and its floor are timed
as 20 launches captured in one CUDA graph, replayed 20 times between two events, alternating over 3 rounds (medians).
Host baseline, per frame, best of 3: the sample's pre_process and ctdet_decode (oracle/_ref/ref_centernet.pyc; "not
built" elsewhere) on torch CPU, and the D2H copy of hm, wh and reg into pinned memory plus a synchronise (median of 200)."""
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from probe_timing import alternating, d2h_sync_us, probe_main  # noqa: E402
from oracle import centernet as CO  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)
NC, H, W, K = 80, 128, 128, 100
MIXED = [(1920, 1080), (1280, 720), (640, 480), (3840, 2160), (1080, 1920), (800, 600), (1024, 576), (427, 240)]


def _best_s(fn, reps=3):
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def _heads(B, seed=0, background=False):
    """uniform logits in [-15, 15] (many sigmoids near 1 round to equal floats, so plateaus of equal peaks are common), or a
    background of N(-6, 2) logits, closer to a trained head's mostly negative map"""
    g = torch.Generator(device=dev).manual_seed(seed)
    if background:
        heat = torch.randn((B, NC, H, W), generator=g, device=dev) * 2 - 6
    else:
        heat = torch.rand((B, NC, H, W), generator=g, device=dev) * 30 - 15
    wh = torch.rand((B, 2, H, W), generator=g, device=dev) * 60
    reg = torch.rand((B, 2, H, W), generator=g, device=dev)
    return heat, wh, reg


def decode(res):
    sizes_all = [(1920, 1080)] * 32
    for B, bg in ((1, False), (8, False), (32, False), (32, True)):
        heat, wh, reg = _heads(B, background=bg)
        dets = torch.empty((B, K, 6), device=dev)
        rows = torch.empty((B, 1 + K * 6), device=dev)
        ws = torch.empty(8 * B * NC * K + 512, dtype=torch.uint8, device=dev)  # >= trtx_centernet_workspace_size
        sizes = sizes_all[:B]
        red = torch.empty((), device=dev)
        t = alternating({
            "call": lambda: P.centernet_decode(heat, wh, reg, K, image_sizes=sizes, workspace=ws, out=dets, rows_out=rows),
            "floor": lambda: torch.amax(heat, out=red),
        })
        d2h = d2h_sync_us(torch.cat([heat.reshape(-1), wh.reshape(-1), reg.reshape(-1)]), reps=200)
        res[f"decode_b{B}" + ("_background" if bg else "")] = {
            "call_us": t["call"], "amax_floor_us": t["floor"], "ratio": t["call"] / t["floor"], "heat_MB": heat.numel() * 4 / 1e6,
            "d2h_hm_wh_reg_us": d2h}


def preprocess(res):
    rng = np.random.default_rng(0)
    loads = {"720p_b8": [(1280, 720)] * 8, "1080p_b8": [(1920, 1080)] * 8, "mixed_b8": MIXED, "1080p_b32": [(1920, 1080)] * 32}
    for name, sizes in loads.items():
        frames = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).to(dev) for w, h in sizes]
        out = torch.empty((len(sizes), 3, 512, 512), device=dev)
        t = alternating({"call": lambda: P.centernet_preprocess(frames, out=out), "floor": lambda: out.fill_(0.0)})
        res[f"pre_{name}"] = {"call_us": t["call"], "fill_floor_us": t["floor"], "ratio": t["call"] / t["floor"]}


def host(res):
    ref = CO.reference()
    if ref is None:
        res["host"] = "not built"
        return
    torch.set_num_threads(1)
    img = np.random.default_rng(1).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    heat, wh, reg = (t[:1].cpu() for t in _heads(1))
    res["host"] = {"threads": 1, "pre_process_1080p_ms": _best_s(lambda: ref.pre_process(img)) * 1e3,
                   "ctdet_decode_ms": _best_s(lambda: ref.ctdet_decode(heat, wh, reg, K=K)) * 1e3}


def main(outdir):
    res = {}
    decode(res)
    preprocess(res)
    host(res)
    for k, v in res.items():
        print(k, v)
    return res


if __name__ == "__main__":
    probe_main("centernet_probe", main)
