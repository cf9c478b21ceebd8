"""RoIAlign and Decode_TRT kernel time, fp32 against fp16 tensors, on tools/probe_timing.py's harness.

RoIAlign at the reference's configuration (rcnn.cpp:39-43,150): B = 2 images, N = 1000 proposals, C = 1024 channels, 14 x 14
bins, sampling_ratio 0 (adaptive) and 2, on the 50 x 67 map (shared-memory window kernel) and a 70 x 67 map (direct kernel).
Both precisions are warmed, then timed in turn within each of ROUNDS rounds in this one process (graph_us: LAUNCHES launches
in a CUDA graph, REPS replays between two events), so a drift of the card's clock hits both alike; the median and the
min .. max of the rounds are reported.

Per row: microseconds per launch, milliseconds per image, the ALGORITHMIC bytes (feature map read once + proposals + bins
written, from the shapes) over the kernel time, and two floors computed from shapes and data-sheet rates, not measured:
  hbm_floor_us   algorithmic bytes / 3.35 TB/s (H100 SXM HBM3, data sheet)
  lds_floor_us   window kernel only: the bytes of its shared-memory tap loads (bins x channels x samples x 4 taps x element
                 size; the samples counted from the proposals as the kernel counts them) / (128 B per clock per SM x SMs x
                 the card's max SM clock)
`nearer` names the larger floor, the limit the kernel is nearer to.  What TensorRT's reformat copies around an fp32-only
plugin cost is NOT measured here (no TensorRT on the machine).

    python tools/roi_half_probe.py OUTDIR      ->  OUTDIR/roi_half_probe.json
"""
import re
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from probe_timing import graph_us, probe_main  # noqa: E402

from tensorrtx_b200 import plugins as P  # noqa: E402
from tensorrtx_b200 import synth  # noqa: E402

B, N, C, W, PP = 2, 1000, 1024, 67, 14
ROUNDS, LAUNCHES, REPS = 5, 20, 25
HBM_BPS = 3.35e12


def rounds(fns: dict, **kw) -> dict:
    """graph_us of every fn in turn, ROUNDS times: {name: [us per round]}"""
    t = {k: [] for k in fns}
    for _ in range(ROUNDS):
        for k, fn in fns.items():
            t[k].append(graph_us(fn, **kw))
    return t


def samples_per_bin(rois: np.ndarray, sampling: int) -> float:
    """mean over the proposals of grid_h * grid_w as roi_geom computes it (fp32)"""
    if sampling > 0:
        return float(sampling * sampling)
    f = np.float32
    s = f(1 / 16)
    rw = (rois[..., 2] * s - f(0.5)) - (rois[..., 0] * s - f(0.5))
    rh = (rois[..., 3] * s - f(0.5)) - (rois[..., 1] * s - f(0.5))
    return float(np.mean(np.ceil(rh / f(PP)) * np.ceil(rw / f(PP))))


def main(outdir):
    dev = torch.device("cuda", 0)
    prop = torch.cuda.get_device_properties(0)
    rng = np.random.default_rng(0)
    x1 = rng.uniform(0, 900, (B, N)); y1 = rng.uniform(0, 700, (B, N))
    w = np.exp(rng.uniform(np.log(16), np.log(600), (B, N))); h = np.exp(rng.uniform(np.log(16), np.log(500), (B, N)))
    rois_np = np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)
    rois = torch.from_numpy(rois_np).to(dev)
    out = {torch.float32: torch.empty((B, N, C, PP, PP), dtype=torch.float32, device=dev),
           torch.float16: torch.empty((B, N, C, PP, PP), dtype=torch.float16, device=dev)}
    rows = []
    res = {"shape": {"images": B, "proposals": N, "channels": C, "bins": PP, "rounds": ROUNDS, "launches_per_round": LAUNCHES * REPS},
           "sms": prop.multi_processor_count, "rows": rows}
    sm_clock_hz = None
    for name, fh in (("window (50x67 map)", 50), ("direct (70x67 map)", 70)):
        f32 = torch.from_numpy(rng.standard_normal((B, C, fh, W)).astype(np.float32)).to(dev)
        feats = {torch.float32: f32, torch.float16: f32.half()}
        for sampling in (0, 2):
            plug = P.RoiAlignPlugin(PP, 1 / 16, sampling, N, C, fh, W)
            fns = {dt: (lambda dt=dt: plug.enqueue(B, [rois, feats[dt]], [out[dt]])) for dt in feats}
            for fn in fns.values():          # warm both before either is timed
                for _ in range(3):
                    assert fn() == 0
            torch.cuda.synchronize()
            t = rounds(fns, n=LAUNCHES, reps=REPS)
            spb = samples_per_bin(rois_np, sampling)
            for dt, us in t.items():
                es = 4 if dt == torch.float32 else 2
                nbytes = B * C * fh * W * es + B * N * 16 + B * N * C * PP * PP * es
                med = float(np.median(us))
                row = {"kernel": "roi_align " + name, "dtype": "fp32" if es == 4 else "fp16", "sampling_ratio": sampling,
                       "us": round(med, 1), "us_min": round(min(us), 1), "us_max": round(max(us), 1),
                       "ms_per_image": round(med / B / 1e3, 3), "algorithmic_MB": round(nbytes / 1e6, 1),
                       "algorithmic_GBps": round(nbytes / med / 1e3, 1), "hbm_floor_us": round(nbytes / HBM_BPS * 1e6, 1),
                       "samples_per_bin": round(spb, 2)}
                if fh == 50:
                    row["_tap_bytes"] = B * N * C * PP * PP * spb * 4 * es
                rows.append(row)
    # Decode_TRT at batch 16, 640 x 640
    Bd = 16
    heads = [torch.from_numpy(x).to(dev) for x in synth.retina_heads(Bd, seed=1)]
    dheads = {torch.float32: heads, torch.float16: [x.half() for x in heads]}
    dplug = P.DecodePlugin(640, 640)
    ws = torch.empty(max(dplug.getWorkspaceSize(Bd), 256), dtype=torch.uint8, device=dev)
    drows = torch.empty((Bd, dplug.output_elems()), dtype=torch.float32, device=dev)
    fns = {dt: (lambda dt=dt: dplug.enqueue(Bd, dheads[dt], [drows], ws)) for dt in dheads}
    for fn in fns.values():
        for _ in range(3):
            assert fn() == 0
    torch.cuda.synchronize()
    t = rounds(fns, n=50, reps=200)
    for dt, us in t.items():
        es = 4 if dt == torch.float32 else 2
        rows.append({"kernel": "Decode_TRT scan + pack (b16, 640x640)", "dtype": "fp32" if es == 4 else "fp16", "us": round(float(np.median(us)), 2),
                     "us_min": round(min(us), 2), "us_max": round(max(us), 2), "head_MB": round(sum(x.numel() for x in heads) * es / 1e6, 2)})
    # the shared-memory floor needs the card's max SM clock (nvidia-smi, the same call as the timings)
    from probe_timing import card
    m = re.search(r"(\d+)\s*MHz,\s*(\d+)\s*MHz\s*$", card()["nvidia_smi"])
    if m:
        sm_clock_hz = int(m.group(1)) * 1e6
        res["max_sm_clock_MHz"] = int(m.group(1))
    for row in rows:
        tap = row.pop("_tap_bytes", None)
        if tap is not None and sm_clock_hz:
            row["lds_floor_us"] = round(tap / (128 * prop.multi_processor_count * sm_clock_hz) * 1e6, 1)
            row["nearer"] = "shared-memory tap bandwidth" if row["lds_floor_us"] > row["hbm_floor_us"] else "HBM write bandwidth"
            row["share_of_nearer_floor"] = round(max(row["lds_floor_us"], row["hbm_floor_us"]) / row["us"], 2)
        elif "hbm_floor_us" in row:
            row["share_of_hbm_floor"] = round(row["hbm_floor_us"] / row["us"], 2)
        print(row, flush=True)
    return res


if __name__ == "__main__":
    probe_main("roi_half_probe", main)
