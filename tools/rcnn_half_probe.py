"""RpnDecode and PredictorDecode time, fp32 against fp16 scores and deltas, on tools/probe_timing.py's harness.

The reference's Mask R-CNN configuration at bench.py's rcnn_b8 batch: B = 8 images; RpnDecode on scores [15, 50, 67] and deltas
[60, 50, 67] per image, top 6000; PredictorDecode on scores [1000, 80] and deltas [80000, 4] per image with fp32 proposals.
Three legs per plugin, timed in turn within each of ROUNDS rounds in this one process (graph_us: LAUNCHES launches in a CUDA
graph, REPS replays between two events), so a drift of the card's clock hits all three alike:
  fp32               the fp32 call on fp32 tensors (what an FP32 engine runs)
  fp16               the half call on the half tensors (what an FP16 engine runs after this change)
  fp16 -> widen      STAND-IN for TensorRT's reformat layer in front of an fp32-only plugin: torch's copy kernel widens the half
                     scores and deltas into fp32 buffers, then the fp32 call, in the same graph.  TensorRT's own reformat
                     kernels are NOT measured (no TensorRT on the machine); the copy kernel reads and writes the same bytes.
Per row: the median and the min .. max of the rounds, microseconds per launch of the whole batch, and the bytes of the plugin
inputs (scores + deltas [+ proposals]) at the row's element size.

    python tools/rcnn_half_probe.py OUTDIR      ->  OUTDIR/rcnn_half_probe.json
"""
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

B, A, H, W, TOP_N = 8, 15, 50, 67, 6000
N, CLS = 1000, 80
ROUNDS, LAUNCHES, REPS = 7, 20, 50


def rounds(fns: dict, **kw) -> dict:
    """graph_us of every fn in turn, ROUNDS times: {name: [us per round]}"""
    t = {k: [] for k in fns}
    for _ in range(ROUNDS):
        for k, fn in fns.items():
            t[k].append(graph_us(fn, **kw))
    return t


def legs(plug, half_in, wide_bufs, fixed_in, outs, ws):
    """{leg: fn} for one plugin: fp32 tensors, half tensors, half tensors widened by a copy kernel then the fp32 call"""
    wide_in = [h.float() for h in half_in]

    def widened():
        for dst, src in zip(wide_bufs, half_in):
            dst.copy_(src)
        return plug.enqueue(B, [*wide_bufs, *fixed_in], outs, ws)

    return {"fp32": lambda: plug.enqueue(B, [*wide_in, *fixed_in], outs, ws),
            "fp16": lambda: plug.enqueue(B, [*half_in, *fixed_in], outs, ws),
            "fp16 -> widen (reformat stand-in)": widened}


def main(outdir):
    dev = torch.device("cuda", 0)
    ws = torch.empty(4096, dtype=torch.uint8, device=dev)
    s, d = synth.rpn_inputs(B, seed=0, A=A, H=H, W=W)
    rpn_half = [torch.from_numpy(x.astype(np.float16)).to(dev) for x in (s, d)]
    rpn = P.RpnDecodePlugin(TOP_N, synth.rcnn_anchors(), 16.0, 800, 1067, H, W)
    rpn_out = [torch.empty((B, TOP_N), device=dev), torch.empty((B, TOP_N, 4), device=dev)]
    cs, cd, props = synth.predictor_inputs(B, seed=1, N=N, Ccls=CLS)
    pred_half = [torch.from_numpy(x.astype(np.float16)).to(dev) for x in (cs, cd)]
    pred = P.PredictorDecodePlugin(N, 800, 1067, (10.0, 10.0, 5.0, 5.0), CLS)
    pred_out = [torch.empty((B, N), device=dev), torch.empty((B, N, 4), device=dev), torch.empty((B, N), device=dev)]
    pd = torch.from_numpy(props).to(dev)
    plugins = {
        "RpnDecode (b8, 15x50x67, top 6000)": (legs(rpn, rpn_half, [torch.empty_like(h, dtype=torch.float32) for h in rpn_half], [],
                                                     rpn_out, ws), sum(h.numel() for h in rpn_half), 0),
        "PredictorDecode (b8, 1000x80)": (legs(pred, pred_half, [torch.empty_like(h, dtype=torch.float32) for h in pred_half], [pd],
                                                pred_out, ws), sum(h.numel() for h in pred_half), pd.numel() * 4),
    }
    rows = []
    res = {"shape": {"batch": B, "rpn": [A, H, W], "top_n": TOP_N, "predictor": [N, CLS], "rounds": ROUNDS,
                     "launches_per_round": LAUNCHES * REPS}, "rows": rows}
    for name, (fns, elems, fixed_bytes) in plugins.items():
        for fn in fns.values():          # warm every leg before any is timed
            for _ in range(3):
                assert fn() == 0
        torch.cuda.synchronize()
        t = rounds(fns, n=LAUNCHES, reps=REPS)
        for leg, us in t.items():
            es = 4 if leg == "fp32" else 2
            row = {"plugin": name, "leg": leg, "us": round(float(np.median(us)), 1), "us_min": round(min(us), 1),
                   "us_max": round(max(us), 1), "input_MB": round((elems * es + fixed_bytes) / 1e6, 2)}
            rows.append(row)
            print(row, flush=True)
    return res


if __name__ == "__main__":
    probe_main("rcnn_half_probe", main)
