"""Timing of the Python runners' pre- and post-process on the device, next to the numpy they replace on the host cores.

  python tools/pyrunner_probe.py OUTDIR      -> OUTDIR/pyrunner_probe.json (and the card line on stdout)

Workload: b32 1920 x 1080 u8 frames into a 640 x 640 input (PyRunnerPreprocessPlan, TRTX_LINEAR_PY), and yolov8_det_trt's
post_process on b32 plugin buffers of 1000 rows of 90 floats (seeded boxes over the net, distinct confidences, about 60 %
of them above CONF_THRESH 0.5; PyRunnerPostprocess).  Device figures are probe_timing.alternating: 20 launches in one CUDA
graph, replayed 20 times between two events, 3 rounds, medians in microseconds per call.  The host figure runs the
runner's own preprocess_image + post_process per frame (from the reference tree where it is present, else the oracle's
numpy restatement of them, oracle/pyrunner.py; the JSON says which), one core, wall clock, median of 3 passes over the
32 frames, in microseconds per b32."""
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from probe_timing import alternating, probe_main  # noqa: E402
from oracle import pyrunner as PR  # noqa: E402
from tensorrtx_b200 import plugins as P  # noqa: E402

dev = torch.device("cuda", 0)


def main(outdir):
    B, K, F, W, H = 32, 1000, 90, 1920, 1080
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(B)]
    frames_d = [torch.from_numpy(f).to(dev) for f in frames]
    preset = P.PYRUNNER_PRESETS["yolov8_det_trt"]
    dets = np.stack([PR.plugin_rows(rng, preset, K, K, 640, 640, "distinct") for _ in range(B)])
    dets_d = torch.from_numpy(dets).to(dev)
    sizes = [(W, H)] * B
    pre = P.PyRunnerPreprocessPlan(frames_d)
    post = P.PyRunnerPostprocess("yolov8_det_trt", max_rows=K)
    rows = torch.empty((B, 1 + K * 6), dtype=torch.float32, device=dev)
    t = alternating({"pre b32 1920x1080 -> 640x640": pre.enqueue,
                     "post b32 x 1000 rows x 90": lambda: post(dets_d, sizes, rows_out=rows)})
    kept = int(rows[:, 0].sum().item())

    runner = PR.reference_runner("yolov8_det_trt")
    if runner is not None:
        impl, host_pre = "reference runner", lambda f: runner.preprocess_image(f)
        host_post = lambda d: runner.post_process(d, H, W)  # noqa: E731
    else:
        impl, host_pre = "oracle restatement", lambda f: PR.preprocess(f, 640, 640)
        host_post = lambda d: PR.postprocess(d, W, H, preset)  # noqa: E731
    passes = []
    for _ in range(3):
        t0 = time.perf_counter()
        for f, d in zip(frames, dets):
            host_pre(f)
            host_post(d.copy())
        passes.append((time.perf_counter() - t0) * 1e6)
    host_us = float(np.median(passes))
    dev_us = sum(t.values())
    res = [{"workload": k, "us": round(v, 2)} for k, v in t.items()]
    res[-1]["rows_kept_b32"] = kept
    res.append({"workload": "host numpy pre + post, b32, one core", "impl": impl, "us": round(host_us, 1),
                "device_speedup": round(host_us / dev_us, 1)})
    for r in res:
        print(r, flush=True)
    return {"rows": res}


if __name__ == "__main__":
    probe_main("pyrunner_probe", main)
