"""Timing of the REFERENCE's own roiAlign (oracle/_ref/libref_rcnn.so, built from /root/reference/rcnn/RoiAlign.cu) next to
trtx_roi_align on the same inputs -- test infrastructure (it executes oracle/_ref), not collected by pytest.
Run on a GPU: python tests/perf_roi_align_vs_reference.py"""
import runpy
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
g = runpy.run_path(str(ROOT / "tools" / "roi_probe.py"))   # prints the trtx_roi_align timings and leaves its tensors in g
json, torch, rois, feat, out = g["json"], g["torch"], g["rois"], g["feat"], g["out"]
B, N, H, W, Pp = g["B"], g["N"], g["H"], g["W"], g["Pp"]
# the reference's own roiAlign (oracle/_ref/libref_rcnn.so, built from /root/reference/rcnn/RoiAlign.cu) on the same inputs
import ctypes as C, time
from oracle.golden import RefOutputs  # importable: roi_probe put the repository root on sys.path
lib = RefOutputs.lib("libref_rcnn.so")
if lib is not None:
    for sampling in (0, 2):
        args = (B, C.c_void_p(rois.data_ptr()), C.c_void_p(feat.data_ptr()), C.c_void_p(out.data_ptr()), Pp, C.c_float(1 / 16),
                sampling, N, 1024, H, W)
        lib.ref_roi_align(*args)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(3):
            lib.ref_roi_align(*args)   # synchronises the device itself (RoiAlign.cu:178)
        us = (time.perf_counter() - t0) / 3 * 1e6
        print(json.dumps({"kernel": "reference roiAlign", "sampling_ratio": sampling, "images": B, "us": round(us, 1)}), flush=True)
