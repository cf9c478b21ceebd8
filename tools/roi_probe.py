"""RoIAlign kernel timing at the Faster R-CNN C4 shapes: N=1000 proposals, C=1024, 14x14 bins.  trtx_roi_align picks the
kernel from the shape: the 50x67 feature map runs the shared-memory window kernel, the 70x67 map (more than 4096 cells)
the direct kernel."""
import json, sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tensorrtx_b200 import plugins as P
dev = torch.device("cuda", 0)
rng = np.random.default_rng(0)
B, N, C, H, W, Pp = 2, 1000, 1024, 50, 67, 14
feat = torch.from_numpy(rng.standard_normal((B, C, H, W)).astype(np.float32)).to(dev)
x1 = rng.uniform(0, 900, (B, N)); y1 = rng.uniform(0, 700, (B, N))
w = np.exp(rng.uniform(np.log(16), np.log(600), (B, N))); h = np.exp(rng.uniform(np.log(16), np.log(500), (B, N)))
rois = torch.from_numpy(np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)).to(dev)
out = torch.empty((B, N, C, Pp, Pp), dtype=torch.float32, device=dev)
H_direct = 70
feat_direct = torch.from_numpy(rng.standard_normal((B, C, H_direct, W)).astype(np.float32)).to(dev)
for sampling in (0, 2):
    for name, f, fh in (("roi_align window (50x67 map)", feat, H), ("roi_align direct (70x67 map)", feat_direct, H_direct)):
        plug = P.RoiAlignPlugin(Pp, 1 / 16, sampling, N, C, fh, W)
        for _ in range(2):
            assert plug.enqueue(B, [rois, f], [out]) == 0
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        K = 5
        e0.record()
        for _ in range(K):
            plug.enqueue(B, [rois, f], [out])
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / K * 1e3
        print(json.dumps({"kernel": name, "sampling_ratio": sampling, "images": B, "us": round(us, 1), "ms_per_image": round(us / B / 1e3, 3),
                          "written_GBps": round(out.numel() * 4 / us / 1e3, 1)}), flush=True)
