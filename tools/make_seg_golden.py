"""Write tests/golden/ref_seg_post_host.npz: what the reference's own draw_mask_bbox (oracle/_ref/libref_seg_host.so, built by
oracle/Makefile where the reference tree is present) selects for the cases of tests/test_seg_post_cpu.py, as a sha256 of
each packed selection and its pixel count, so that machines without the reference still pin the oracle to it."""
import hashlib
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from oracle import seg_post as SP  # noqa: E402
import test_seg_post_cpu as T  # noqa: E402


def main():
    if SP.load_ref() is None:
        raise SystemExit("oracle/_ref/libref_seg_host.so is missing (build it where the reference tree is present)")
    digests, counts = [], []
    for variant, w, h, b, seed in T._ref_cases():
        M, _ = T._ref_selection(variant, w, h, b, seed)
        sel = SP.ref_draw_mask_select(variant, M, b, w, h)
        digests.append(np.frombuffer(hashlib.sha256(np.packbits(sel).tobytes()).digest(), np.uint8))
        counts.append(int(sel.sum()))
    np.savez_compressed(T.GOLDEN, digests=np.stack(digests), counts=np.array(counts, np.int64))
    print(f"{T.GOLDEN}: {len(counts)} cases, {sum(counts)} selected pixels")


if __name__ == "__main__":
    main()
