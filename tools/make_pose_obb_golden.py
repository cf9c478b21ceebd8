"""Write tests/golden/ref_pose_obb_host.npz: what the reference's own draw_bbox_obb and draw_bbox_keypoints_line
(oracle/_ref/libref_pose_obb_host.so, built by oracle/Makefile where the reference tree is present) produce for the cases
of tests/test_pose_obb_post_cpu.py, as one sha256 per frame size (corners of the boxes whose get_rect is defined; rectangles
and mapped keypoints), so that machines without the reference still pin trtx_get_corner and trtx_get_rect_adapt_landmark."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from oracle import pose_obb as PO  # noqa: E402
import test_pose_obb_post_cpu as T  # noqa: E402


def main():
    if PO.load_ref() is None:
        raise SystemExit("oracle/_ref/libref_pose_obb_host.so is missing (build it where the reference tree is present)")
    g = {}
    for tree, net in T.TREES:
        g[f"obb_{tree}"] = T.obb_digests(tree, net, lambda w, h, b, tree=tree: PO.ref_draw_bbox_obb(tree, w, h, b)[0])
        g[f"pose_{tree}"] = T.pose_digests(tree, lambda w, h, l, k, tree=tree: PO.ref_draw_bbox_keypoints_line(tree, w, h, l, k))
    np.savez_compressed(T.GOLDEN, **g)
    print(f"{T.GOLDEN}: {len(T.SIZES)} frame sizes x {len(g)} sets")


if __name__ == "__main__":
    main()
