"""Write tests/golden/ref_face_obb26_host.npz: what the reference's own compiled code produces for the cases of
tests/test_face_obb26_post_cpu.py, as one sha256 per frame size -- RetinaFace's get_rect_adapt_landmark
(oracle/_ref/libref_retina_host.so; the -O0 build must agree) at both input sizes, and yolo26's draw_bbox_obb
(oracle/_ref/libref_obb26_host.so) at net 1024 -- so that machines without the reference still pin
trtx_retina_get_rect_adapt_landmark and trtx_get_corner."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from oracle import face_obb26 as FO  # noqa: E402
from oracle.golden import RefOutputs  # noqa: E402
import test_face_obb26_post_cpu as T  # noqa: E402


def main():
    o2, o0 = RefOutputs.lib("libref_retina_host.so"), RefOutputs.lib("libref_retina_host_O0.so")
    if o2 is None or o0 is None or FO.load_obb26() is None:
        raise SystemExit("oracle/_ref is missing the reference's retina or yolo26 host build (build it where the "
                         "reference tree is present)")
    g = {}
    for in_w, in_h in T.INPUTS:
        d = [T.face_digests(in_w, in_h, lambda w, h, b, k, lib=lib: T.ref_faces(lib, in_w, in_h, w, h, b, k))
             for lib in (o2, o0)]
        assert np.array_equal(d[0], d[1]), "the reference's -O2 and -O0 builds disagree"
        g[f"face_{in_w}x{in_h}"] = d[0]
    g["obb_v26"] = T.obb26_digests(lambda w, h, b: FO.ref_draw_bbox_obb_v26(w, h, b)[0])
    np.savez_compressed(T.GOLDEN, **g)
    print(f"{T.GOLDEN}: {len(T.SIZES)} frame sizes x {len(g)} sets")


if __name__ == "__main__":
    main()
