"""Every route of the YoloLayer scans (yolo_decode.cu) against the CPU oracle, the reference's own kernels and each other.

yolo_pick_vec picks a scan route from the input dtype, the grid sizes and the alignment of the level pointers, and
launch_v8 then picks one of 13 (class slices, rows in flight) pairs.  This module forces each route by construction: the
same heads are read through contiguous views that start 0, 2, 4 or 8 bytes into their allocation (fp32 at +4 B and fp16
at +2 B -> VEC 1; fp16 at +8 B -> VEC 4), and grids decide the rest (an odd cell count -> VEC 1 for any dtype; a level
with g % 8 == 4, such as the 22x22 level of a 704x704 net, sends fp16 to VEC 4).  Every call fills its workspace with
0xff first and checks afterwards that exactly B * tiles(VEC) tile counts were written and that each image's add up to its
candidate count, so a test fails if the library took another route than the one it was meant to cover.

| scan | fp32, VEC 4 | fp32, VEC 1 | fp16, VEC 8 | fp16, VEC 4 | fp16, VEC 1 |
|---|---|---|---|---|---|
| v8 detect | 13 of 13 pairs | 13 of 13 pairs | 13 of 13 pairs | 13 of 13 pairs (+8 B; 704 net) | 13 of 13 pairs |
| v8 seg / pose / obb (pack kernel's extras) | 13 of 13 pairs | 13 of 13 pairs | 13 of 13 pairs | 13 of 13 pairs | 13 of 13 pairs |
| v5 / v5-seg / v7 (`yolo_v5_scan_kernel`) | yes | yes (+4 B; 648 net) | n/a | yes | yes |
| v3 (same kernel, `TRTX_YOLO_V3`) | yes (640 net) | yes (+4 B; 608 net) | n/a | yes (640 net) | yes |
| v3net: yolov3, yolov3-tiny (same kernel, `TRTX_YOLO_V3_NET`) | yes (20/40/80, 28x16, 20x12 two levels) | yes (+4 B; 19/38/76, 19x11) | n/a | yes | yes |
| v4: yolov4 (same kernel, `TRTX_YOLO_V4`, double Logist) | yes (20/40/80, 28x16, two levels) | yes (+4 B; 19/38/76, 19x11) | n/a | yes | yes |
| csp: scaled-yolov4 (same kernel, `TRTX_YOLO_V4_CSP`, double Logist) | yes (20/40/80, 28x16, two levels) | yes (+4 B; 19/38/76, 19x11) | n/a | yes | yes |

The yolov3 family runs on grid sets of its own (V3F_GRIDS: square and non-square, an odd cell count, two levels) at each
driver's compiled-in net (608 x 608; 512 x 512 for scaled-yolov4), and once at a 608 x 352 net against the oracle alone.
Its driver's own CalDetection kernel takes the same grids, anchors and class count from the plugin's serialized blob
(ref_v3f_plugin_enqueue_blob of oracle/_ref/libref_v3f_blob_<driver>.so), so every family case is also held to that
kernel bit for bit: count, box, both confidences and class, NaNs at the same places.

On these routes:
  * route matrix: all routes give byte-identical plugin buffers, fp16 heads exactly the fp32 call on the widened heads,
    and one run per variant matches the CPU oracle with the tolerances of tests/test_yolo_gpu.py;
  * fused and split: FusedYoloDecodeNms.enqueue, enqueue_scan + enqueue_nms, and the plugin buffer + batch_nms give the
    same bytes and the same kept anchor ids, equal to oracle.nms of the oracle's decode (also the BASELINE YOLOv8n fp16
    b32 configuration);
  * fused and split also write every row, count and anchor id themselves: the split form's buffers start poisoned, the
    object's own and a separate `out` (bench.py's double buffer);
  * non-finite and edge logits in class, objectness and box rows and in the seg / pose / obb extras, fp32 and fp16, for
    every variant, against the oracle (NaNs at the same places) and the reference's kernels (bit for bit where the
    reference build contracts no differently);
  * the gate window (+-64 ulps around logf(0.1f / 0.9f), x_lo and one ulp either side) and near-ulp sigmoid collisions,
    where only the reference's kernels (same CUDA expf) can arbitrate; for the family also pairs on which its float and
    double Logist disagree about a collision, the case where finish_best replays the class loop with the double form;
  * class-slice edges: nc smaller than the slice count, ties and saturated collisions on both sides of every slice
    boundary, for every pair.
Reference outputs come through RefOutputs("ref_gpu"): tests/golden/ref_gpu.npz where oracle/_ref was not built."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import v3family
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

from test_yolov3_family_cpu import LIBNAME, _sig

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_gpu")
ATOL = 1e-4
RTOL_EXP = 2e-6   # anchor-based boxes pass through expf / a sigmoid scaled to pixels (tests/test_yolo_gpu.py)
KT = 0.3          # keypoint threshold of the pose runs
PAIRS = ((1, 8), (1, 16), (2, 4), (2, 5), (2, 8), (2, 10), (2, 20), (4, 4), (4, 5), (4, 10), (4, 20), (8, 5), (8, 10))
V8 = {"v8": (80, 0), "seg": (80, 32), "pose": (1, 51), "obb": (15, 1)}   # mode -> (classes, extra channels)
# the yolov3 family: mode -> its driver in plugins.V3_FAMILY_DRIVERS (v3net's two-level grid sets: yolov3-tiny)
V3F = {"v3net": "yolov3", "v4": "yolov4", "csp": "scaled-yolov4"}
DET = {"v8": 90, "seg": 90, "pose": 90, "obb": 90, "v5": 38, "v5seg": 38, "v7": 6, "v3": 7, **{v: 7 for v in V3F}}
V3_ANCHORS = [k.anchors for k in P.YOLOV3_KERNELS]
# the family's grid sets: (gw, gh) per level in the plugin's level order (stride 32 first, as synth.yolov3_heads lays them
# out), and a net other than the driver's compiled-in INPUT_W x INPUT_H (None: the driver's)
V3F_GRIDS = {
    "square": (((20, 20), (40, 40), (80, 80)), None),       # every cell count % 4 == 0: VEC 4 where the view allows it
    "odd": (((19, 19), (38, 38), (76, 76)), None),          # 361 cells: VEC 1 on every route
    "rect": (((28, 16), (56, 32), (112, 64)), None),        # non-square: gw != gh and net_w / gw != net_h / gh
    "rect_odd": (((19, 11), (38, 22), (76, 44)), None),     # non-square, 209 cells: VEC 1
    "two": (((20, 12), (40, 24)), None),                    # two levels, non-square (v3net: yolov3-tiny's plugin)
    "net608x352": (((20, 20), (40, 40), (80, 80)), (608, 352)),   # a net no driver compiles in: the oracle alone
}
FOUR = {(torch.float32, 4), (torch.float32, 1), (torch.float16, 4), (torch.float16, 1)}
# route -> (dtype, byte offset of every level's view into its allocation)
ROUTES = {"f32": (torch.float32, 0), "f32+4": (torch.float32, 4), "f16": (torch.float16, 0), "f16+8": (torch.float16, 8),
          "f16+2": (torch.float16, 2)}


# ------------------------------------------------------------------ plumbing -----------------------------
def _grids(heads):
    return [int(np.prod(h.shape[2:])) for h in heads]


def _expect_vec(var, grids, dtype, offset):
    """yolo_pick_vec restated for views `offset` bytes into 256-byte-aligned allocations."""
    if dtype == torch.float16 and var in V8 and all(g % 8 == 0 for g in grids) and offset % 16 == 0:
        return 8
    need = 8 if dtype == torch.float16 else 16
    return 1 if any(g % 4 for g in grids) or offset % need else 4


def _place(heads, dtype, offset, dev):
    """Each head (numpy fp16 for fp16 routes, fp32 otherwise) as a contiguous device view starting `offset` bytes into
    its own allocation."""
    es = torch.empty(0, dtype=dtype).element_size()
    out = []
    for h in heads:
        buf = torch.empty(h.size + 64, dtype=dtype, device=dev)
        t = buf[offset // es: offset // es + h.size].view(h.shape)
        t.copy_(torch.from_numpy(np.ascontiguousarray(h)))
        assert (t.data_ptr() - offset) % 256 == 0 and t.is_contiguous()
        out.append(t)
    return out


def _route_heads(h16, dtype):
    return h16 if dtype == torch.float16 else [h.astype(np.float32) for h in h16]


def _assert_route(ws, B, grids, vec, count, max_out):
    """The scan wrote the tile counts of a 32*vec-cell tiling: B * tiles ints from offset 0, whose per-image sums are the
    images' candidate counts (`count`, the plugin buffer's count, clamped at max_out), and nothing after them.  Another
    tiling puts other tiles in each image's range, which then misses candidates or takes the next image's."""
    T = sum((g + 32 * vec - 1) // (32 * vec) for g in grids)
    n = B * T
    counts = ws.view(torch.int32)[:n + 1].cpu().numpy().astype(np.int64)
    assert (counts[:n] >= 0).all(), f"fewer tile counts than a VEC {vec} tiling has"
    if (4 * n) % 256:   # the candidate records start at the next 256-byte boundary
        assert counts[n] == -1, f"more tile counts than a VEC {vec} tiling has"
    total = counts[:n].reshape(B, T).sum(1)
    assert np.array_equal(np.minimum(total, max_out), np.asarray(count)), (f"tile counts of a VEC {vec} tiling", total, count)


def _v3f_driver(var, gset):
    return "yolov3-tiny" if var == "v3net" and len(V3F_GRIDS[gset][0]) == 2 else V3F[var]


def _v3f_net(var, gset):
    return V3F_GRIDS[gset][1] or P.V3_FAMILY_DRIVERS[_v3f_driver(var, gset)]["net"]


def _v3f_kernels(var, gset):
    """The grid set's levels with the driver's anchors, stride 32 first."""
    d = P.V3_FAMILY_DRIVERS[_v3f_driver(var, gset)]
    anchors = [a for _, _, a in sorted(d["kernels"], key=lambda k: k[0])]
    return [P.YoloKernel(gw, gh, a) for (gw, gh), a in zip(V3F_GRIDS[gset][0], anchors)]


def _plugin(var, dtype, net=640, nc=None, max_out=1000, gset="rect"):
    """The variant's plugin; the yolov3 family's takes its grids from `gset` (V3F_GRIDS) instead of `net`."""
    f16 = L.F16 if dtype == torch.float16 else L.F32
    if var in V3F:
        (w, h), variant = _v3f_net(var, gset), P.V3_FAMILY_DRIVERS[V3F[var]]["variant"]
        return P.YoloLayerPluginV3Net(80 if nc is None else nc, _v3f_kernels(var, gset), w, h, variant, maxOut=max_out,
                                      in_dtype=f16)
    if var in V8:
        nc = V8[var][0] if nc is None else nc
        return P.YoloLayerPlugin(nc, 17, KT, net, net, max_out, var == "seg", var == "pose", var == "obb", (8, 16, 32),
                                 in_dtype=f16)
    nc = 80 if nc is None else nc
    if var == "v3":
        return P.YoloLayerPluginV3(nc, maxOut=max_out, in_dtype=f16)
    ks = [P.YoloKernel(net // s, net // s, a) for s, a in zip((8, 16, 32), synth.V5_ANCHORS)]
    if var == "v7":
        return P.YoloLayerPluginV7(nc, net, net, max_out, ks, in_dtype=f16)
    return P.YoloLayerPluginV5(nc, net, net, max_out, var == "v5seg", ks, in_dtype=f16)


def _decode(plug, hd, B, dev, vec, grids):
    if isinstance(plug, P.YoloLayerPluginV3):
        plug.configure(hd)   # its grids come from the input tensors, and the workspace size from the grids
    out = torch.full((B, plug.output_elems()), -7.0, dtype=torch.float32, device=dev)
    ws = torch.full((plug.getWorkspaceSize(B),), 255, dtype=torch.uint8, device=dev)
    rc = plug.enqueue(hd, [out], ws) if isinstance(plug, P.YoloLayerPluginV3) else plug.enqueue(B, hd, [out], ws)
    assert rc == 0, rc
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    _assert_route(ws, B, grids, vec, got[:, 0], plug.mMaxOutObject)
    return got


def _heads16(var, B, seed, net=640, nc=None, n_obj=64, gset="rect"):
    """Synthetic heads of `var`, rounded to fp16 (every route reads the same values)."""
    if var in V3F:
        grids = V3F_GRIDS[gset][0]
        hs = synth.yolov3_heads(B, seed=seed, nc=80 if nc is None else nc, net_w=32 * grids[0][0], net_h=32 * grids[0][1],
                                strides=(32, 16, 8)[:len(grids)], n_obj=n_obj)
        assert [h.shape[2:] for h in hs] == [(gh, gw) for gw, gh in grids]
    elif var in V8:
        c, extra = V8[var]
        hs = synth.yolov8_heads(B, seed=seed, nc=c if nc is None else nc, extra=extra, net_w=net, net_h=net, n_obj=n_obj)
    elif var == "v3":
        hs = synth.yolov3_heads(B, seed=seed, nc=80 if nc is None else nc, net_w=net, net_h=net, n_obj=n_obj)
    else:
        hs = synth.yolov5_heads(B, seed=seed, nc=80 if nc is None else nc, net_w=net, net_h=net, n_obj=n_obj, seg=var == "v5seg")
    return [h.astype(np.float16) for h in hs]


def _oracle(oracle, var, wide, net=640, nc=None, max_out=1000, gset="rect"):
    if var in V3F:
        return v3family.decode(wide, [k.anchors for k in _v3f_kernels(var, gset)], P.V3_FAMILY_DRIVERS[V3F[var]]["variant"],
                               net=_v3f_net(var, gset), nc=80 if nc is None else nc, max_out=max_out)
    if var in V8:
        return oracle.yolov8_decode(wide, net_w=net, net_h=net, nc=V8[var][0] if nc is None else nc, max_out=max_out,
                                    kpt_thresh=KT, is_seg=var == "seg", is_pose=var == "pose", is_obb=var == "obb")
    nc = 80 if nc is None else nc
    if var == "v3":
        return oracle.yolov3_decode(wide, V3_ANCHORS, nc=nc, max_out=max_out)
    return oracle.yolov5_decode(wide, synth.V5_ANCHORS, net_w=net, net_h=net, nc=nc, max_out=max_out, det_floats=DET[var],
                                is_seg=var == "v5seg")


def _cols(var):
    return {"seg": list(range(38)), "pose": list(range(6)) + list(range(38, 89)), "obb": list(range(6)) + [89],
            "v5seg": list(range(38)), "v3": list(range(7)), **{v: list(range(7)) for v in V3F}}.get(var, list(range(6)))


def _check_oracle(var, got, ref, max_out=1000):
    """Counts and classes exact, values within ATOL (+ RTOL_EXP for anchor-based boxes), NaN and inf at the same places."""
    F = DET[var]
    assert np.array_equal(np.minimum(ref[:, 0], max_out), got[:, 0]), (got[:, 0], ref[:, 0])
    rtol = 0.0 if var in V8 else RTOL_EXP
    for b in range(got.shape[0]):
        n = int(got[b, 0])
        g = got[b, 1:1 + n * F].reshape(n, F)[:, _cols(var)]
        r = ref[b, 1:1 + n * F].reshape(n, F)[:, _cols(var)]
        np.testing.assert_allclose(g, r, atol=ATOL, rtol=rtol, err_msg=var)
        assert np.array_equal(g[:, 5], r[:, 5])


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------ reference kernels -------------------------------
REF_LIB_SCAN = {"v8": "libref_yolov8.so", "v5": "libref_yolov5.so", "v7": "libref_yolov7.so", "v3": "libref_yolov3.so"}
REF_LIB = {**REF_LIB_SCAN, "seg": "libref_yolov8.so", "pose": "libref_yolov8.so", "obb": "libref_yolov8.so",
           "v5seg": "libref_yolov5.so"}


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _ref_decode(var, wide, dev, nc=80, gset="rect"):
    """The reference's own plugin kernel on fp32 heads (640x640, the variant's classes, 1000 rows; the yolov3 family: its
    driver's kernel built from our plugin's blob, so on gset's grids with nc classes), or None where it was not built."""
    lib = G.lib(f"libref_v3f_blob_{LIBNAME[_v3f_driver(var, gset)]}.so" if var in V3F else REF_LIB[var])
    if lib is None:
        return None
    B = wide[0].shape[0]
    hd = [torch.from_numpy(np.ascontiguousarray(h)).to(dev) for h in wide]
    out = torch.zeros((B, 1 + 1000 * DET[var]), dtype=torch.float32, device=dev)
    po = C.c_void_p(out.data_ptr())
    if var in V3F:
        wh = (C.c_int * 2)()
        lib.ref_v3f_net(wh)
        assert V3F_GRIDS[gset][1] is None and tuple(wh) == _v3f_net(var, gset) and lib.ref_v3f_max_out() == 1000
        blob = _plugin(var, torch.float32, nc=nc, gset=gset).serialize()
        rc = lib.ref_v3f_plugin_enqueue_blob(blob, C.c_size_t(len(blob)), B, _ptrs(hd), po)
    elif var in V8:
        rc = lib.ref_v8_plugin_enqueue(_nc(var), 17, C.c_float(KT), 640, 640, 1000, int(var == "seg"), int(var == "pose"),
                                       int(var == "obb"), (C.c_int * 3)(8, 16, 32), 3, B, _ptrs(hd), po, None)
    elif var == "v3":
        rc = lib.ref_v3_plugin_enqueue(B, (C.c_int * 3)(*[h.shape[2] for h in wide]), (C.c_int * 3)(*[h.shape[3] for h in wide]),
                                       _ptrs(hd), po)
    else:
        ks = np.zeros((3, 8), np.float32)
        for l, (s, a) in enumerate(zip((8, 16, 32), synth.V5_ANCHORS)):
            ks.view(np.int32)[l, :2] = 640 // s
            ks[l, 2:] = a
        kp = ks.ctypes.data_as(C.c_void_p)
        if var in ("v5", "v5seg"):
            rc = lib.ref_v5_plugin_enqueue(80, 640, 640, 1000, int(var == "v5seg"), kp, 3, B, _ptrs(hd), po, None)
        else:
            rc = lib.ref_v7_plugin_enqueue(80, 640, 640, 1000, kp, 3, B, _ptrs(hd), po, None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _lead(var):
    """Positions, within _cols(var), of the confidence, the class (and v3's class confidence)."""
    return [4, 5, 6] if var == "v3" or var in V3F else [4, 5]


def _canon(buf, b, var):
    """Image b's rows (the columns the reference writes), sorted by their uint32 bit patterns: conf, class (and v3's class
    confidence) first, the box after -- the reference's slot order is atomicAdd arrival."""
    if buf is None:
        return None
    F = DET[var]
    n = int(buf[b, 0])
    rows = np.ascontiguousarray(buf[b, 1:1 + n * F].reshape(n, F)[:, _cols(var)])
    u = rows.view(np.uint32)
    keys = [u[:, c] for c in _lead(var) + [0, 1, 2, 3]]
    return rows[np.lexsort(keys[::-1])]


def _vs_ref(key, var, got, ref):
    """Our plugin buffer against the reference kernel's: count exact; v8 and yolov3-family rows bit for bit (the family's
    box as tests/test_yolov3_family_gpu.py holds it); elsewhere conf / class bit for bit, anchor-based boxes within 3e-7
    (the reference build contracts its box arithmetic into FMAs differently), and the rest of a seg / pose / obb row within
    1e-6 (fp64 trigonometry and keypoint arithmetic, as tests/test_vs_reference_gpu.py compares them); NaNs at the same
    places."""
    G.equal(key + ".count", got[:, 0], None if ref is None else ref[:, 0])
    for b in range(got.shape[0]):
        g, r = _canon(got, b, var), _canon(ref, b, var)
        if var == "v8" or var in V3F:
            G.equal(f"{key}.{b}", g.view(np.uint32), None if r is None else r.view(np.uint32))
            continue
        lead = _lead(var)
        rest = [c for c in range(g.shape[1]) if c not in lead]
        G.equal(f"{key}.{b}.conf_class", np.ascontiguousarray(g[:, lead]).view(np.uint32),
                None if r is None else np.ascontiguousarray(r[:, lead]).view(np.uint32))
        if var in REF_LIB_SCAN:
            G.close(f"{key}.{b}.box", g[:, rest], None if r is None else r[:, rest], rtol=3e-7, atol=0)
        else:
            G.close(f"{key}.{b}.rest", g[:, rest], None if r is None else r[:, rest], rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------ route matrix -----------------------------------
def _route_matrix_case(oracle, dev, var, seed, net=640, gset="rect"):
    """One heads set through every route (and every built (slices, rows) pair of the v8 scan); returns the (dtype, VEC)
    pairs it ran."""
    B = 2
    h16 = _heads16(var, B, seed=seed, net=net, gset=gset, n_obj=24 if var in ("seg", "pose", "obb", "v5seg") else 64)
    grids = _grids(h16)
    first, seen = None, set()
    for route, (dtype, off) in ROUTES.items():
        vec = _expect_vec(var, grids, dtype, off)
        seen.add((dtype, vec))
        hd = _place(_route_heads(h16, dtype), dtype, off, dev)
        for pair in (PAIRS if var in V8 else (None,)):
            plug = _plugin(var, dtype, net, gset=gset)
            if pair:
                plug.tune(slices=pair[0], rows=pair[1])
            got = _decode(plug, hd, B, dev, vec, grids)
            if first is None:
                first = got
                assert got[:, 0].min() > 10
            assert _bits_equal(got, first), (route, pair)
    wide = [h.astype(np.float32) for h in h16]
    ref, _ = _oracle(oracle, var, wide, net=net, gset=gset)
    _check_oracle(var, first, ref)
    if var in V3F and V3F_GRIDS[gset][1] is None:   # the driver's own kernel, at the net it compiles in
        _vs_ref(f"scan_route.{var}.{gset}", var, first, _ref_decode(var, wide, dev, gset=gset))
    return seen


@pytest.mark.parametrize("var,net", [("v8", 640), ("v8", 704), ("seg", 640), ("pose", 640), ("obb", 640), ("v5", 640),
                                     ("v5", 648), ("v5seg", 640), ("v7", 640), ("v3", 640), ("v3", 608)] +
                         [(v, None) for v in V3F])
def test_route_matrix(oracle, dev, var, net):
    """The same heads through every route (and every built (slices, rows) pair of the v8 scan): byte-identical plugin
    buffers; fp16 heads give exactly the fp32 call on the widened heads; one run matches the oracle.  The yolov3 family
    (net None) runs every grid set of V3F_GRIDS, each also against its driver's own kernel, and covers all four routes
    across them."""
    if var in V3F:
        seen = set()
        for i, gset in enumerate(V3F_GRIDS):
            s = _route_matrix_case(oracle, dev, var, seed=720 + 10 * i + len(var), gset=gset)
            odd = any(gw * gh % 4 for gw, gh in V3F_GRIDS[gset][0])
            assert s == ({(torch.float32, 1), (torch.float16, 1)} if odd else FOUR), gset
            seen |= s
        assert seen == FOUR
        return
    seen = _route_matrix_case(oracle, dev, var, seed=700 + net + len(var), net=net)
    expected = set(FOUR)
    if var in V8 and net == 640:
        expected.add((torch.float16, 8))
    if net in (648, 608):      # an odd level: VEC 1 whatever the alignment
        expected = {(torch.float32, 1), (torch.float16, 1)}
    assert seen == expected


# ------------------------------------------------------------------ fused and split -------------------------------
# mode -> (oracle.nms variant, box format, conf threshold, IoU threshold); the yolov3 family: its driver's nms() parameters
FUSED = {"v8": (0, L.BOX_LTRB, 0.5, 0.45), "v5": (1, L.BOX_CXCYWH, 0.5, 0.45), "v3": (1, L.BOX_CXCYWH, 0.5, 0.4),
         **{v: (1, L.BOX_CXCYWH, P.V3_FAMILY_DRIVERS[d]["conf_thresh"], P.V3_FAMILY_DRIVERS[d]["nms_thresh"])
            for v, d in V3F.items()}}


def _fused_three_ways(oracle, dev, var, route, B, seed, net=640):
    dtype, off = ROUTES[route]
    h16 = _heads16(var, B, seed=seed, net=net)
    grids = _grids(h16)
    vec = _expect_vec(var, grids, dtype, off)
    hd = _place(_route_heads(h16, dtype), dtype, off, dev)
    nms_var, box, conf, iou = FUSED[var]
    F = DET[var]
    plug = _plugin(var, dtype, net)
    if var == "v3":
        plug.configure(hd)   # its grids come from the input tensors, and the workspace size from the grids
    buf = _decode(plug, hd, B, dev, vec, grids)
    if var in V3F:
        _vs_ref(f"scan_fused.{var}.{route}", var, buf, _ref_decode(var, [h.astype(np.float32) for h in h16], dev))
    fused = P.FusedYoloDecodeNms(plug, B, conf, iou, device=dev)
    comp1, idx1 = (t.clone() for t in fused.enqueue(B, hd))
    # split form, into the object's own buffers and (as bench.py's double buffer does) into another `out`: every buffer
    # the second half writes starts poisoned, so a row, count or anchor id it leaves out cannot pass
    split = []
    for out in (None, torch.full_like(fused.out, float("nan"))):
        fused.out.fill_(float("nan"))
        fused.idx.fill_(-7)
        fused.ws.fill_(255)
        fused.enqueue_scan(B, hd)
        torch.cuda.synchronize()
        _assert_route(fused.ws, B, grids, vec, buf[:, 0], 1000)
        split.append([t.clone() for t in fused.enqueue_nms(B, hd, out=out)])
        torch.cuda.synchronize()
        if out is not None:
            assert torch.isnan(fused.out).all()   # the object's own output is left alone
    comp3, row3 = P.batch_nms(torch.from_numpy(buf).to(dev), B, buf.shape[1], conf, iou, box_format=box, det_floats=F,
                              return_index=True)
    comp1, idx1, comp3, row3 = (t.cpu().numpy() for t in (comp1, idx1, comp3, row3))
    assert _bits_equal(comp1, comp3)
    for comp2, idx2 in split:
        comp2, idx2 = comp2.cpu().numpy(), idx2.cpu().numpy()
        assert _bits_equal(comp1, comp2)
        for b in range(B):
            assert np.array_equal(idx1[b, :int(comp1[b, 0])], idx2[b, :int(comp1[b, 0])])
    ref, ref_idx = _oracle(oracle, var, [h.astype(np.float32) for h in h16], net=net)
    _check_oracle(var, buf, ref)
    for b in range(B):
        res, src = oracle.nms(nms_var, ref[b], 1000, F, conf, iou)
        n = int(comp1[b, 0])
        assert n == len(res) and n > 5
        ids = ref_idx[b][src]
        assert np.array_equal(idx1[b, :n], ids) and np.array_equal(ref_idx[b][row3[b, :n]], ids)
        np.testing.assert_allclose(comp1[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL,
                                   rtol=0.0 if var == "v8" else RTOL_EXP)


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("var", list(FUSED))
def test_fused_split_and_two_stage_agree_on_every_route(oracle, dev, var, route):
    """FusedYoloDecodeNms.enqueue, enqueue_scan + enqueue_nms (the split form bench.py times), and the plugin buffer +
    batch_nms: identical bytes and kept anchor ids on every route, equal to oracle.nms of the oracle's decode (the yolov3
    family: with its driver's thresholds, and its plugin buffer equal to the driver's own kernel)."""
    _fused_three_ways(oracle, dev, var, route, 3, seed=760 + list(ROUTES).index(route), net=640)


def test_fused_split_fp16_b32_baseline_config(oracle, dev):
    """The BASELINE "YOLOv8n FP16 b32" configuration (bench.py --head-dtype f16): fp16 heads, 8 anchors per lane."""
    _fused_three_ways(oracle, dev, "v8", "f16", 32, seed=780)


# ------------------------------------------------------------------ non-finite and edge logits -------------------
H = np.float16
NAN, INF = np.nan, np.inf
# fp16 NaN payloads: signalling with payload 1, quiet with payload 1, negative quiet
NAN_BITS = (0x7C01, 0x7E01, 0xFE00)


def _all(v, nc=80):
    return {c: v for c in range(nc)}


# class-row cases: classes {index: value}; values -8 elsewhere; objectness 3 (anchor-based)
CLASS_CASES = [
    _all(NAN),                                          # every class NaN: P == 0
    {10: NAN, 20: 2.0, 30: NAN},                        # NaN beside a real maximum
    {0: NAN, 1: 1.25},
    {7: INF},
    {3: -INF, 50: 1.0},
    {12: INF, 40: INF},                                 # two +inf: the first
    {5: 17.0, 9: INF},                                  # +inf after a saturating 17.0: sigmoid 1.0f twice, class 5
    {4: -0.0, 8: 0.0},                                  # -0.0 / +0.0: one probability, the first class
    {4: 0.0, 8: -0.0},
    {**_all(-90.0), 3: -INF, 70: -65504.0},             # every logit <= -88: P == 0, class 0
    _all(-INF),
    {6: 65504.0, 60: 65504.0},                          # fp16 extremes
    {**_all(-65504.0), 33: -2.0},
    {2: 2.0 ** -24, 3: -(2.0 ** -24), 4: 2.0 ** -14},   # subnormals and the smallest normal: sigmoid 0.5
    {0: "nan0", 1: "nan1", 2: "nan2", 11: 1.5},         # NaN payloads
    {0: "nan0", 1: "nan1", 2: "nan2"},
]
# objectness cases (anchor-based): (objectness, classes)
OBJ_CASES = [
    (NAN, {5: 2.0}),
    (NAN, {}),                                          # NaN objectness, background classes
    (NAN, _all(-INF)),                                  # ... and P == 0
    ("nan0", {5: 2.0}), ("nan1", {77: 0.5}), ("nan2", {}),
    (INF, {5: 2.0}), (-INF, {5: 2.0}), (-90.0, {5: 2.0}), (-0.0, {5: 2.0}), (0.0, {6: -0.0}), (65504.0, {5: 2.0}),
    (-65504.0, {5: 2.0}), (2.0 ** -24, {5: 2.0}),
]
# box-row cases: the four box values of an anchor whose class 5 passes
BOX_CASES = [(NAN, 1.0, 1.5, 0.5), (1.0, INF, 0.5, 0.25), (0.5, 1.0, -INF, 2.0), (-0.0, -0.0, -0.0, -0.0),
             (65504.0, -65504.0, 65504.0, -65504.0), ("nan1", 0.5, "nan0", 2.0 ** -24)]


def _put(vec, i, v):
    if isinstance(v, str):
        vec.view(np.uint16)[i] = NAN_BITS[int(v[3])]
    else:
        vec[i] = H(v)


def _anchor(h, var, b, level_cell, k):
    flat = h.reshape(h.shape[0], h.shape[1], -1)
    if var in V8:
        return flat[b, :, level_cell]
    return flat.reshape(h.shape[0], 3, h.shape[1] // 3, -1)[b, k, :, level_cell]


def _nc(var):
    return V8[var][0] if var in V8 else 80


def _set_anchor(vec, var, classes, obj=3.0, box=None, extra=()):
    """Box, objectness and class logits of one anchor (classes past the variant's count are left out), and the first
    len(extra) channels after the classes: seg coefficients, pose keypoints (x, y, conf per point), the obb angle."""
    c0, nc = (4 if var in V8 else 5), _nc(var)
    box = box if box is not None else ((1.0, 1.5, 2.0, 2.5) if var in V8 else (0.25, -0.5, 0.75, 0.125))
    for i, v in enumerate(box):
        _put(vec, i, v)
    if c0 == 5:
        _put(vec, 4, obj)
    vec[c0:c0 + nc] = H(-8.0)
    for c, v in classes.items():
        if c < nc:
            _put(vec, c0 + c, v)
    for i, v in enumerate(extra):
        _put(vec, c0 + nc + i, v)


def _plant(h16, var, cases):
    """Each case on one anchor of image 0's largest level and one of image 1's smallest level (lanes, tiles and the three
    anchors k spread)."""
    g = _grids(h16)
    big, small = int(np.argmax(g)), int(np.argmin(g))
    for i, case in enumerate(cases):
        for b, l, cell in ((0, big, 3 + 97 * i), (1, small, 1 + 9 * i)):
            assert cell < g[l]
            _set_anchor(_anchor(h16[l], var, b, cell, (i + b) % 3), var, **case)


SPECIALS = (NAN, INF, -INF, -0.0, 65504.0, -65504.0, 2.0 ** -24, "nan1")
# pose keypoint (x, y, conf) logits; the default box holds a keypoint at x = y = 0
KPT_CASES = [(0.0, 0.0, NAN), (0.0, 0.0, INF), (0.0, 0.0, -INF), (NAN, 0.0, 2.0), (0.0, INF, 2.0), (-0.0, -0.0, 2.0),
             (0.0, 0.0, 65504.0), (0.0, 0.0, -65504.0), (65504.0, 0.0, 2.0), (0.0, "nan1", 2.0),
             (2.0 ** -24, -(2.0 ** -24), "nan0")]


def _extra_cases(var):
    if var in ("seg", "v5seg"):   # 32 mask coefficients, copied as they are
        return [[SPECIALS[(i + r) % len(SPECIALS)] for i in range(32)] for r in range(len(SPECIALS))]
    if var == "obb":              # the angle logit
        return [[s] for s in SPECIALS]
    # pose: one (x, y, conf) for all 17 points, then every case on a point of its own
    return [list(t) * 17 for t in KPT_CASES] + [[v for k in range(17) for v in KPT_CASES[k % len(KPT_CASES)]]]


def _edge_cases(group, var):
    passing = {min(5, _nc(var) - 1): 2.0}
    if group == "class":
        return [dict(classes=c) for c in CLASS_CASES]
    if group == "objectness":
        return [dict(obj=o, classes=c) for o, c in OBJ_CASES]
    if group == "extras":
        return [dict(classes=passing, extra=e) for e in _extra_cases(var)]
    return [dict(classes=passing, box=bx) for bx in BOX_CASES]


def _same_bits(a, b, nan_payloads):
    """Bit-identical; with nan_payloads, a NaN matches any NaN (fp16 widening of a raw-copied NaN may or may not keep its
    payload) and everything else bit for bit."""
    if not nan_payloads:
        return _bits_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


@pytest.mark.parametrize("var,group", [("v8", "class"), ("v8", "box")] +
                         [(v, g) for v in ("v5", "v7", "v3", *V3F) for g in ("class", "objectness", "box")] +
                         [(v, g) for v in ("seg", "pose", "obb") for g in ("class", "box", "extras")] +
                         [("v5seg", "objectness"), ("v5seg", "extras")])
def test_non_finite_and_edge_logits(oracle, dev, var, group):
    """NaN, +-inf, -0.0, saturating and underflowing logits, fp16 extremes, subnormals and NaN payloads in class,
    objectness and box rows, and in the extra channels the pack kernel gathers (seg coefficients, pose keypoints against
    the keypoint threshold, the obb angle).  A NaN objectness passes the objectness gate as `box_prob < kIgnoreThresh`
    lets it (its row carries a NaN confidence); NaN class logits never win a class.  Every route gives the same bytes
    (NaN for NaN where an extra is copied raw); the oracle agrees with NaNs at the same places, the reference's kernels
    bit for bit in the scan's columns; and with a capacity of 30 rows the same first 30 rows are kept as the oracle
    keeps."""
    B = 2
    h16 = _heads16(var, B, seed=800 + len(var) + len(group), n_obj=8)
    _plant(h16, var, _edge_cases(group, var))
    grids = _grids(h16)
    wide = [h.astype(np.float32) for h in h16]
    extras = var in ("seg", "pose", "obb", "v5seg")
    first = None
    for route, (dtype, off) in ROUTES.items():
        vec = _expect_vec(var, grids, dtype, off)
        hd = _place(_route_heads(h16, dtype), dtype, off, dev)
        for pair in ((None,) if var not in V8 else ((0, 0), (1, 8), (2, 5), (8, 10))):
            plug = _plugin(var, dtype)
            if pair:
                plug.tune(slices=pair[0], rows=pair[1])
            got = _decode(plug, hd, B, dev, vec, grids)
            first = got if first is None else first
            assert _same_bits(got, first, extras), (route, pair)
    ref, _ = _oracle(oracle, var, wide)
    _check_oracle(var, first, ref)
    if group in ("class", "objectness"):
        assert np.isnan(first[:, 1:].reshape(B, 1000, DET[var])[:, :, 4]).any() == (group == "objectness")
    _vs_ref(f"scan_edges.{var}.{group}", var, first, _ref_decode(var, wide, dev))
    small, _ = _oracle(oracle, var, wide, max_out=30)
    plug = _plugin(var, torch.float32, max_out=30)
    _check_oracle(var, _decode(plug, _place(wide, torch.float32, 0, dev), B, dev, _expect_vec(var, grids, torch.float32, 0),
                               grids), small, max_out=30)


# ------------------------------------------------------------------ gate window and near-ulp collisions ----------
def _ulps(x, k):
    x = np.float32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return x


def _gate_values():
    """Logits within +-64 ulps of logf(0.1f / 0.9f), then x_lo = that - 0.05f and one ulp either side."""
    x0 = np.float32(np.log(np.float64(np.float32(0.1) / np.float32(0.9))))
    x_lo = np.float32(x0 - np.float32(0.05))
    return [_ulps(x0, k) for k in range(-64, 65)] + [_ulps(x_lo, k) for k in (-1, 0, 1)]


def _collision_classes():
    """Near-ulp pairs (tests/test_vs_reference_gpu.py::test_yolov8_near_ulp_sigmoid_collisions_vs_reference_kernel):
    class 60 holds x, class 60-k the value k ulps below it (the earlier class wins if their sigmoids round together), class
    70 the same value (a later class never wins)."""
    out = []
    for x0 in (0.3, 1.5, 2.75, 5.0, 9.0, 14.0):
        for k in range(1, 25):
            y = _ulps(x0, -k)
            out.append({60 - k: y, 60: np.float32(x0), 70: y})
    return out


def _logist_split_pairs(n=24):
    """Logit pairs (y, x), y 1 to 8 ulps below x, on which the family's two Logist forms (float: yolov3, yolov3-tiny;
    double: yolov4, scaled-yolov4), as the oracle evaluates them with glibc expf, disagree about a collision: n whose
    probabilities round together under the double form only, then n under the float form only, at most one of each per x
    so that they spread over x from 0.3 up (to about 4.6).  CUDA expf may round otherwise, so the drivers' kernels decide
    these on the device."""
    kinds = {True: [], False: []}   # True: the double form collides
    for i in range(200):
        x = np.float32(0.3 + 0.0587 * i)
        found = set()
        for k in range(1, 9):
            y = _ulps(x, -k)
            c64, c32 = _sig(y, True) == _sig(x, True), _sig(y, False) == _sig(x, False)
            if c64 != c32 and c64 not in found and len(kinds[c64]) < n:
                kinds[c64].append((y, x))
                found.add(c64)
    return kinds[True], kinds[False]


def _plant32(heads, var, cases):
    """fp32 cases, one anchor each on image 0's largest level; every other objectness and class logit is -9 (no other
    anchor passes)."""
    g = _grids(heads)
    big = int(np.argmax(g))
    c0 = 4 if var in V8 else 5
    for h in heads:
        if var in V8:
            h[:, 4:] = np.float32(-9.0)
        else:
            h.reshape(h.shape[0], 3, h.shape[1] // 3, -1)[:, :, 4:] = np.float32(-9.0)
    for i, (obj, classes) in enumerate(cases):
        cell = 5 + 11 * i
        assert cell < g[big]
        vec = _anchor(heads[big], var, 0, cell, i % 3)
        vec[c0:c0 + 80] = np.float32(-9.0)
        if c0 == 5:
            vec[4] = np.float32(obj)
        for c, v in classes.items():
            vec[c0 + c] = v


@pytest.mark.parametrize("var", ["v8", "v5", "v7", "v3", *V3F])
def test_gate_window_and_near_ulp_collisions_vs_reference_kernel(oracle, dev, var):
    """Whether Logist(x) reaches 0.1f, and whether two logits a few ulps apart round to one probability, depends on CUDA
    expf: only the reference's kernels arbitrate.  The gate window is on the class maximum (v8), the objectness (v5, v7)
    and both (v3 and its family); the collision pairs sit in the class rows, and for the family also the pairs on which
    its float and double Logist disagree (the earlier class wins only where this driver's form collides).  fp32 heads,
    VEC 4 and VEC 1; every pair for v8."""
    B = 1
    heads = [h.astype(np.float32) for h in _heads16(var, B, seed=850 + len(var), n_obj=0)]
    win = _gate_values()
    cases = []
    if var in V8:   # window classes stay below 30, so classes 36..60 come from the collision pairs only
        cases += [(None, {i % 30: x}) for i, x in enumerate(win)]
    else:
        cases += [(x, {i % 30: np.float32(2.0)}) for i, x in enumerate(win)]
        if var == "v3" or var in V3F:
            cases += [(np.float32(3.0), {i % 30: x}) for i, x in enumerate(win)]
    cases += [(np.float32(3.0), c) for c in _collision_classes()]
    if var in V3F:
        dbl, flt = _logist_split_pairs()
        assert len(dbl) == len(flt) == 24   # both kinds, as the oracle's two forms judge them
        # the earlier class in slices 0 and 1 (below the collision pairs' 36..60), the later one in slice 3
        cases += [(np.float32(3.0), {(7 * j) % 36: y, 75: x}) for j, (y, x) in enumerate(dbl + flt)]
    _plant32(heads, var, cases)
    grids = _grids(heads)
    ref = _ref_decode(var, heads, dev)
    key = f"scan_gate_ulp.{var}"
    for route in ("f32", "f32+4"):
        dtype, off = ROUTES[route]
        hd = _place(heads, dtype, off, dev)
        for pair in (PAIRS if var in V8 else (None,)):
            plug = _plugin(var, dtype)
            if pair:
                plug.tune(slices=pair[0], rows=pair[1])
            got = _decode(plug, hd, B, dev, _expect_vec(var, grids, dtype, off), grids)
            _vs_ref(key, var, got, ref)
    # the window really straddles the gate, and both collision outcomes occur (judged by the oracle's glibc expf)
    orc, idx = _oracle(oracle, var, heads)
    big = int(np.argmax(grids))
    level_off = sum(grids[:big]) * (1 if var in V8 else 3)
    apc = 1 if var in V8 else 3
    ids = {level_off + (5 + 11 * i) * apc + (0 if var in V8 else i % 3) for i in range(len(win))}
    kept = set(idx[0, :int(orc[0, 0])].tolist())
    assert 0 < len(ids & kept) < len(ids)
    g = _canon(got, 0, var)
    assert (g[:, 5] == 60).any() and ((g[:, 5] > 35) & (g[:, 5] < 60)).any()


# ------------------------------------------------------------------ class-slice edges ----------------------------
def _slice_cases(bounds, base=2.5):
    """At each class-slice boundary c: an exact tie across it, saturated collisions both ways, a tie inside the later
    slice that beats the earlier one, and -0.0 / +0.0 -- all decided without expf (ties, or sigmoid == 1.0f)."""
    cases = []
    for c in bounds:
        cases += [{c - 1: base, c: base}, {c - 1: 18.0, c: 25.0}, {c - 1: 25.0, c: 18.0},
                  {c - 1: 1.0, c: 3.0, c + 1: 3.0}, {c - 1: -0.0, c: 0.0}, {c - 2: 17.0, c - 1: 16.0, c: INF}]
    return [dict(classes=x) for x in cases]


@pytest.mark.parametrize("var", ["v8", "v5", *V3F])
def test_class_slice_boundaries_on_every_pair(oracle, dev, var):
    """Ties and collisions on both sides of every class-slice boundary of every built pair (v8: 80 classes in 1, 2, 4 or
    8 slices; v5 and the yolov3 family: 4 slices of 20), every route, against the oracle and byte-identical across pairs
    and routes; the family also against its driver's own kernel."""
    B = 2
    h16 = _heads16(var, B, seed=870 + len(var), n_obj=8)
    bounds = range(10, 80, 10) if var == "v8" else (20, 40, 60)
    _plant(h16, var, _slice_cases(bounds))
    grids = _grids(h16)
    first = None
    for route, (dtype, off) in ROUTES.items():
        hd = _place(_route_heads(h16, dtype), dtype, off, dev)
        for pair in (PAIRS if var in V8 else (None,)):
            plug = _plugin(var, dtype)
            if pair:
                plug.tune(slices=pair[0], rows=pair[1])
            got = _decode(plug, hd, B, dev, _expect_vec(var, grids, dtype, off), grids)
            first = got if first is None else first
            assert _bits_equal(got, first), (route, pair)
    wide = [h.astype(np.float32) for h in h16]
    ref, _ = _oracle(oracle, var, wide)
    _check_oracle(var, first, ref)
    if var in V3F:
        _vs_ref(f"scan_slices.{var}", var, first, _ref_decode(var, wide, dev))


@pytest.mark.parametrize("nc", [1, 3, 5])
@pytest.mark.parametrize("var", ["v8", "v5", *V3F])
def test_fewer_classes_than_slices(oracle, dev, var, nc):
    """nc below the slice count (v8 at 8 slices, v5's and the yolov3 family's 4): warps with no class rows must not disturb
    the others; every pair, every route, against the oracle; the family also against its driver's own kernel, whose blob
    carries the class count."""
    B = 2
    h16 = _heads16(var, B, seed=890 + nc, nc=nc, n_obj=40)
    grids = _grids(h16)
    first = None
    for route, (dtype, off) in ROUTES.items():
        hd = _place(_route_heads(h16, dtype), dtype, off, dev)
        for pair in (PAIRS if var in V8 else (None,)):
            plug = _plugin(var, dtype, nc=nc)
            if pair:
                plug.tune(slices=pair[0], rows=pair[1])
            got = _decode(plug, hd, B, dev, _expect_vec(var, grids, dtype, off), grids)
            first = got if first is None else first
            assert _bits_equal(got, first), (route, pair)
    wide = [h.astype(np.float32) for h in h16]
    ref, _ = _oracle(oracle, var, wide, nc=nc)
    assert ref[:, 0].min() > 10
    _check_oracle(var, first, ref)
    if var in V3F:
        _vs_ref(f"scan_fewer.{var}.nc{nc}", var, first, _ref_decode(var, wide, dev, nc=nc))
