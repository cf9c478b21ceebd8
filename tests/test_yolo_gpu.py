"""Parity of the YoloLayer scan / pack / NMS kernels against the CPU oracle, through the C ABI
(tensorrtx_b200.plugins forwards to libtrtx_hot.so).  Tolerances: boxes/scores abs 1e-4
(BASELINE.json north_star), counts / classes / kept-index sets exact."""
import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
ATOL = 1e-4
# v5 / retinaface boxes pass through expf(): the oracle uses glibc expf, the kernels CUDA expf (<= 2 ulp), and the
# result is scaled by up to ~1500 px, so those columns get a relative slack of 16 fp32 ulps on top of ATOL.
RTOL_EXP = 2e-6


def _to_dev(heads, dev, dtype=torch.float32):
    return [torch.from_numpy(h).to(dev).to(dtype).contiguous() for h in heads]


def _decode_gpu(plug, heads_dev, B, dev):
    out = torch.full((B, plug.output_elems()), -123.0, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, heads_dev, [out], ws) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _check_rows(got, ref, B, F, ncols, max_out, rtol=0.0):
    assert np.array_equal(np.minimum(ref[:, 0], max_out), got[:, 0])
    for b in range(B):
        n = int(got[b, 0])
        g = got[b, 1:1 + n * F].reshape(n, F)[:, :ncols]
        r = ref[b, 1:1 + n * F].reshape(n, F)[:, :ncols]
        np.testing.assert_allclose(g, r, atol=ATOL, rtol=rtol)
        assert np.array_equal(g[:, 5], r[:, 5])  # class ids exact


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 4), (2, 5)])
def test_v8_decode_parity(oracle, dev, seed, B):
    heads = synth.yolov8_heads(B, seed=seed)
    ref, _ = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    got = _decode_gpu(plug, _to_dev(heads, dev), B, dev)
    assert ref[:, 0].min() > 100  # the synthetic set really has candidates
    _check_rows(got, ref, B, 90, 6, 1000)


def test_v8_decode_empty_and_overflow(oracle, dev):
    # empty: background only
    heads = synth.yolov8_heads(2, seed=5, n_obj=0)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    got = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    ref, _ = oracle.yolov8_decode(heads)
    assert np.array_equal(got[:, 0], ref[:, 0])
    # overflow: ~3000 candidates / image, capacity 1000 -> first 1000 in anchor order, count clamped
    heads = synth.yolov8_heads(2, seed=6, n_obj=220)
    ref, _ = oracle.yolov8_decode(heads)
    assert ref[:, 0].min() > 1000
    got = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    _check_rows(got, ref, 2, 90, 6, 1000)
    # determinism: identical bytes on a second run
    got2 = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    assert np.array_equal(got[:, :1 + 1000 * 90].reshape(2, -1)[:, 0], got2[:, 0])
    for b in range(2):
        a = got[b, 1:].reshape(1000, 90)[:, :6]
        c = got2[b, 1:].reshape(1000, 90)[:, :6]
        assert np.array_equal(a, c)


def test_v8_scalar_path_odd_grid(oracle, dev):
    # 648x648 -> grids 81^2, 40^2 (648/16=40.5 -> 40), 20^2: level 0 has an odd cell count -> scalar kernels
    net = 648
    strides = (8, 16, 32)
    heads = synth.yolov8_heads(3, seed=7, net_w=net, net_h=net, strides=strides)
    ref, _ = oracle.yolov8_decode(heads, strides=strides, net_w=net, net_h=net)
    plug = P.YoloLayerPlugin(80, 17, 0.0, net, net, 1000, False, False, False, strides)
    got = _decode_gpu(plug, _to_dev(heads, dev), 3, dev)
    _check_rows(got, ref, 3, 90, 6, 1000)


def test_v8_nonsquare_and_classes(oracle, dev):
    heads = synth.yolov8_heads(2, seed=8, nc=15, net_w=1024, net_h=576, strides=(8, 16, 32))
    ref, _ = oracle.yolov8_decode(heads, net_w=1024, net_h=576, nc=15)
    plug = P.YoloLayerPlugin(15, 17, 0.0, 1024, 576, 1000, False, False, False, (8, 16, 32))
    got = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    _check_rows(got, ref, 2, 90, 6, 1000)


@pytest.mark.parametrize("mode", ["seg", "pose", "obb"])
def test_v8_extras(oracle, dev, mode):
    seg, pose, obb = mode == "seg", mode == "pose", mode == "obb"
    nc = 1 if pose else (15 if obb else 80)
    extra = 32 if seg else (51 if pose else 1)
    heads = synth.yolov8_heads(2, seed=9, nc=nc, extra=extra, n_obj=20)
    kt = 0.3
    ref, _ = oracle.yolov8_decode(heads, nc=nc, is_seg=seg, is_pose=pose, is_obb=obb, kpt_thresh=kt)
    plug = P.YoloLayerPlugin(nc, 17, kt, 640, 640, 1000, seg, pose, obb, (8, 16, 32))
    got = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    assert np.array_equal(got[:, 0], ref[:, 0])
    for b in range(2):
        n = int(got[b, 0])
        g = got[b, 1:1 + n * 90].reshape(n, 90)
        r = ref[b, 1:1 + n * 90].reshape(n, 90)
        cols = list(range(6))
        if seg:
            cols += list(range(6, 38))
        if pose:
            cols += list(range(38, 89))
        if obb:
            cols += [89]
        np.testing.assert_allclose(g[:, cols], r[:, cols], atol=ATOL, rtol=0)


def test_v8_fp16_inputs(oracle, dev):
    heads = [h.astype(np.float16).astype(np.float32) for h in synth.yolov8_heads(2, seed=10)]  # fp16-representable
    ref, _ = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32), in_dtype=L.F16)
    got = _decode_gpu(plug, _to_dev(heads, dev, torch.float16), 2, dev)
    _check_rows(got, ref, 2, 90, 6, 1000)


@pytest.mark.parametrize("slices,unroll", [(1, 8), (1, 16), (2, 4), (2, 8), (2, 10), (2, 20), (4, 4), (4, 5), (4, 10), (4, 20), (8, 5), (8, 10)])
def test_v8_all_register_scan_variants(oracle, dev, slices, unroll):
    heads = synth.yolov8_heads(2, seed=11)
    ref, _ = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)).tune(slices=slices, rows=unroll)
    got = _decode_gpu(plug, _to_dev(heads, dev), 2, dev)
    _check_rows(got, ref, 2, 90, 6, 1000)


@pytest.mark.parametrize("slices,unroll", [(1, 8), (2, 5), (2, 10), (4, 5), (4, 20), (8, 10)])
@pytest.mark.parametrize("B,n_obj", [(2, 64), (5, 200)])
def test_v8_fp16_eight_anchors_per_lane_scan(oracle, dev, slices, unroll, B, n_obj):
    """fp16 inputs take the 8-anchors-per-lane scan (16-byte loads, packed half2 running maxima, exact per-anchor replay in
    fp32): every built (slices, rows) pair on fp16-representable heads against the fp32 oracle, including dense images
    (n_obj = 200: most groups of rows raise some anchor) and exact ties between halfs."""
    heads = [h.astype(np.float16).astype(np.float32) for h in synth.yolov8_heads(B, seed=17 + B, n_obj=n_obj)]
    heads[0][0, 4 + 11, 300] = 3.5
    heads[0][0, 4 + 70, 300] = 3.5          # exact tie: the first class wins
    heads[1][B - 1, 4 + 3, 8] = 12.0        # saturating sigmoids in fp32: collision replay
    heads[1][B - 1, 4 + 2, 8] = 11.5
    ref, _ = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32), in_dtype=L.F16).tune(slices=slices, rows=unroll)
    got = _decode_gpu(plug, _to_dev(heads, dev, torch.float16), B, dev)
    _check_rows(got, ref, B, 90, 6, 1000)


def test_v8_unbuilt_tuning_is_refused_and_tunings_are_per_plugin(oracle, dev):
    """trtx_yolo_params.tune_* is per-call data: a pair that is not built -> TRTX_ERR_UNSUPPORTED (no silent default),
    and two plugins with different tunings used alternately give the same (oracle) rows -- no shared state."""
    heads = synth.yolov8_heads(2, seed=14)
    hd = _to_dev(heads, dev)
    ref, _ = oracle.yolov8_decode(heads)
    bad = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)).tune(slices=3, rows=7)
    out = torch.zeros((2, bad.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(bad.getWorkspaceSize(2), dtype=torch.uint8, device=dev)
    assert bad.enqueue(2, hd, [out], ws) == L.ERR_UNSUPPORTED
    a = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)).tune(slices=4, rows=10, box=3)
    b = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)).tune(slices=2, rows=5, box=1)
    for plug in (a, b, a, b):
        _check_rows(_decode_gpu(plug, hd, 2, dev), ref, 2, 90, 6, 1000)


def test_first_argmax_on_sigmoid_collisions(oracle, dev):
    # saturating logits: sigmoid(18) == sigmoid(25) == 1.0f -> the reference keeps the FIRST class
    heads = synth.yolov8_heads(1, seed=12, n_obj=0)
    h = heads[0]
    h[0, 4 + 7, 100] = 25.0
    h[0, 4 + 3, 100] = 18.0   # earlier class, smaller logit, same sigmoid
    h[0, 4 + 50, 200] = 6.0000
    h[0, 4 + 20, 200] = 6.0000  # exact tie -> first class wins
    ref, _ = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    for slices, unroll in ((2, 5), (4, 10), (1, 8)):
        plug.tune(slices=slices, rows=unroll)
        got = _decode_gpu(plug, _to_dev(heads, dev), 1, dev)
        assert got[0, 0] == ref[0, 0] == 2
        g = got[0, 1:181].reshape(2, 90)
        assert g[0, 5] == 3 and g[1, 5] == 20
        _check_rows(got, ref, 1, 90, 6, 1000)


# ------------------------------------------------------------------ NMS ------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_batch_nms_matches_reference_nms(oracle, dev, seed):
    B = 3
    heads = synth.yolov8_heads(B, seed=20 + seed)
    ref, _ = oracle.yolov8_decode(heads)
    comp, idx = P.batch_nms(torch.from_numpy(ref).to(dev), B, ref.shape[1], 0.5, 0.45, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(0, ref[b], 1000, 90, 0.5, 0.45)
        n = int(comp[b, 0])
        assert n == len(res) and n > 20
        assert np.array_equal(idx[b, :n], src)            # identical kept rows, identical (class, conf) order
        rows = comp[b, 1:1 + n * 7].reshape(n, 7)
        assert np.array_equal(rows[:, :6], res[:, :6])    # rows are copies: bit-exact
        assert np.all(rows[:, 6] == 1)
        assert np.all(comp[b, 1 + n * 7:] == 0)


def test_fused_decode_nms(oracle, dev):
    B = 4
    heads = synth.yolov8_heads(B, seed=30)
    ref, ref_idx = oracle.yolov8_decode(heads)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    fused = P.FusedYoloDecodeNms(plug, B, 0.5, 0.45, device=dev)
    comp, idx = fused.enqueue(B, _to_dev(heads, dev))
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(0, ref[b], 1000, 90, 0.5, 0.45)
        n = int(comp[b, 0])
        assert n == len(res)
        assert np.array_equal(idx[b, :n], ref_idx[b][src])  # identical kept ANCHOR ids
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=0)


def test_nms_dense_single_class_and_ties(oracle, dev):
    # all candidates in one class, heavy overlap, duplicated confidences (ties broken by box[0], then row)
    rng = np.random.default_rng(5)
    n = 1000
    buf = np.zeros((1, 1 + n * 90), np.float32)
    rows = buf[0, 1:].reshape(n, 90)
    cx, cy = rng.uniform(100, 540, n), rng.uniform(100, 540, n)
    w, h = rng.uniform(40, 200, n), rng.uniform(40, 200, n)
    rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3] = cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2
    rows[:, 4] = np.round(rng.uniform(0.3, 1.0, n), 2)   # many exact ties
    rows[:, 5] = 3
    buf[0, 0] = n
    comp, idx = P.batch_nms(torch.from_numpy(buf).to(dev), 1, buf.shape[1], 0.5, 0.45, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    res, src = oracle.nms(0, buf[0], n, 90, 0.5, 0.45)
    k = int(comp[0, 0])
    assert k == len(res)
    assert np.array_equal(idx[0, :k], src)


def test_nms_class_segments_of_65_to_96_rows(oracle, dev):
    """Class segments of 65..96 rows take the 3-chunk bitmap resolve of nms_kernel phase E (a warp walks three 32-row
    chunks, later chunks see the kept rows of earlier ones); the synthetic detector sets top out near 47 rows per class.
    Plugin rows built directly: 12 classes with 65, 66, 72, 80, 88, 95, 96 ... rows each, in overlapping clusters so that
    suppression chains cross chunk boundaries; also one 97-row class (long-segment path) and one 33-row class."""
    rng = np.random.default_rng(91)
    sizes = [65, 66, 72, 80, 88, 95, 96, 96, 70, 90, 97, 33]
    B, F = 2, 90
    buf = np.zeros((B, 1 + 1000 * F), np.float32)
    for b in range(B):
        rows = []
        for cls, m in enumerate(sizes):
            centres = rng.uniform(80, 560, (6, 2))                     # 6 clusters per class
            for i in range(m):
                c = centres[rng.integers(0, 6)] + rng.normal(0, 6, 2)
                wh = rng.uniform(40, 90, 2)
                rows.append([c[0] - wh[0] / 2, c[1] - wh[1] / 2, c[0] + wh[0] / 2, c[1] + wh[1] / 2,
                             rng.uniform(0.51, 0.99), float(cls * 3 + b)])
        rows = np.asarray(rows, np.float32)
        rows = rows[rng.permutation(len(rows))]                        # arrival order is arbitrary in the reference
        buf[b, 0] = len(rows)
        buf[b, 1:1 + len(rows) * F].reshape(-1, F)[:, :6] = rows
    comp, idx = P.batch_nms(torch.from_numpy(buf).to(dev), B, buf.shape[1], 0.5, 0.45, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(0, buf[b], 1000, F, 0.5, 0.45)
        n = int(comp[b, 0])
        assert n == len(res) and 60 < n < 400
        assert np.array_equal(idx[b, :n], src)
        assert np.array_equal(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6])


def test_nms_empty_and_below_threshold(oracle, dev):
    buf = np.zeros((2, 1 + 1000 * 90), np.float32)
    buf[1, 0] = 3
    buf[1, 1:1 + 3 * 90].reshape(3, 90)[:, 4] = 0.4  # all below conf 0.5
    comp = P.batch_nms(torch.from_numpy(buf).to(dev), 2, buf.shape[1], 0.5, 0.45).cpu().numpy()
    assert np.all(comp == 0)


def test_nms_oneshot_mode(oracle, dev):
    heads = synth.yolov8_heads(1, seed=40)
    ref, _ = oracle.yolov8_decode(heads)
    comp, idx = P.batch_nms(torch.from_numpy(ref).to(dev), 1, ref.shape[1], 0.5, 0.45, mode=L.NMS_ONESHOT,
                            return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    exp = oracle.cuda_decode_nms(ref[0], 1000, 90, 0.5, 0.45, 1000)
    n = int(comp[0, 0])
    rows = comp[0, 1:1 + n * 7].reshape(n, 7)
    exp_rows = exp[1:].reshape(1000, 7)
    exp_valid = {i for i in range(int(exp[0])) if exp_rows[i, 4] > 0}
    assert set(idx[0, :n].tolist()) == exp_valid
    kept_gpu = {int(idx[0, i]) for i in range(n) if rows[i, 6] == 1}
    kept_ref = {i for i in exp_valid if exp_rows[i, 6] == 1}
    assert kept_gpu == kept_ref


def _obb_rows(oracle, seed, B):
    heads = synth.yolov8_heads(B, seed=seed, nc=15, extra=1, n_obj=40)
    out, _ = oracle.yolov8_decode(heads, nc=15, is_obb=True)
    return out


@pytest.mark.parametrize("thr", [0.5, 0.2])
def test_batch_nms_obb_matches_reference_nms_obb(oracle, dev, thr):
    """Oriented boxes, greedy: nms_obb + probiou (yolov8/src/postprocess.cpp:303-385); the oracle is pinned bit for bit
    to the reference's own host code (tests/test_oracle_vs_ref_cpu.py::test_v8_nms_obb_equals_reference)."""
    B = 3
    ref = _obb_rows(oracle, 140, B)
    comp, idx = P.batch_nms_obb(torch.from_numpy(ref).to(dev), B, ref.shape[1], 0.3, thr, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(3, ref[b], 1000, 90, 0.3, thr)
        n = int(comp[b, 0])
        assert n == len(res) and 10 < n < int(ref[b, 0])
        assert np.array_equal(idx[b, :n], src)            # identical kept rows, identical (class, conf) order
        rows = comp[b, 1:1 + n * 8].reshape(n, 8)
        assert np.array_equal(rows[:, :6], res[:, :6])    # cx, cy, w, h, conf, cls: copies
        assert np.array_equal(rows[:, 7], res[:, 89])     # the angle rides along as the 8th float
        assert np.all(rows[:, 6] == 1) and np.all(comp[b, 1 + n * 8:] == 0)


def test_nms_obb_oneshot_mode(oracle, dev):
    """decode_kernel_obb + nms_kernel_obb semantics (postprocess.cu:7-40, 113-166) with 8-float elements.  (The
    reference strides its 8-float rows by bbox_element = 7, so its own GPU path lets neighbouring rows overwrite each
    other -- DESIGN.md section 2; the oracle restates the intended layout.)"""
    ref = _obb_rows(oracle, 141, 1)
    comp, idx = P.batch_nms_obb(torch.from_numpy(ref).to(dev), 1, ref.shape[1], 0.3, 0.3, mode=L.NMS_ONESHOT,
                                return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    exp = oracle.cuda_decode_nms_obb(ref[0], 1000, 90, 0.3, 0.3, 1000)
    n = int(comp[0, 0])
    rows = comp[0, 1:1 + n * 8].reshape(n, 8)
    exp_rows = exp[1:].reshape(1000, 8)
    exp_valid = {i for i in range(int(exp[0])) if exp_rows[i, 4] > 0}
    assert set(idx[0, :n].tolist()) == exp_valid and len(exp_valid) > 50
    kept_gpu = {int(idx[0, i]) for i in range(n) if rows[i, 6] == 1}
    kept_ref = {i for i in exp_valid if exp_rows[i, 6] == 1}
    assert kept_gpu == kept_ref and 5 < len(kept_ref) < len(exp_valid)
    for i in range(n):
        assert np.array_equal(rows[i, [0, 1, 2, 3, 4, 5, 7]], exp_rows[idx[0, i], [0, 1, 2, 3, 4, 5, 7]])


def test_overflow_fused_equals_two_stage_equals_oracle(oracle, dev):
    """More candidates than the plugin capacity (max_out): the reference plugin keeps the first max_out that grab a slot
    (yololayer.cu:206-208; ours: ascending anchor order) and nms() filters those.  The fused call, the two-stage call
    (plugin buffer -> batch_nms) and the oracle (decode with the same capacity -> nms) must give the same rows."""
    B = 2
    heads = synth.yolov8_heads(B, seed=41, n_obj=300)
    hd = _to_dev(heads, dev)
    ref, ref_idx = oracle.yolov8_decode(heads)
    assert ref[:, 0].min() > 1000
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    fused = P.FusedYoloDecodeNms(plug, B, 0.5, 0.45, device=dev)
    comp, idx = fused.enqueue(B, hd)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    two = P.batch_nms(out, B, plug.output_elems(), 0.5, 0.45).cpu().numpy()
    assert np.array_equal(two, comp)                      # identical bytes, both paths
    for b in range(B):
        one = ref[b].copy()
        one[0] = min(one[0], 1000)                        # the host reader must not run past the buffer (count is clamped)
        res, src = oracle.nms(0, one, 1000, 90, 0.5, 0.45)
        n = int(comp[b, 0])
        assert n == len(res) and n > 20
        assert np.array_equal(idx[b, :n], ref_idx[b][src])
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=0)


def test_nms_row_cap_above_2048_rows(oracle, dev):
    """trtx_nms_enqueue with max_rows > TRTX_NMS_MAX_ROWS (2048): the 2048 highest-confidence rows above conf_thresh enter
    NMS (documented in trtx_hot.h; the reference has no cap).  3000 rows above the threshold, distinct confidences."""
    rng = np.random.default_rng(77)
    n_rows, F = 3000, 15
    buf = np.zeros((1, 1 + n_rows * F), np.float32)
    buf[0, 0] = n_rows
    rows = buf[0, 1:].reshape(n_rows, F)
    cx, cy = rng.uniform(50, 590, n_rows), rng.uniform(50, 590, n_rows)
    w, h = rng.uniform(8, 60, n_rows), rng.uniform(8, 60, n_rows)
    rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3] = cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2
    rows[:, 4] = rng.permutation(n_rows).astype(np.float32) / n_rows * 0.8 + 0.15   # all > 0.1, distinct
    rows[:, 5:] = rng.standard_normal((n_rows, 10))
    top = np.sort(np.argsort(-rows[:, 4], kind="stable")[:2048])
    sub = np.zeros(1 + 2048 * F, np.float32)
    sub[0] = 2048
    sub[1:].reshape(2048, F)[:] = rows[top]
    res, src = oracle.nms(2, sub, 2048, F, 0.1, 0.4)
    comp, idx = P.batch_nms(torch.from_numpy(buf).to(dev), 1, buf.shape[1], 0.1, 0.4, det_floats=F, box_format=L.BOX_RETINA,
                            max_det=2048, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    n = int(comp[0, 0])
    assert n == len(res) and n > 100
    assert np.array_equal(idx[0, :n], top[src])


# ------------------------------------------------------------------ v5 -------------------------
def _v5_plugin(seg=False):
    ks = [P.YoloKernel(640 // s, 640 // s, a) for s, a in zip((8, 16, 32), synth.V5_ANCHORS)]
    return P.YoloLayerPluginV5(80, 640, 640, 1000, seg, ks)


@pytest.mark.parametrize("seed,B,seg", [(0, 1, False), (1, 3, False), (2, 2, True)])
def test_v5_decode_parity(oracle, dev, seed, B, seg):
    heads = synth.yolov5_heads(B, seed=50 + seed, seg=seg)
    ref, _ = oracle.yolov5_decode(heads, synth.V5_ANCHORS, is_seg=seg)
    plug = _v5_plugin(seg)
    got = _decode_gpu(plug, _to_dev(heads, dev), B, dev)
    assert ref[:, 0].min() > 100
    _check_rows(got, ref, B, 38, 38 if seg else 6, 1000, rtol=RTOL_EXP)


def test_v5_fused_nms(oracle, dev):
    B = 2
    heads = synth.yolov5_heads(B, seed=60)
    ref, ref_idx = oracle.yolov5_decode(heads, synth.V5_ANCHORS)
    fused = P.FusedYoloDecodeNms(_v5_plugin(), B, 0.5, 0.45, device=dev)
    comp, idx = fused.enqueue(B, _to_dev(heads, dev))
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(1, ref[b], 1000, 38, 0.5, 0.45)
        n = int(comp[b, 0])
        assert n == len(res)
        assert np.array_equal(idx[b, :n], ref_idx[b][src])
        np.testing.assert_allclose(comp[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=RTOL_EXP)


# ------------------------------------------------------------------ full size ------------------
def test_full_size_b32_properties(oracle, dev):
    """BASELINE configs[1] size: b32.  Size-independent properties + every image against the oracle."""
    B = 32
    heads = synth.yolov8_heads(B, seed=70)
    hd = _to_dev(heads, dev)
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    fused = P.FusedYoloDecodeNms(plug, B, 0.5, 0.45, device=dev)
    comp, idx = fused.enqueue(B, hd)
    comp, idx = comp.clone(), idx.clone()
    # determinism / idempotence of the whole path
    comp2, idx2 = fused.enqueue(B, hd)
    assert torch.equal(comp, comp2) and torch.equal(idx, idx2)
    c = comp.cpu().numpy()
    counts = c[:, 0].astype(int)
    assert counts.min() > 20 and counts.max() <= 1000
    # NMS of the NMS output is the identity (kept rows never suppress each other)
    again = P.batch_nms(comp.contiguous(), B, comp.shape[1], 0.5, 0.45, det_floats=7, max_det=1000).cpu().numpy()
    assert np.array_equal(again[:, 0], c[:, 0])
    # rows sorted by (class asc, conf desc); anchors unique
    ii = idx.cpu().numpy()
    for b in range(B):
        n = counts[b]
        rows = c[b, 1:1 + n * 7].reshape(n, 7)
        key = list(zip(rows[:, 5], -rows[:, 4]))
        assert key == sorted(key)
        assert len(set(ii[b, :n].tolist())) == n
    # every image against the oracle
    for b in range(B):
        one = [h[b:b + 1] for h in heads]
        ref, ref_idx = oracle.yolov8_decode(one)
        res, src = oracle.nms(0, ref[0], 1000, 90, 0.5, 0.45)
        assert counts[b] == len(res)
        assert np.array_equal(ii[b, :counts[b]], ref_idx[0][src])
