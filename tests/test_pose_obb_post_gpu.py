"""Pose and oriented-box post-process on the GPU (trtx_yolo_pose_obb_postprocess_enqueue) against the library's host
functions applied row by row -- trtx_get_rect_adapt_landmark and trtx_get_corner, which tests/test_pose_obb_post_cpu.py pins
to the reference's compiled draw_bbox_keypoints_line and draw_bbox_obb.  The comparison is exact: the device's double cos /
sin are not correctly rounded, so a corner could in principle differ from glibc's; any mismatch is printed with its angle."""
import ctypes as C

import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
F = np.float32
SENTINEL = -7.0
MIXED = [(1920, 1080), (1080, 1920), (1280, 720), (640, 480), (333, 1001), (640, 640), (5000, 20), (17, 3000)]
POSE_R, OBB_R = 58, 8


def _keep_flag(v):
    return 1.0 <= v < 2.0   # (int)v == 1


def host_rows(task, dets_b, img_w, img_h, K, R, off=7, nk=17, net=640):
    """The expected output of one frame: the host functions on the kept rows of the first min(count, K), input order."""
    lib = L.load()
    n = min(max(int(dets_b[0]), 0), K)
    src = dets_b[1:1 + K * R].reshape(K, R)
    Fo = 6 + 3 * nk if task == L.TASK_POSE else 10
    out = np.zeros((K, Fo), F)
    m = 0
    for i in range(n):
        r = src[i]
        if not _keep_flag(r[6]):
            continue
        bb = (C.c_float * 4)(*[float(v) for v in r[:4]])
        if task == L.TASK_POSE:
            k = np.ascontiguousarray(r[off:off + 3 * nk], F).copy()
            rect = (C.c_int * 4)()
            lib.trtx_get_rect_adapt_landmark(net, net, img_w, img_h, bb, k.ctypes.data_as(C.POINTER(C.c_float)), nk, rect)
            out[m, :4], out[m, 4:6], out[m, 6:] = list(rect), r[4:6], k
        else:
            c = (C.c_int * 8)()
            lib.trtx_get_corner(net, net, img_w, img_h, bb, float(r[off]), c)
            out[m, :8], out[m, 8:10] = list(c), r[4:6]
        m += 1
    return m, out


def check(task, got, dets, sizes, K, R, off=7, nk=17, net=640):
    """Exact comparison of every frame; mismatching OBB rows are printed with their angle before failing."""
    rows = 0
    for b, (w, h) in enumerate(sizes):
        m, want = host_rows(task, dets[b], w, h, K, R, off, nk, net)
        g = got[b, 1:].reshape(K, -1)
        assert got[b, 0] == m, (b, got[b, 0], m)
        bad = [i for i in range(K) if not np.array_equal(g[i], want[i], equal_nan=True)]
        if bad and task == L.TASK_OBB:
            src = dets[b, 1:1 + K * R].reshape(K, R)
            kept = [i for i in range(min(max(int(dets[b, 0]), 0), K)) if _keep_flag(src[i, 6])]
            for i in bad:
                s = src[kept[i]] if i < len(kept) else None
                print(f"frame {b} ({w}x{h}) row {i}: angle {None if s is None else repr(s[off])} box "
                      f"{None if s is None else s[:4].tolist()} device {g[i].tolist()} host {want[i].tolist()}")
        assert not bad, (b, bad[:10])
        rows += m
    return rows


def pose_dets(rng, B, K, counts, keep_p=1.0):
    d = np.zeros((B, 1 + K * POSE_R), F)
    for b in range(B):
        d[b, 0] = counts[b]
        r = d[b, 1:].reshape(K, POSE_R)
        x, y = rng.uniform(-60, 660, K), rng.uniform(-60, 660, K)
        r[:, :4] = np.stack([x, y, x + rng.uniform(0, 300, K), y + rng.uniform(0, 300, K)], 1)
        r[:, 4], r[:, 5] = rng.uniform(0.5, 1, K), 0
        r[:, 6] = np.where(rng.uniform(0, 1, K) < keep_p, 1.0, 0.0)
        r[:, 7:] = rng.uniform(-80, 720, (K, 51))
        r[:, 9::3] = rng.uniform(0, 1, (K, 17))
        r[:3, 0] = [np.nan, np.inf, 3e9]            # undefined rectangles
        r[3, 8] = np.nan                            # a NaN keypoint
        r[4, 6], r[5, 6] = 1.5, np.nan              # (int)1.5 == 1 is kept, NaN is not
    return d


def obb_dets(rng, B, K, counts, net, keep_p=1.0):
    d = np.zeros((B, 1 + K * OBB_R), F)
    for b in range(B):
        d[b, 0] = counts[b]
        r = d[b, 1:].reshape(K, OBB_R)
        r[:, 0:2] = rng.uniform(-0.1 * net, 1.1 * net, (K, 2))
        r[:, 2:4] = rng.uniform(1, 0.5 * net, (K, 2))
        r[:, 4], r[:, 5] = rng.uniform(0.3, 1, K), rng.integers(0, 15, K)
        r[:, 6] = np.where(rng.uniform(0, 1, K) < keep_p, 1.0, 0.0)
        r[:, 7] = rng.uniform(-np.pi / 2, np.pi, K)
        r[:8, 7] = [0, np.pi / 2, -np.pi / 2, np.nan, np.inf, np.pi, 1e-30, -0.0]
        r[8:12, 0] = [np.nan, np.inf, 5e8, 4e9]     # undefined rectangles and a wrapping centre
        r[12:20, 3] = r[12:20, 2]                   # h == w: swapped
    return d


def run(task, dets, sizes, K, dev, **kw):
    R = POSE_R if task == L.TASK_POSE else OBB_R
    Fo = 57 if task == L.TASK_POSE else 10
    out = torch.full((len(sizes), 1 + K * Fo), SENTINEL, dtype=torch.float32, device=dev)
    P.yolo_pose_obb_postprocess(torch.from_numpy(dets).to(dev), sizes, task=task, max_rows=K, row_floats=R, rows_out=out,
                                **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("keep_p", [1.0, 0.6], ids=["greedy", "oneshot"])
def test_pose_rows_equal_host(dev, keep_p):
    """b8 of mixed frame sizes, 300 rows: counts 0, below and above max_rows, keep flags all 1 (greedy NMS output) or
    0 / 1 (one-shot), undefined rectangles and NaN keypoints -> the host trtx_get_rect_adapt_landmark, the tail zeroed."""
    rng = np.random.default_rng(11)
    K = 300
    counts = [300, 0, 120, 450, 1, 299, 77, 300]
    dets = pose_dets(rng, len(MIXED), K, counts, keep_p)
    got = run(L.TASK_POSE, dets, MIXED, K, dev)
    print(f"pose {keep_p}: {check(L.TASK_POSE, got, dets, MIXED, K, POSE_R)} rows equal")


@pytest.mark.parametrize("net", [640, 1024])
@pytest.mark.parametrize("keep_p", [1.0, 0.6], ids=["greedy", "oneshot"])
def test_obb_rows_equal_host(dev, net, keep_p):
    """The same for oriented boxes at both network sizes (yolov8-obb 640, yolo11-obb 1024): 8 x 2000 rows with angles at 0,
    +-pi/2, pi, NaN and inf, h == w swaps, undefined rectangles -> the host trtx_get_corner, bit for bit."""
    rng = np.random.default_rng(net + int(keep_p * 10))
    K = 2000
    counts = [2000, 0, 1500, 2600, 3, 1999, 800, 2000]
    dets = obb_dets(rng, len(MIXED), K, counts, net, keep_p)
    got = run(L.TASK_OBB, dets, MIXED, K, dev, net_w=net, net_h=net)
    print(f"obb net {net} {keep_p}: {check(L.TASK_OBB, got, dets, MIXED, K, OBB_R, net=net)} rows equal, 0 differ")


def test_70_frames_two_launches(dev):
    """70 frames of assorted sizes in one call (two launches of <= 64 frames), both tasks."""
    rng = np.random.default_rng(70)
    sizes = [(int(rng.integers(1, 3000)), int(rng.integers(1, 3000))) for _ in range(70)]
    K = 40
    counts = [int(rng.integers(0, 50)) for _ in range(70)]
    dets = pose_dets(np.random.default_rng(71), 70, K, counts, 0.7)
    check(L.TASK_POSE, run(L.TASK_POSE, dets, sizes, K, dev), dets, sizes, K, POSE_R)
    dets = obb_dets(np.random.default_rng(72), 70, K, counts, 640, 0.7)
    check(L.TASK_OBB, run(L.TASK_OBB, dets, sizes, K, dev), dets, sizes, K, OBB_R)


def _heads_chain(dev, task, B, seed):
    """synthetic heads -> YoloLayerPlugin decode -> trtx_nms_enqueue; also the oracle's decode of the same heads."""
    if task == L.TASK_POSE:
        heads = synth.yolov8_heads(B, seed=seed, nc=1, extra=51, n_obj=30)
        plug = P.YoloLayerPlugin(1, 17, 0.0, 640, 640, 1000, False, True, False, (8, 16, 32))
    else:
        heads = synth.yolov8_heads(B, seed=seed, nc=15, extra=1, n_obj=40)
        plug = P.YoloLayerPlugin(15, 17, 0.0, 640, 640, 1000, False, False, True, (8, 16, 32))
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(h).to(dev) for h in heads], [out], ws) == 0
    return heads, out, plug.output_elems()


def test_decode_nms_pose_chain(dev, oracle):
    """Pose heads (nc 1, 51 keypoint floats) -> decode -> trtx_nms_enqueue with 51 extras -> the new call: the kept counts
    equal the oracle chain's, the rows equal the host functions on the same NMS output, and they agree with the host
    functions on the oracle's NMS rows up to the decode's float tolerance."""
    B, K, sizes = 4, 100, [(1920, 1080), (640, 480), (1080, 1920), (333, 1001)]
    heads, out, elems = _heads_chain(dev, L.TASK_POSE, B, 31)
    comp = P.batch_nms(out, B, elems, 0.5, 0.45, det_floats=90, max_det=K, extra_floats=51, extra_offset=38)
    rows = P.yolo_pose_obb_postprocess(comp, sizes, task=L.TASK_POSE, max_rows=K)
    torch.cuda.synchronize()
    dets, got = comp.cpu().numpy(), rows.cpu().numpy()
    check(L.TASK_POSE, got, dets, sizes, K, POSE_R)
    ref_dec, _ = oracle.yolov8_decode(heads, nc=1, is_pose=True)
    for b, (w, h) in enumerate(sizes):
        res, _ = oracle.nms(0, ref_dec[b], 1000, 90, 0.5, 0.45)
        n = len(res)
        assert int(got[b, 0]) == n > 0
        ref_rows = np.zeros((K, POSE_R), F)
        ref_rows[:n, :6], ref_rows[:n, 6], ref_rows[:n, 7:] = res[:, :6], 1, res[:, 38:89]
        _, want = host_rows(L.TASK_POSE, np.concatenate([[n], ref_rows.ravel()]).astype(F), w, h, K, POSE_R)
        g = got[b, 1:].reshape(K, 57)[:n]
        assert np.abs(g[:, :4] - want[:n, :4]).max() <= 1
        assert np.allclose(g[:, 6:], want[:n, 6:], rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("mode", [L.NMS_GREEDY, L.NMS_ONESHOT])
def test_decode_nms_obb_chain(dev, oracle, mode):
    """OBB heads (nc 15, one angle) -> decode -> batch_nms_obb (greedy, or one-shot with keep 0 / 1 rows) -> the new call at
    both network sizes' geometry: rows equal the host trtx_get_corner on the same NMS output; greedy counts equal the
    oracle's nms_obb."""
    B, K, sizes = 3, 1000, [(1920, 1080), (1024, 1024), (720, 1280)]
    heads, out, elems = _heads_chain(dev, L.TASK_OBB, B, 41)
    comp = P.batch_nms_obb(out, B, elems, 0.3, 0.45, max_det=K, mode=mode)
    dets = comp.cpu().numpy()
    for net in (640, 1024):
        rows = P.yolo_pose_obb_postprocess(comp, sizes, task=L.TASK_OBB, max_rows=K, net_w=net, net_h=net)
        torch.cuda.synchronize()
        got = rows.cpu().numpy()
        n = check(L.TASK_OBB, got, dets, sizes, K, OBB_R, net=net)
        assert n > 30
    if mode == L.NMS_GREEDY:
        ref_dec, _ = oracle.yolov8_decode(heads, nc=15, is_obb=True)
        for b in range(B):
            res, _ = oracle.nms(3, ref_dec[b], 1000, 90, 0.3, 0.45)
            assert int(got[b, 0]) == len(res)
    else:
        assert any((dets[b, 1:1 + int(dets[b, 0]) * 8].reshape(-1, 8)[:, 6] == 0).any() for b in range(B))


def test_graph_capture_replay(dev):
    """Both tasks captured into one CUDA graph: replays give the eager result."""
    rng = np.random.default_rng(5)
    K = 200
    pd = torch.from_numpy(pose_dets(rng, 8, K, [200] * 8, 0.8)).to(dev)
    od = torch.from_numpy(obb_dets(rng, 8, K, [200] * 8, 1024, 0.8)).to(dev)
    eager_p = P.yolo_pose_obb_postprocess(pd, MIXED, task=L.TASK_POSE, max_rows=K)
    eager_o = P.yolo_pose_obb_postprocess(od, MIXED, task=L.TASK_OBB, max_rows=K, net_w=1024, net_h=1024)
    out_p, out_o = torch.full_like(eager_p, SENTINEL), torch.full_like(eager_o, SENTINEL)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            P.yolo_pose_obb_postprocess(pd, MIXED, task=L.TASK_POSE, max_rows=K, rows_out=out_p)
            P.yolo_pose_obb_postprocess(od, MIXED, task=L.TASK_OBB, max_rows=K, net_w=1024, net_h=1024, rows_out=out_o)
        torch.cuda.synchronize()
        assert torch.all(out_p == SENTINEL)            # capture ran nothing
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
    assert torch.equal(out_p.nan_to_num(5.5), eager_p.nan_to_num(5.5)) and torch.equal(out_o, eager_o)


def test_rejected_call_writes_nothing(dev):
    dets = torch.zeros((2, 1 + 4 * POSE_R), device=dev)
    rows = torch.full((2, 1 + 4 * 57), SENTINEL, device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.yolo_pose_obb_postprocess(dets, [(64, 64), (0, 64)], task=L.TASK_POSE, max_rows=4, rows_out=rows)
    torch.cuda.synchronize()
    assert torch.all(rows == SENTINEL)
