"""yolov9, yolov10 and yolov13 on the device:
(1) the library's decode (TRTX_YOLO_V8 with det_floats 38 / 6, yolov9's is_seg) against each driver's OWN compiled
    CalDetection (oracle/_ref/libref_af_<driver>.so, same GPU, same inputs; where it was not built, its outputs stored in
    tests/golden/ref_af_gpu.npz) at batch 1 and 3, bit for bit, rows compared in anchor order (the reference's order is
    atomicAdd arrival);
(2) TRTX_BOX_V9 on plugin rows and through the fused and split decode + NMS, bit for bit against the oracle of yolov9's nms()
    (oracle/anchor_free.py), and fused against split and against the plugin-row path;
(3) trtx_yolo_topk_postprocess_enqueue against the oracle of get_topk + get_rect: more than 64 frames of mixed sizes, NaN
    and threshold confidences, sentinel-filled outputs with guard elements, rejected calls that write nothing, graph replay;
(4) yolov13 through the greedy and one-shot NMS on its 6-float rows;
and the TensorRT creators enqueued through tests/trt_adapter_anchor_free_check.cpp --gpu."""
import ctypes as C
import subprocess

import numpy as np
import pytest
import torch

from oracle import anchor_free as A
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

from test_anchor_free_cpu import SIZES, _build_check, v9_rows, v10_rows

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_af_gpu")
SENT = -12345.0


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _heads(B, seed, nc=80, seg=False, strides=(8, 16, 32), net=640):
    """[B, 4 + nc (+32), grid] per level: ltrb distances > 0, class logits N(-9, 2) (some 2 % of the anchors pass the 0.1
    gate), mask coefficients N(0, 1); and per level and image 30 objects, each a 2 x 2 block of cells of one class with a
    logit N(1.5, 1.5) and similar distances, so that their boxes overlap."""
    rng = np.random.default_rng(seed)
    out = []
    for s in strides:
        gw = net // s
        g = gw * gw
        h = rng.normal(0, 1, (B, 4 + nc + (32 if seg else 0), g)).astype(np.float32)
        h[:, :4] = np.abs(h[:, :4]) * 3 + 0.25
        h[:, 4:4 + nc] = rng.normal(-9.0, 2.0, (B, nc, g))
        for b in range(B):
            for _ in range(30):
                c0 = int(rng.integers(0, gw - 1)) * gw + int(rng.integers(0, gw - 1))
                cls, dist = int(rng.integers(0, nc)), rng.uniform(1.5, 4.0, 4)
                for c in (c0, c0 + 1, c0 + gw, c0 + gw + 1):
                    h[b, 4 + cls, c] = rng.normal(1.5, 1.5)
                    h[b, :4, c] = dist * rng.uniform(0.9, 1.1, 4)
        out.append(h)
    return out


def _plugin(driver, seg=False):
    d = P.ANCHOR_FREE_DRIVERS[driver]
    if driver == "yolov9":
        return P.YoloLayerPluginV9(d["classes"], *d["net"], d["max_out"], seg)
    return P.YoloLayerPluginV10(d["classes"], *d["net"], d["max_out"], (8, 16, 32))


def _decode(dev, plug, heads):
    B = heads[0].shape[0]
    d_heads = [torch.from_numpy(h).to(dev) for h in heads]
    out = torch.full((B, plug.output_elems()), SENT, dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, d_heads, [out], ws) == 0
    return d_heads, out


def _canon(rows):
    return rows[np.lexsort(tuple(rows[:, k] for k in range(rows.shape[1] - 1, -1, -1)))]


@pytest.mark.parametrize("driver,seg", [("yolov9", False), ("yolov9", True), ("yolov10", False), ("yolov13", False)])
@pytest.mark.parametrize("B", [1, 3])
def test_decode_equals_driver_kernel(dev, driver, seg, B):
    plug = _plugin(driver, seg)
    F = plug.DET_FLOATS
    heads = _heads(B, 950 + B + 2 * seg, seg=seg)
    d_heads, out = _decode(dev, plug, heads)
    got = out.cpu().numpy()
    lib = G.lib(f"libref_af_{driver}.so")
    ref = None
    if lib is not None:
        assert lib.ref_af_det_floats() == F
        r = torch.zeros_like(out)
        st = (C.c_int * 3)(8, 16, 32)
        assert lib.ref_af_enqueue(80, 640, 640, plug.mMaxOutObject, int(seg), st, 3, B, _ptrs(d_heads), C.c_void_p(r.data_ptr()),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        ref = r.cpu().numpy()
    W = 6 + (32 if seg else 0)  # the floats a row's decode writes (yolov9 without is_seg leaves the mask floats alone)
    for b in range(B):
        n = int(got[b, 0])
        assert 50 < n < plug.mMaxOutObject
        rows = got[b, 1:1 + n * F].reshape(n, F)[:, :W]
        assert (rows[:, 4] >= np.float32(0.1)).all()
        refb = None if ref is None else \
            np.concatenate([[ref[b, 0]], _canon(ref[b, 1:1 + int(ref[b, 0]) * F].reshape(-1, F)[:, :W]).ravel()])
        G.equal(f"decode.{driver}.{int(seg)}.{B}.{b}", np.concatenate([[got[b, 0]], _canon(rows).ravel()]), refb)


def _nms_rows(dev, buf_np, det_floats, extra):
    """trtx_nms_enqueue with TRTX_BOX_V9 on plugin rows already on the device (or numpy rows) -> (compact, keep index)"""
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    buf = buf_np if isinstance(buf_np, torch.Tensor) else torch.from_numpy(np.atleast_2d(buf_np)).to(dev)
    out, idx = P.batch_nms(buf, buf.shape[0], buf.shape[1], d["conf_thresh"], d["nms_thresh"], box_format=L.BOX_V9,
                           det_floats=det_floats, max_det=d["max_out"], extra_floats=extra, extra_offset=6 if extra else 0,
                           return_index=True)
    return out.cpu().numpy(), idx.cpu().numpy()


def _check_v9(comp, b, res, extra):
    R = 7 + extra
    n = int(comp[b, 0])
    assert n == len(res)
    rows = comp[b, 1:1 + n * R].reshape(n, R)
    assert np.array_equal(rows[:, :6], res[:, :6]) and (rows[:, 6] == 1).all()
    if extra:
        assert np.array_equal(rows[:, 7:], res[:, 6:38])
    assert not comp[b, 1 + n * R:].any()


@pytest.mark.parametrize("seg", [False, True])
def test_box_v9_plugin_rows_equal_oracle(dev, seg):
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    plug = _plugin("yolov9", seg)
    heads = _heads(3, 960 + seg, seg=seg)
    _, out = _decode(dev, plug, heads)
    extra = 32 if seg else 0
    comp, _ = _nms_rows(dev, out, 38, extra)
    host = out.cpu().numpy()
    for b in range(3):
        res, _ = A.v9_nms(host[b], d["max_out"], 38, d["conf_thresh"], d["nms_thresh"])
        assert len(res) > 10
        _check_v9(comp, b, res, extra)


def test_box_v9_crafted_rows_equal_oracle(dev):
    """Straddling pairs, confidences at 0.1f, tied confidences in row order, a NaN confidence, and more rows than the
    2000 the driver reads."""
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    rows = [v9_rows(s) for s in (910, 911)]
    rows[1] = np.concatenate([rows[1], rows[1][:5]])
    rows[1][-1, 4] = np.nan
    big = np.zeros((d["max_out"] + 100, 38), np.float32)
    rng = np.random.default_rng(962)
    xy = rng.uniform(0, 3000, (len(big), 2))
    big[:, :2], big[:, 2:4] = xy, xy + rng.uniform(5, 40, (len(big), 2))
    big[:, 4], big[:, 5] = rng.uniform(0.05, 1, len(big)), rng.integers(0, 3, len(big))
    rows.append(big)
    cap = len(big)
    bufs = np.zeros((3, 1 + cap * 38), np.float32)
    for b, r in enumerate(rows):
        bufs[b, 0] = len(r)
        bufs[b, 1:1 + r.size] = r.ravel()
    comp, _ = _nms_rows(dev, bufs, 38, 32)
    for b in range(3):
        # the library reads min(count, max_rows) rows, yolov9 min(count, 2000): pass the driver's limit
        lim = bufs[b].copy()
        lim[0] = min(lim[0], d["max_out"])
        res, _ = A.v9_nms(lim, cap, 38, d["conf_thresh"], d["nms_thresh"])
        if b == 2:
            comp2, _ = _nms_rows(dev, lim[None], 38, 32)
            _check_v9(comp2, 0, res, 32)
        else:
            _check_v9(comp, b, res, 32)


def test_box_v9_fused_equals_split_and_plugin_rows(dev):
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    plug = _plugin("yolov9")
    B = 4
    heads = _heads(B, 970)
    d_heads, out = _decode(dev, plug, heads)
    rows_comp, rows_idx = _nms_rows(dev, out, 38, 0)
    fused = P.FusedYoloDecodeNms(plug, B, d["conf_thresh"], d["nms_thresh"], box_format=L.BOX_V9, device=dev)
    comp, idx = fused.enqueue(B, d_heads)
    comp, idx = comp.cpu().numpy().copy(), idx.cpu().numpy().copy()
    fused.enqueue_scan(B, d_heads)
    split, _ = fused.enqueue_nms(B, d_heads)
    split = split.cpu().numpy()
    assert np.array_equal(comp, split) and np.array_equal(comp, rows_comp)
    host = out.cpu().numpy()
    for b in range(B):
        res, src = A.v9_nms(host[b], d["max_out"], 38, d["conf_thresh"], d["nms_thresh"])
        _check_v9(comp, b, res, 0)
    # one-shot has no yolov9 reference: refused
    q = P.nms_params(L.BOX_V9, L.NMS_ONESHOT, 0.1, 0.45, 100)
    lib = L.load()
    assert lib.trtx_nms_workspace_size(C.byref(q), 1, 100) == 0
    f1 = P.FusedYoloDecodeNms(plug, B, 0.1, 0.45, mode=L.NMS_ONESHOT, box_format=L.BOX_V9, device=dev)
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        f1.enqueue(B, d_heads)


def _topk_expect(host, sizes, max_rows, conf=0.5):
    exp = np.zeros((len(sizes), 1 + max_rows * 6), np.float32)
    for b, (w, h) in enumerate(sizes):
        r = A.topk(host[b], max_rows, 6, conf, w, h)
        exp[b, 0] = len(r)
        exp[b, 1:1 + r.size] = r.ravel()
    return exp


def _sentinel(dev, B, K, guard=64):
    full = torch.full((B * (1 + K * 6) + guard,), SENT, dtype=torch.float32, device=dev)
    return full, full[:B * (1 + K * 6)].view(B, 1 + K * 6)


def test_topk_rows_equal_oracle(dev):
    d = P.ANCHOR_FREE_DRIVERS["yolov10"]
    K = d["max_out"]
    B = 70  # two launches
    plug = _plugin("yolov10")
    heads = _heads(B, 980)
    _, out = _decode(dev, plug, heads)
    host = out.cpu().numpy()
    # frame 1: crafted rows with NaN and threshold confidences, in place of the decoded ones
    crafted = v10_rows(930)
    host[1] = 0
    host[1, 0] = len(crafted)
    host[1, 1:1 + crafted.size] = crafted.ravel()
    dets = torch.from_numpy(host).to(dev)
    sizes = [SIZES[i % len(SIZES)] for i in range(B)]
    full, rows = _sentinel(dev, B, K)
    P.yolo_topk_postprocess(dets, sizes, max_rows=K, conf_thresh=d["conf_thresh"], rows_out=rows)
    got = rows.cpu().numpy()
    exp = _topk_expect(host, sizes, K)
    assert np.array_equal(got, exp, equal_nan=True)
    assert (full[-64:] == SENT).all()
    assert np.isnan(got[1, 1:1 + int(got[1, 0]) * 6].reshape(-1, 6)[:, 4]).sum() == 1
    assert (got[:, 0] > 0).all()
    # the unclamped variant gives other rectangles on the same rows
    other = P.yolo_topk_postprocess(dets, sizes, max_rows=K, conf_thresh=d["conf_thresh"], variant=L.YOLO_V5).cpu().numpy()
    assert not np.array_equal(other, got)
    # max_rows below the count: the first max_rows rows
    k2 = 40
    small = torch.from_numpy(np.ascontiguousarray(host[:, :1 + k2 * 6])).to(dev)
    g2 = P.yolo_topk_postprocess(small, sizes, max_rows=k2, conf_thresh=d["conf_thresh"]).cpu().numpy()
    assert np.array_equal(g2, _topk_expect(host, sizes, k2)[:, :1 + k2 * 6], equal_nan=True)


def test_topk_rejected_calls_write_nothing(dev):
    lib = L.load()
    B, K = 3, 10
    dets = torch.zeros((B, 1 + K * 6), dtype=torch.float32, device=dev)
    dets[:, 0] = 5
    dets[:, 5::6] = 0.9
    full, rows = _sentinel(dev, B, K)
    wh = (C.c_int32 * (2 * B))(640, 480, 640, 480, 640, 480)
    bad_wh = (C.c_int32 * (2 * B))(640, 480, 0, 480, 640, 480)
    ok = L.YoloTopkParams(L.YOLO_V8, 640, 640, 6, 0.5)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cases = [(L.YoloTopkParams(L.YOLO_V3, 640, 640, 6, 0.5), wh, B, K), (L.YoloTopkParams(L.YOLO_V8, 640, 640, 5, 0.5), wh, B, K),
             (L.YoloTopkParams(L.YOLO_V8, 0, 640, 6, 0.5), wh, B, K), (ok, bad_wh, B, K), (ok, wh, 0, K), (ok, wh, B, 0)]
    for q, w, b, k in cases:
        assert lib.trtx_yolo_topk_postprocess_enqueue(C.byref(q), w, b, C.c_void_p(dets.data_ptr()), k,
                                                      C.c_void_p(rows.data_ptr()), st) == L.ERR_INVALID
    assert lib.trtx_yolo_topk_postprocess_enqueue(None, wh, B, C.c_void_p(dets.data_ptr()), K, C.c_void_p(rows.data_ptr()), st) == L.ERR_INVALID
    torch.cuda.synchronize()
    assert (full == SENT).all()
    assert lib.trtx_yolo_topk_postprocess_enqueue(C.byref(ok), wh, B, C.c_void_p(dets.data_ptr()), K, C.c_void_p(rows.data_ptr()), st) == 0
    torch.cuda.synchronize()
    assert (rows[:, 0] == 5).all() and (full[-64:] == SENT).all()


def test_topk_graph_replay(dev):
    d = P.ANCHOR_FREE_DRIVERS["yolov10"]
    K, B = d["max_out"], 5
    plug = _plugin("yolov10")
    _, out_a = _decode(dev, plug, _heads(B, 990))
    _, out_b = _decode(dev, plug, _heads(B, 991))
    sizes = SIZES[:B]
    dets = out_a.clone()
    rows = torch.empty((B, 1 + K * 6), dtype=torch.float32, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        P.yolo_topk_postprocess(dets, sizes, max_rows=K, rows_out=rows, stream=s)   # warm-up
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        P.yolo_topk_postprocess(dets, sizes, max_rows=K, rows_out=rows, stream=torch.cuda.current_stream())
    for src in (out_b, out_a):
        dets.copy_(src)
        rows.fill_(SENT)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(rows.cpu().numpy(), _topk_expect(src.cpu().numpy(), sizes, K), equal_nan=True)


def test_yolov13_greedy_and_oneshot(oracle, dev):
    d = P.ANCHOR_FREE_DRIVERS["yolov13"]
    plug = _plugin("yolov13")
    B = 3
    _, out = _decode(dev, plug, _heads(B, 995))
    host = out.cpu().numpy()
    K = d["max_out"]
    greedy = P.batch_nms(out, B, out.shape[1], d["conf_thresh"], d["nms_thresh"], box_format=d["box_format"], det_floats=6,
                         max_det=K).cpu().numpy()
    oneshot, idx = P.batch_nms(out, B, out.shape[1], d["conf_thresh"], d["nms_thresh"], box_format=d["box_format"], det_floats=6,
                               max_det=K, mode=L.NMS_ONESHOT, return_index=True)
    oneshot, idx = oneshot.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, _ = oracle.nms(0, host[b], K, 6, d["conf_thresh"], d["nms_thresh"])
        n = int(greedy[b, 0])
        assert n == len(res) > 0 and np.array_equal(greedy[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res)
        # one-shot: every row >= conf_thresh with the keep flag of decode_kernel + nms_kernel (rows in input order there)
        exp = oracle.cuda_decode_nms(host[b], K, 6, d["conf_thresh"], d["nms_thresh"], K)[1:].reshape(K, 7)
        m = int(oneshot[b, 0])
        got = oneshot[b, 1:1 + m * 7].reshape(m, 7)
        assert m == int((host[b, 1:1 + int(host[b, 0]) * 6].reshape(-1, 6)[:, 4] >= np.float32(0.5)).sum())
        assert np.array_equal(got, exp[idx[b, :m]]) and 0 < got[:, 6].sum() < m


def test_creators_enqueue(tmp_path):
    r = subprocess.run([str(_build_check(tmp_path)), "--gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "gpu enqueue ok" in r.stdout
