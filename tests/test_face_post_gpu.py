"""RetinaFace post-process on the GPU (trtx_retina_postprocess_enqueue) against the library's host
trtx_retina_get_rect_adapt_landmark applied row by row, and yolo26-obb's NMS-free rows (TASK_OBB_NMS_FREE of
trtx_yolo_pose_obb_postprocess_enqueue) against trtx_get_corner -- the host functions tests/test_face_obb26_post_cpu.py pins
to the reference's compiled code.  Exact comparisons (NaN-equal)."""
import ctypes as C
import math

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


def _keep_flag(v):
    return 1.0 <= v < 2.0   # (int)v == 1


def _extras(variant):
    return 11 if variant == L.RETINA_ANTICOV else 10


def face_host_rows(variant, dets_b, img_w, img_h, K, in_w, in_h, thr, R=None, off=7):
    """The expected output of one frame: the rows of the first min(count, K) with keep 1 and !(conf < thr) through the host
    trtx_retina_get_rect_adapt_landmark, input order."""
    lib = L.load()
    R = R or 7 + _extras(variant)
    n = min(max(int(dets_b[0]), 0), K)
    src = dets_b[1:1 + K * R].reshape(K, R)
    out = np.zeros((K, 5 + _extras(variant)), F)
    t = F(P.float_ge_threshold(thr))
    m = 0
    for i in range(n):
        r = src[i]
        if not _keep_flag(r[6]) or r[4] < t:
            continue
        bb = (C.c_float * 4)(*[float(v) for v in r[:4]])
        k = np.ascontiguousarray(r[off:off + 10], F).copy()
        rect = (C.c_int * 4)()
        assert lib.trtx_retina_get_rect_adapt_landmark(in_w, in_h, img_w, img_h, bb, k.ctypes.data_as(C.POINTER(C.c_float)),
                                                       rect) == 0
        out[m, :4], out[m, 4], out[m, 5:15] = list(rect), r[4], k
        if variant == L.RETINA_ANTICOV:
            out[m, 15] = r[off + 10]
        m += 1
    return m, out


def check_faces(variant, got, dets, sizes, K, in_w, in_h, thr, R=None):
    rows = 0
    for b, (w, h) in enumerate(sizes):
        m, want = face_host_rows(variant, dets[b], w, h, K, in_w, in_h, thr, R)
        g = got[b, 1:].reshape(K, -1)
        assert got[b, 0] == m, (b, got[b, 0], m)
        bad = [i for i in range(K) if not np.array_equal(g[i], want[i], equal_nan=True)]
        assert not bad, (b, bad[:10], [(g[i].tolist(), want[i].tolist()) for i in bad[:3]])
        rows += m
    return rows


def face_dets(rng, variant, B, K, counts, keep_p=1.0):
    """Compact NMS rows (x1, y1, x2, y2, conf, 0, keep, landmarks[, mask_conf]) with the threshold's edge cases (exactly 0.75,
    one ulp below, NaN), keep flags 0 / 1 / 1.5 / NaN, non-finite and out-of-int boxes and landmarks, a wrapping width."""
    R = 7 + _extras(variant)
    d = np.zeros((B, 1 + K * R), F)
    for b in range(B):
        d[b, 0] = counts[b]
        r = d[b, 1:].reshape(K, R)
        x, y = rng.uniform(-30, 650, K), rng.uniform(-30, 650, K)
        r[:, :4] = np.stack([x, y, x + rng.uniform(-5, 300, K), y + rng.uniform(-5, 300, K)], 1)
        r[:, 4] = rng.uniform(0.5, 1, K)
        r[:, 6] = np.where(rng.uniform(0, 1, K) < keep_p, 1.0, 0.0)
        r[:, 7:17] = rng.uniform(-20, 660, (K, 10))
        if variant == L.RETINA_ANTICOV:
            r[:, 17] = rng.uniform(0, 1, K)
        r[:3, 4] = [0.75, np.nextafter(F(0.75), F(0)), np.nan]
        r[:12, 6] = 1
        r[3, 0], r[4, 2], r[5, 1], r[6, 3], r[7, 0] = np.nan, np.inf, -np.inf, 3e9, -1e38
        r[8, :4] = [-7e8, 10, 7e8, 30]          # r - l leaves the int range for the wide frames: wraps
        r[9, 7], r[10, 10], r[11, 16] = np.nan, np.inf, -3e9
        r[12, 6], r[13, 6] = 1.5, np.nan       # (int)1.5 == 1 is used, NaN is not
        r[3:14, 4] = 0.9
    return d


def run_faces(variant, dets, sizes, K, dev, **kw):
    out = torch.full((len(sizes), 1 + K * (5 + _extras(variant))), SENTINEL, dtype=torch.float32, device=dev)
    P.retina_postprocess(torch.from_numpy(dets).to(dev), sizes, variant=variant, max_rows=K, rows_out=out, **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy()


CASES = [(L.RETINA_FACE, 640, 480, 0.75), (L.RETINA_FACE, 640, 640, 0.75), (L.RETINA_ANTICOV, 640, 640, -math.inf),
         (L.RETINA_ANTICOV, 640, 480, 0.75)]


@pytest.mark.parametrize("variant,in_w,in_h,thr", CASES, ids=["face480", "face640", "anticov640", "anticov480-thr"])
@pytest.mark.parametrize("keep_p", [1.0, 0.6], ids=["greedy", "keep01"])
def test_face_rows_equal_host(dev, variant, in_w, in_h, thr, keep_p):
    """b8 of mixed frame sizes, 300 rows: counts 0, below and above max_rows; the threshold's edge cases; non-finite
    boxes and landmarks -> the host trtx_retina_get_rect_adapt_landmark row by row, the tail zeroed."""
    rng = np.random.default_rng(in_h + variant + int(10 * keep_p))
    K = 300
    counts = [300, 0, 120, 450, 1, 299, 77, 300]
    dets = face_dets(rng, variant, len(MIXED), K, counts, keep_p)
    got = run_faces(variant, dets, MIXED, K, dev, conf_thresh=thr, in_w=in_w, in_h=in_h)
    n = check_faces(variant, got, dets, MIXED, K, in_w, in_h, thr)
    g = got[0, 1:].reshape(K, -1)
    if thr == 0.75:   # frame 0: conf 0.75 and NaN are used, one ulp below 0.75 is not
        assert g[0, 4] == F(0.75) and np.isnan(g[1, 4]) and g[2, 4] == F(0.9)
    print(f"variant {variant} {in_w}x{in_h} thr {thr} keep {keep_p}: {n} rows equal")


def test_70_frames_two_launches(dev):
    """70 frames of assorted sizes in one call (two launches of <= 64 frames), both variants."""
    rng = np.random.default_rng(70)
    sizes = [(int(rng.integers(1, 3000)), int(rng.integers(1, 3000))) for _ in range(70)]
    K = 40
    counts = [int(rng.integers(0, 50)) for _ in range(70)]
    for variant in (L.RETINA_FACE, L.RETINA_ANTICOV):
        dets = face_dets(np.random.default_rng(71 + variant), variant, 70, K, counts, 0.7)
        got = run_faces(variant, dets, sizes, K, dev, conf_thresh=0.75, in_w=640, in_h=640)
        check_faces(variant, got, dets, sizes, K, 640, 640, 0.75)


def _retina_chain(dev, variant, B, seed):
    """synthetic heads -> Decode_TRT -> trtx_nms_enqueue (TRTX_BOX_RETINA, the landmarks [+ mask conf] as extras)."""
    anticov = variant == L.RETINA_ANTICOV
    heads = synth.anticov_heads(B, seed=seed) if anticov else synth.retina_heads(B, seed=seed)
    plug = P.DecodePlugin(640, 640, anticov=anticov)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(h).to(dev) for h in heads], [out], ws) == 0
    return P.batch_nms(out, B, plug.output_elems(), P.float_le_threshold(0.1), 0.4, box_format=L.BOX_RETINA,
                       det_floats=plug.det_floats, max_det=1000, extra_floats=_extras(variant), extra_offset=5)


@pytest.mark.parametrize("variant", [L.RETINA_FACE, L.RETINA_ANTICOV], ids=["retinaface", "anticov"])
def test_decode_nms_face_chain(dev, variant):
    """Heads -> decode -> NMS -> the new call at BASELINE config 3's 640x640, b16 of mixed sizes: the rows equal the host
    path over the same NMS output (CONF_THRESH 0.75 for retinaface, no threshold for AntiCov)."""
    B, K = 16, 1000
    sizes = (MIXED * 2)[:B]
    thr = 0.75 if variant == L.RETINA_FACE else -math.inf
    comp = _retina_chain(dev, variant, B, 21 + variant)
    rows = P.retina_postprocess(comp, sizes, variant=variant, max_rows=K, conf_thresh=thr, in_w=640, in_h=640)
    torch.cuda.synchronize()
    dets, got = comp.cpu().numpy(), rows.cpu().numpy()
    n = check_faces(variant, got, dets, sizes, K, 640, 640, thr)
    assert n > 0 and (variant == L.RETINA_FACE or got[:, 0].sum() == dets[:, 0].sum())
    print(f"variant {variant}: {int(dets[:, 0].sum())} NMS rows, {n} faces equal")


def _obb26_host_rows(dets_b, img_w, img_h, K, net=1024, R=90):
    lib = L.load()
    n = min(max(int(dets_b[0]), 0), K)
    src = dets_b[1:1 + K * R].reshape(K, R)
    out = np.zeros((K, 10), F)
    c = (C.c_int * 8)()
    for i in range(n):
        r = src[i]
        bb = (C.c_float * 4)(*[float(v) for v in r[:4]])
        lib.trtx_get_corner(net, net, img_w, img_h, bb, float(r[R - 1]), c)
        out[i, :8], out[i, 8:10] = list(c), r[4:6]
    return n, out


def test_yolo26_obb_gather_chain(dev):
    """yolo26-obb rows -> the NMS-free gather (YoloLayerPlugin26, is_obb) -> TASK_OBB_NMS_FREE at net 1024: every row of the
    first min(count, max_rows), no keep test (column 6 is mask[0] = 0 there), = trtx_get_corner row by row."""
    nc, A, K, B = 15, 21504, 300, 4
    sizes = MIXED[:B]
    rows = synth.yolo26_rows(B, seed=660, nc=nc, anchors=A, obb=True, n_obj=400)
    plug = P.YoloLayerPlugin26(nc, 17, K, False, False, False, True, A, conf_thresh=0.3)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(rows).to(dev)], [out], ws) == 0
    assert (out[:, 0] == K).all()   # more candidates than max_detections
    for K_call in (K, 100):         # and max_rows below the count: the first 100 rows of each frame
        part = out[:, :1 + K_call * 90].contiguous()
        got = P.yolo_pose_obb_postprocess(part, sizes, task=L.TASK_OBB_NMS_FREE, max_rows=K_call, net_w=1024, net_h=1024)
        torch.cuda.synchronize()
        dets = part.cpu().numpy()
        g = got.cpu().numpy()
        assert (dets[:, 1:].reshape(B, K_call, 90)[:, :, 6] == 0).all()
        total = 0
        for b, (w, h) in enumerate(sizes):
            m, want = _obb26_host_rows(dets[b], w, h, K_call)
            assert g[b, 0] == m and np.array_equal(g[b, 1:].reshape(K_call, 10), want), (b, K_call)
            total += m
        assert total > 30


def test_graph_capture_replay(dev):
    """Both face variants and the NMS-free OBB rows captured into one CUDA graph: replays give the eager result."""
    rng = np.random.default_rng(5)
    K = 200
    fd = torch.from_numpy(face_dets(rng, L.RETINA_FACE, 8, K, [200] * 8, 0.8)).to(dev)
    ad = torch.from_numpy(face_dets(rng, L.RETINA_ANTICOV, 8, K, [150] * 8, 0.8)).to(dev)
    od = torch.from_numpy(rng.uniform(1, 500, (8, 1 + K * 90)).astype(F)).to(dev)
    od[:, 0] = 180

    def calls(out_f=None, out_a=None, out_o=None):
        return (P.retina_postprocess(fd, MIXED, variant=L.RETINA_FACE, max_rows=K, conf_thresh=0.75, in_w=640, in_h=480,
                                     rows_out=out_f),
                P.retina_postprocess(ad, MIXED, variant=L.RETINA_ANTICOV, max_rows=K, conf_thresh=-math.inf, in_w=640,
                                     in_h=640, rows_out=out_a),
                P.yolo_pose_obb_postprocess(od, MIXED, task=L.TASK_OBB_NMS_FREE, max_rows=K, net_w=1024, net_h=1024,
                                            rows_out=out_o))

    eager = calls()
    outs = [torch.full_like(e, SENTINEL) for e in eager]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            calls(*outs)
        torch.cuda.synchronize()
        assert all(torch.all(o == SENTINEL) for o in outs)     # capture ran nothing
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
    for o, e in zip(outs, eager):
        assert torch.equal(o.nan_to_num(5.5), e.nan_to_num(5.5))


def test_rejected_call_writes_nothing(dev):
    dets = torch.zeros((2, 1 + 4 * 17), device=dev)
    rows = torch.full((2, 1 + 4 * 15), SENTINEL, device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.retina_postprocess(dets, [(64, 64), (0, 64)], variant=L.RETINA_FACE, max_rows=4, conf_thresh=0.75, in_w=640,
                             in_h=480, rows_out=rows)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.retina_postprocess(dets, [(64, 64), (64, 64)], variant=L.RETINA_FACE, max_rows=4, conf_thresh=0.75, in_w=640,
                             in_h=480, lmk_offset=8, rows_out=rows)
    obb = torch.zeros((2, 1 + 4 * 90), device=dev)
    orows = torch.full((2, 1 + 4 * 10), SENTINEL, device=dev)
    with pytest.raises(L.TrtxError, match="INVALID"):
        P.yolo_pose_obb_postprocess(obb, [(64, 64), (64, 0)], task=L.TASK_OBB_NMS_FREE, max_rows=4, rows_out=orows)
    torch.cuda.synchronize()
    assert torch.all(rows == SENTINEL) and torch.all(orows == SENTINEL)
