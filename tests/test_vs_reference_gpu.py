"""Parity against the REFERENCE'S OWN CUDA KERNELS run on the same GPU: oracle/_ref/libref_*.so are the
reference's plugin / helper sources compiled by oracle/Makefile against the mock NvInfer.h and the OpenCV shim;
tests/ only calls their public entry points (plugin enqueue(), free functions).  These are the strongest parity checks
of the suite: same inputs, the reference's code vs ours.  Where oracle/_ref was not built, the reference's outputs of
an H100 run come from tests/golden/ref_gpu.npz (oracle/golden.py).
The reference's slot order is atomicAdd arrival, so decode outputs are compared as canonically sorted sets."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
G = RefOutputs("ref_gpu")


def _ptrs(ts):
    a = (C.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        a[i] = t.data_ptr()
    return a


def _canon(rows):
    order = np.lexsort(tuple(rows[:, k] for k in range(rows.shape[1] - 1, -1, -1)))
    return rows[order]


def _rows(buf, b, F, cols, n=None):
    """canonically sorted rows of image b (n rows, default its count), columns `cols`; None for None"""
    if buf is None:
        return None
    n = int(buf[b, 0]) if n is None else n
    return _canon(buf[b, 1:1 + n * F].reshape(n, F)[:, cols])


def _np(t):
    return None if t is None else t.cpu().numpy()


def _ours_decode(plug, hd, B, dev):
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    ws = torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, hd, [out], ws) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _ref_v8(lib, hd, B, dev, nc=80, gate=0.0, seg=0, pose=0, obb=0):
    if lib is None:
        return None
    ref = torch.zeros((B, 1 + 1000 * 90), dtype=torch.float32, device=dev)
    strides = (C.c_int * 3)(8, 16, 32)
    assert lib.ref_v8_plugin_enqueue(nc, 17, C.c_float(gate), 640, 640, 1000, seg, pose, obb, strides, 3, B, _ptrs(hd),
                                     C.c_void_p(ref.data_ptr()), None) == 0
    return ref.cpu().numpy()


@pytest.mark.parametrize("seed,B", [(0, 1), (1, 8)])
def test_yolov8_plugin_vs_reference_kernel(dev, seed, B):
    lib = G.lib("libref_yolov8.so")
    heads = synth.yolov8_heads(B, seed=400 + seed)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    ref = _ref_v8(lib, hd, B, dev)
    got = _ours_decode(P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32)), hd, B, dev)
    G.equal(f"v8_plugin.{seed}.count", got[:, 0], None if ref is None else ref[:, 0])
    assert got[:, 0].min() > 100
    for b in range(B):
        G.equal(f"v8_plugin.{seed}.{b}", _rows(got, b, 90, slice(0, 6)), _rows(ref, b, 90, slice(0, 6)))  # same CUDA expf, same operation order: bit-exact


def test_yolov8_near_ulp_sigmoid_collisions_vs_reference_kernel(dev):
    """Logits a few ulps apart: whether two of them round to the same probability (-> the EARLIER class wins the
    reference's strict `p > max`) depends on expf itself, so this is checked against the reference kernel (same CUDA
    expf), for every scan variant (class slices merge their running state; the TMA pipeline replays from smem)."""
    lib = G.lib("libref_yolov8.so")
    heads = synth.yolov8_heads(1, seed=430, n_obj=0)
    h = heads[0]
    n = 0
    for x0 in (0.3, 1.5, 2.75, 5.0, 9.0, 14.0):
        x = np.float32(x0)
        for k in range(1, 25):
            y = x
            for _ in range(k):
                y = np.nextafter(y, np.float32(0))
            cell = 40 * n + k
            h[0, 4 + 60 - k, cell] = y      # earlier class, k ulps below the maximum
            h[0, 4 + 60, cell] = x
            h[0, 4 + 70, cell] = y          # later class: never wins
        n += 1
    hd = [torch.from_numpy(a).to(dev) for a in heads]
    ref = _ref_v8(lib, hd, 1, dev)
    r = _rows(ref, 0, 90, slice(0, 6))
    plug = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, False, False, (8, 16, 32))
    for pipe, slices, unroll in ((1, 2, 5), (0, 2, 5), (0, 4, 10), (0, 1, 8), (0, 8, 5)):
        plug.tune(tma=pipe, slices=slices, rows=unroll)
        got = _ours_decode(plug, hd, 1, dev)
        G.equal("v8_ulp.count", got[:, 0], None if ref is None else ref[:, 0])
        g = _rows(got, 0, 90, slice(0, 6))
        G.equal("v8_ulp.rows", g, r, msg=(pipe, slices, unroll))
        assert len(g) >= 6 * 24
        assert (g[:, 5] == 60).any() and (g[:, 5] != 60).any()     # both outcomes occur


@pytest.mark.parametrize("mode", ["seg", "pose", "obb"])
def test_yolov8_plugin_extras_vs_reference_kernel(dev, mode):
    lib = G.lib("libref_yolov8.so")
    seg, pose, obb = mode == "seg", mode == "pose", mode == "obb"
    nc = 1 if pose else (15 if obb else 80)
    extra = 32 if seg else (51 if pose else 1)
    B = 2
    heads = synth.yolov8_heads(B, seed=410, nc=nc, extra=extra, n_obj=20)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    ref = _ref_v8(lib, hd, B, dev, nc, 0.3, int(seg), int(pose), int(obb))
    got = _ours_decode(P.YoloLayerPlugin(nc, 17, 0.3, 640, 640, 1000, seg, pose, obb, (8, 16, 32)), hd, B, dev)
    G.equal(f"v8_extras.{mode}.count", got[:, 0], None if ref is None else ref[:, 0])
    cols = list(range(6)) + (list(range(6, 38)) if seg else []) + (list(range(38, 89)) if pose else []) + ([89] if obb else [])
    for b in range(B):
        # obb/pose use fp64 sin/cos/mul in both
        G.close(f"v8_extras.{mode}.{b}", _rows(got, b, 90, cols), _rows(ref, b, 90, cols), rtol=1e-6, atol=1e-6)


def test_yolov5_plugin_vs_reference_kernel(dev):
    lib = G.lib("libref_yolov5.so")
    B = 4
    heads = synth.yolov5_heads(B, seed=420)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    ref = None
    if lib is not None:
        ks = np.zeros((3, 8), np.float32)
        ki = ks.view(np.int32)
        for l, (s, a) in enumerate(zip((8, 16, 32), synth.V5_ANCHORS)):
            ki[l, 0], ki[l, 1] = 640 // s, 640 // s
            ks[l, 2:] = a
        ref = torch.zeros((B, 1 + 1000 * 38), dtype=torch.float32, device=dev)
        assert lib.ref_v5_plugin_enqueue(80, 640, 640, 1000, 0, ks.ctypes.data_as(C.c_void_p), 3, B, _ptrs(hd),
                                         C.c_void_p(ref.data_ptr()), None) == 0
        ref = ref.cpu().numpy()
    kern = [P.YoloKernel(640 // s, 640 // s, a) for s, a in zip((8, 16, 32), synth.V5_ANCHORS)]
    got = _ours_decode(P.YoloLayerPluginV5(80, 640, 640, 1000, False, kern), hd, B, dev)
    G.equal("v5_plugin.count", got[:, 0], None if ref is None else ref[:, 0])
    assert got[:, 0].min() > 100
    for b in range(B):
        # FMA contraction of the reference build: <= 2 ulp
        G.close(f"v5_plugin.{b}", _rows(got, b, 38, slice(0, 6)), _rows(ref, b, 38, slice(0, 6)), rtol=3e-7, atol=0)


def test_retina_plugin_vs_reference_kernel(dev):
    lib = G.lib("libref_retina.so")
    h, w = 480, 640   # the input size compiled into the reference's decode.cu
    assert lib is None or (lib.ref_retina_input_h(), lib.ref_retina_input_w()) == (h, w)
    B = 4
    heads = synth.retina_heads(B, seed=430, in_h=h, in_w=w)
    hd = [torch.from_numpy(x).to(dev) for x in heads]
    plug = P.DecodePlugin(h, w)
    ref = None
    if lib is not None:
        ref = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
        assert lib.ref_retina_plugin_enqueue(B, _ptrs(hd), C.c_void_p(ref.data_ptr()), None) == 0
        ref = ref.cpu().numpy()
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    assert plug.enqueue(B, hd, [out], torch.empty(plug.getWorkspaceSize(B), dtype=torch.uint8, device=dev)) == 0
    got = out.cpu().numpy()
    G.equal("retina_plugin.count", got[:, 0], None if ref is None else ref[:, 0])
    assert got[:, 0].min() > 50
    for b in range(B):
        G.close(f"retina_plugin.{b}", _rows(got, b, 15, slice(0, 15)), _rows(ref, b, 15, slice(0, 15)), rtol=3e-7, atol=1e-5)


def test_cuda_decode_nms_vs_reference_kernels(dev, oracle):
    lib = G.lib("libref_yolov8.so")
    heads = synth.yolov8_heads(1, seed=440)
    plugin_out, _ = oracle.yolov8_decode(heads)
    pd = torch.from_numpy(plugin_out).to(dev)
    rr = None
    if lib is not None:
        parray = torch.zeros(1 + 1000 * 7, dtype=torch.float32, device=dev)
        assert lib.ref_v8_cuda_decode_nms(C.c_void_p(pd.data_ptr()), 1000, C.c_float(0.5), C.c_void_p(parray.data_ptr()), 1000,
                                          C.c_float(0.45), None) == 0
        ref = parray.cpu().numpy()
        cnt = int(ref[0])
        rr = ref[1:1 + cnt * 7].reshape(cnt, 7)
        rr = _canon(rr[rr[:, 4] > 0])          # holes (rows below conf) stay zero
    comp = P.batch_nms(pd, 1, plugin_out.shape[1], 0.5, 0.45, mode=L.NMS_ONESHOT).cpu().numpy()
    n = int(comp[0, 0])
    gg = comp[0, 1:1 + n * 7].reshape(n, 7)
    G.equal("v8_cuda_decode_nms", _canon(gg), rr)   # identical rows AND identical keep flags


def test_preprocess_vs_reference_kernel(dev):
    lib = G.lib("libref_yolov8.so")
    # 640x640 / 640x480 / 480x640 / 416x640: scale == 1 -> the TMA-staged unit-scale kernel (incl. padding and border
    # tiles); 500x640 has a pitch TMA cannot take (1500 B) -> general kernel at scale 1; the others resample.
    for (h, w) in [(640, 640), (1080, 1920), (375, 500), (480, 640), (640, 480), (416, 640), (640, 500), (639, 640), (640, 624)]:
        img = synth.frames(1, seed=h, h=h, w=w)[0]
        ref = None
        if lib is not None:
            ref = torch.zeros((3, 640, 640), dtype=torch.float32, device=dev)
            assert lib.ref_v8_preprocess(img.ctypes.data_as(C.c_void_p), w, h, C.c_void_p(ref.data_ptr()), 640, 640, None) == 0
        dst = torch.zeros((1, 3, 640, 640), dtype=torch.float32, device=dev)
        P.cuda_batch_preprocess([torch.from_numpy(img).to(dev)], dst, 640, 640)
        torch.cuda.synchronize()
        # both builds leave the bilinear sum to nvcc's FMA contraction: bit-identical
        G.equal(f"preprocess.{h}x{w}", dst[0].cpu().numpy(), _np(ref), msg=(h, w))


def test_rcnn_vs_reference_functions(dev):
    lib = G.lib("libref_rcnn.so")
    B, A, H, W, top_n = 2, 15, 50, 67, 6000
    scores, deltas = synth.rpn_inputs(B, seed=450, A=A, H=H, W=W)
    anchors = synth.rcnn_anchors()
    sd, dd = torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)
    rs, rb = None, None
    if lib is not None:
        rs, rb = torch.zeros((B, top_n), device=dev), torch.zeros((B, top_n, 4), device=dev)
        assert lib.ref_rpn_decode(B, C.c_void_p(sd.data_ptr()), C.c_void_p(dd.data_ptr()), C.c_void_p(rs.data_ptr()),
                                  C.c_void_p(rb.data_ptr()), H, W, 800, 1067, C.c_float(16.0),
                                  anchors.ctypes.data_as(C.c_void_p), A, top_n) == 0
    plug = P.RpnDecodePlugin(top_n, anchors, 16.0, 800, 1067, H, W)
    os_, ob = torch.zeros((B, top_n), device=dev), torch.zeros((B, top_n, 4), device=dev)
    ws = torch.empty(256, dtype=torch.uint8, device=dev)
    assert plug.enqueue(B, [sd, dd], [os_, ob], ws) == 0
    G.equal("rpn_decode.scores", _np(os_), _np(rs))                                      # same ordered top-6000
    G.close("rpn_decode.boxes", _np(ob), _np(rb), rtol=3e-7, atol=1e-4)

    # RpnNms on <= 1024 boxes (the reference kernel is only race-free within one block), fed the reference's decode outputs
    pre, post = 1000, 300
    s1 = os_[:, :pre].contiguous()
    b1 = torch.from_numpy(G.array("rpn_nms.in_boxes", None if rb is None else _np(rb[:, :pre].contiguous()))).to(dev)
    rnb = None
    if lib is not None:
        rnb = torch.zeros((B, post, 4), device=dev)
        # The reference is only correct for batch 1: its second sort overwrites the iota `indices` buffer that the next
        # image's first sort uses as payload (RpnNms.cu:100 vs :112-113) -- call it once per image.
        for b in range(B):
            assert lib.ref_rpn_nms(1, C.c_void_p(s1[b].data_ptr()), C.c_void_p(b1[b].data_ptr()), C.c_void_p(rnb[b].data_ptr()),
                                   pre, post, C.c_float(0.7)) == 0
    onb = torch.zeros((B, post, 4), device=dev)
    assert P.RpnNmsPlugin(0.7, post, pre).enqueue(B, [s1, b1], [onb], ws) == 0
    from oracle import oracle as O
    orc = O.rpn_nms(s1.cpu().numpy(), b1.cpu().numpy(), post, 0.7)
    G.equal("rpn_nms.boxes", _np(onb), _np(rnb), msg=f"rows differing from the oracle: ours {int((onb.cpu().numpy() != orc).any(-1).sum())}")


def test_rcnn_predictor_and_batched_nms_vs_reference_functions(dev):
    lib = G.lib("libref_rcnn.so")
    B = 2
    ws = torch.empty(256, dtype=torch.uint8, device=dev)
    # PredictorDecode + BatchedNms (count = 1000: one block)
    N, Cc = 1000, 80
    sc, dl, pr = synth.predictor_inputs(B, seed=451, N=N, Ccls=Cc)
    scd, dld, prd = (torch.from_numpy(x).to(dev) for x in (sc, dl, pr))
    r1 = r2 = r3 = None
    if lib is not None:
        w4 = (C.c_float * 4)(10.0, 10.0, 5.0, 5.0)
        r1, r2, r3 = torch.zeros((B, N), device=dev), torch.zeros((B, N, 4), device=dev), torch.zeros((B, N), device=dev)
        assert lib.ref_predictor_decode(B, C.c_void_p(scd.data_ptr()), C.c_void_p(dld.data_ptr()), C.c_void_p(prd.data_ptr()),
                                        C.c_void_p(r1.data_ptr()), C.c_void_p(r2.data_ptr()), C.c_void_p(r3.data_ptr()), N, Cc,
                                        800, 1067, w4) == 0
    o1, o2, o3 = (torch.zeros((B, N), device=dev), torch.zeros((B, N, 4), device=dev), torch.zeros((B, N), device=dev))
    assert P.PredictorDecodePlugin(N, 800, 1067, (10.0, 10.0, 5.0, 5.0), Cc).enqueue(B, [scd, dld, prd], [o1, o2, o3], ws) == 0
    G.equal("predictor_decode.scores", _np(o1), _np(r1))
    G.equal("predictor_decode.classes", _np(o3), _np(r3))
    # BatchedNms below is fed the reference's outputs: scores / classes are bit-equal to ours, boxes are stored whole
    r2 = torch.from_numpy(G.array("predictor_decode.boxes", _np(r2))).to(dev)
    np.testing.assert_allclose(o2.cpu().numpy(), r2.cpu().numpy(), rtol=3e-7, atol=1e-4)
    r1, r3 = o1, o3
    for method in (0, 1, 2):
        q1 = q2 = q3 = None
        if lib is not None:
            q1, q2, q3 = torch.zeros((B, 100), device=dev), torch.zeros((B, 100, 4), device=dev), torch.zeros((B, 100), device=dev)
            for b in range(B):  # same batch>1 bug as RpnNms (BatchedNms.cu:134 vs :146-148): one reference call per image
                assert lib.ref_batched_nms(method, 1, C.c_void_p(r1[b].data_ptr()), C.c_void_p(r2[b].data_ptr()),
                                           C.c_void_p(r3[b].data_ptr()), C.c_void_p(q1[b].data_ptr()), C.c_void_p(q2[b].data_ptr()),
                                           C.c_void_p(q3[b].data_ptr()), N, 100, C.c_float(0.5)) == 0
        p1, p2, p3 = torch.zeros((B, 100), device=dev), torch.zeros((B, 100, 4), device=dev), torch.zeros((B, 100), device=dev)
        assert P.BatchedNmsPlugin(method, 0.5, 100, N).enqueue(B, [r1, r2, r3], [p1, p2, p3], ws) == 0
        from oracle import oracle as O
        _, ob_, _ = O.batched_nms(method, r1.cpu().numpy(), r2.cpu().numpy(), r3.cpu().numpy(), 100, 0.5)
        info = f"method {method}: rows differing from the oracle: ours {int((p2.cpu().numpy() != ob_).any(-1).sum())}"
        G.close(f"batched_nms.{method}.scores", _np(p1), _np(q1), rtol=1e-6, atol=0, msg=info)
        G.equal(f"batched_nms.{method}.boxes", _np(p2), _np(q2), msg=info)
        G.equal(f"batched_nms.{method}.classes", _np(p3), _np(q3), msg=info)


def test_roi_align_and_mask_rcnn_inference_vs_reference_functions(dev, oracle):
    """roiAlign / maskRcnnInference of rcnn/*.cu (one launch + cudaDeviceSynchronize per image there) vs one launch
    for the batch here: same CUDA compiler, same expressions -> identical floats."""
    lib = G.lib("libref_rcnn.so")
    rng = np.random.default_rng(470)
    B, N, Cc, H, W, Pp = 2, 96, 80, 50, 67, 14
    feat = rng.standard_normal((B, Cc, H, W)).astype(np.float32)
    x1 = rng.uniform(-40, 1000, (B, N)); y1 = rng.uniform(-40, 760, (B, N))
    w = np.exp(rng.uniform(np.log(8), np.log(900), (B, N))); h = np.exp(rng.uniform(np.log(8), np.log(700), (B, N)))
    rois = np.stack([x1, y1, x1 + w, y1 + h], -1).astype(np.float32)
    rois[0, 0] = [100, 100, 100, 100]        # zero-size proposal: count = 0 -> NaN, like the reference
    rois[0, 1] = [300, 300, 200, 250]        # negative size
    rois[1, 0] = [-500, -500, -300, -300]    # entirely outside the feature map
    xi = rng.uniform(0, 700, N); yi = rng.uniform(0, 500, N)
    wi = np.exp(rng.uniform(np.log(8), np.log(300), N)); hi = np.exp(rng.uniform(np.log(8), np.log(250), N))
    rois_in = np.stack([xi, yi, xi + wi, yi + hi], -1).astype(np.float32)
    fd, rd = torch.from_numpy(feat).to(dev), torch.from_numpy(rois).to(dev)
    rois[1, 1] = [0, 0, 1067, 800]           # the whole map: the window of a channel is 50 x 67 cells (several passes)
    rois[1, 2] = [5, 5, 9, 9]                # a fraction of one cell
    rois[1, 3] = [1060, 790, 1200, 900]      # hangs over the bottom-right corner
    for sampling in (0, 2, 5, 19):           # 19: 14 * 19 = 266 table entries per axis > 256 -> coordinates on the fly
        r = None
        if lib is not None:
            ref = torch.zeros((B, N, Cc, Pp, Pp), device=dev)
            assert lib.ref_roi_align(B, C.c_void_p(rd.data_ptr()), C.c_void_p(fd.data_ptr()), C.c_void_p(ref.data_ptr()), Pp,
                                     C.c_float(1 / 16), sampling, N, Cc, H, W) == 0
            r = ref.cpu().numpy()
        plug = P.RoiAlignPlugin(Pp, 1 / 16, sampling, N, Cc)
        plug.configurePlugin([(N, 4), (Cc, H, W)])
        for mode in (None, L.ROI_WINDOW, L.ROI_DIRECT):  # the shared-memory window kernel (default) and the round-1 kernel
            got = torch.full((B, N, Cc, Pp, Pp), -3.0, device=dev)
            assert plug.enqueue(B, [rd, fd], [got], mode=mode) == 0
            torch.cuda.synchronize()
            G.equal(f"roi_align.{sampling}", got.cpu().numpy(), r, nan_ok=True, msg=(sampling, mode))   # bit-identical, NaNs included
        if sampling > 2:
            continue
        # CPU restatement (no FMA contraction) on proposals inside the feature map: at the `x > width -> 0` border of
        # bilinear_interpolate a 1-ulp difference in a sample coordinate flips a whole tap, which only the same-compiler
        # comparison above can pin
        orc = oracle.roi_align(rois_in, feat[1], Pp, 1 / 16, sampling)
        got_in = torch.empty((1, N, Cc, Pp, Pp), device=dev)
        assert plug.enqueue(1, [torch.from_numpy(rois_in).to(dev), fd[1:2].contiguous()], [got_in]) == 0
        np.testing.assert_allclose(got_in[0].cpu().numpy(), orc, rtol=0, atol=2e-5)
    # MaskRcnnInference
    D, nc, S = 100, 80, 14
    masks = rng.standard_normal((B, D, nc, S, S)).astype(np.float32) * 3
    idx = rng.integers(0, nc, (B, D)).astype(np.float32)
    idx[0, 5] = -1.0
    idx[1, 7] = float(nc)                      # out of range: the row is not written
    md, idd = torch.from_numpy(masks).to(dev), torch.from_numpy(idx).to(dev)
    ref = None
    if lib is not None:
        ref = torch.full((B, D, S, S), 9.0, device=dev)
        assert lib.ref_mask_rcnn_inference(B, C.c_void_p(idd.data_ptr()), C.c_void_p(md.data_ptr()), C.c_void_p(ref.data_ptr()),
                                           D, S, nc) == 0
    got = torch.full((B, D, S, S), 9.0, device=dev)
    assert P.MaskRcnnInferencePlugin(D, S, nc).enqueue(B, [idd, md], [got]) == 0
    torch.cuda.synchronize()
    G.equal("mask_rcnn_inference", got.cpu().numpy(), _np(ref))
    assert torch.all(got[0, 5] == 9.0) and torch.all(got[1, 7] == 9.0)
    exp = oracle.mask_rcnn_inference(idx[1], masks[1], out=np.full((D, S, S), 9.0, np.float32))
    np.testing.assert_allclose(got[1].cpu().numpy(), exp, rtol=3e-7, atol=1e-7)
