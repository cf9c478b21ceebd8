"""GPU parity: RetinaFace Decode_TRT, Faster R-CNN plugins, batched letterbox pre-process -- all through
the C ABI (tensorrtx_b200.plugins -> libtrtx_hot.so) against the CPU oracle."""
import numpy as np
import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P
from tensorrtx_b200 import synth

pytestmark = pytest.mark.gpu
ATOL = 1e-4
RTOL_EXP = 2e-6  # columns that pass through expf (CUDA expf vs glibc expf), see test_yolo_gpu.py


def _ws(nbytes, dev):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=dev)


# ------------------------------------------------------------------ RetinaFace ----------------
@pytest.mark.parametrize("B,h,w,seed", [(1, 640, 640, 0), (4, 640, 640, 1), (2, 480, 640, 2), (2, 488, 648, 3)])
def test_retina_decode_parity(oracle, dev, B, h, w, seed):
    heads = synth.retina_heads(B, seed=seed, in_h=h, in_w=w)
    ref, _ = oracle.retina_decode(heads, in_h=h, in_w=w, gate=0.02)
    plug = P.DecodePlugin(h, w)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in heads], [out], _ws(plug.getWorkspaceSize(B), dev)) == 0
    got = out.cpu().numpy()
    assert np.array_equal(got[:, 0], ref[:, 0]) and ref[:, 0].min() > 50
    for b in range(B):
        n = int(ref[b, 0])
        np.testing.assert_allclose(got[b, 1:1 + n * 15], ref[b, 1:1 + n * 15], atol=ATOL, rtol=RTOL_EXP)


def test_retina_nms_with_landmarks(oracle, dev):
    B = 3
    heads = synth.retina_heads(B, seed=5)
    ref, _ = oracle.retina_decode(heads)
    tp = oracle.retina_total_priors(640, 640)
    comp, idx = P.batch_nms(torch.from_numpy(ref).to(dev), B, ref.shape[1], P.float_le_threshold(0.1), 0.4,
                            box_format=L.BOX_RETINA, det_floats=15, max_det=2048, extra_floats=10, extra_offset=5,
                            return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        res, src = oracle.nms(2, ref[b], tp, 15, 0.1, 0.4)
        n = int(comp[b, 0])
        assert n == len(res) and n > 10
        # single class: reference order = conf descending
        assert np.array_equal(idx[b, :n], src)
        rows = comp[b, 1:1 + n * 17].reshape(n, 17)
        assert np.array_equal(rows[:, :5], res[:, :5])
        assert np.array_equal(rows[:, 7:17], res[:, 5:15])  # landmarks travel with the box


# ------------------------------------------------------------------ Faster R-CNN --------------
def test_rpn_decode_parity(oracle, dev):
    B, A, H, W, top_n = 3, 15, 50, 67, 6000
    scores, deltas = synth.rpn_inputs(B, seed=1, A=A, H=H, W=W)
    anchors = synth.rcnn_anchors()
    ref_s, ref_b = oracle.rpn_decode(scores, deltas, 800, 1067, 16.0, anchors, top_n)
    plug = P.RpnDecodePlugin(top_n, anchors, 16.0, 800, 1067, H, W)
    os_ = torch.zeros((B, top_n), device=dev)
    ob = torch.zeros((B, top_n, 4), device=dev)
    rc = plug.enqueue(B, [torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)], [os_, ob],
                      _ws(plug.getWorkspaceSize(B), dev))
    assert rc == 0
    assert np.array_equal(os_.cpu().numpy(), ref_s)       # same ordered top-6000, same -FLT_MAX markers
    np.testing.assert_allclose(ob.cpu().numpy(), ref_b, atol=ATOL, rtol=RTOL_EXP)


def test_rpn_decode_fewer_than_topn(oracle, dev):
    B, A, H, W, top_n = 2, 15, 8, 9, 2000   # 1080 scores < top_n: unsorted pass-through + -FLT_MAX fill
    scores, deltas = synth.rpn_inputs(B, seed=2, A=A, H=H, W=W)
    anchors = synth.rcnn_anchors()
    ref_s, ref_b = oracle.rpn_decode(scores, deltas, 128, 144, 16.0, anchors, top_n)
    plug = P.RpnDecodePlugin(top_n, anchors, 16.0, 128, 144, H, W)
    os_ = torch.zeros((B, top_n), device=dev)
    ob = torch.zeros((B, top_n, 4), device=dev)
    assert plug.enqueue(B, [torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)], [os_, ob], _ws(256, dev)) == 0
    n = A * H * W
    assert np.array_equal(os_.cpu().numpy(), ref_s)
    np.testing.assert_allclose(ob.cpu().numpy()[:, :n], ref_b[:, :n], atol=ATOL, rtol=RTOL_EXP)


@pytest.mark.parametrize("seed,thr", [(0, 0.7), (1, 0.3)])
def test_rpn_nms_parity(oracle, dev, seed, thr):
    B, A, H, W, pre, post = 2, 15, 50, 67, 6000, 1000
    scores, deltas = synth.rpn_inputs(B, seed=10 + seed, A=A, H=H, W=W)
    s6, b6 = oracle.rpn_decode(scores, deltas, 800, 1067, 16.0, synth.rcnn_anchors(), pre)
    ref = oracle.rpn_nms(s6, b6, post, thr)
    plug = P.RpnNmsPlugin(thr, post, pre)
    ob = torch.zeros((B, post, 4), device=dev)
    assert plug.enqueue(B, [torch.from_numpy(s6).to(dev), torch.from_numpy(b6).to(dev)], [ob], _ws(256, dev)) == 0
    assert np.array_equal(ob.cpu().numpy(), ref)          # gathered boxes are copies: bit-exact, same order


def test_rpn_nms_fewer_survivors_than_post(oracle, dev):
    # heavy overlap: < post survivors -> suppressed boxes follow in sorted order (RpnNms.cu:111-117)
    rng = np.random.default_rng(3)
    B, pre, post = 2, 700, 300
    xy = rng.uniform(0, 60, (B, pre, 2)).astype(np.float32)
    wh = rng.uniform(80, 120, (B, pre, 2)).astype(np.float32)
    boxes = np.concatenate([xy, xy + wh], -1)
    scores = rng.standard_normal((B, pre)).astype(np.float32)
    scores[:, ::7] = -np.finfo(np.float32).max            # empty boxes marked by RpnDecode
    ref = oracle.rpn_nms(scores, boxes, post, 0.5)
    plug = P.RpnNmsPlugin(0.5, post, pre)
    ob = torch.zeros((B, post, 4), device=dev)
    assert plug.enqueue(B, [torch.from_numpy(scores).to(dev), torch.from_numpy(boxes).to(dev)], [ob], _ws(256, dev)) == 0
    assert np.array_equal(ob.cpu().numpy(), ref)


def test_predictor_decode_parity(oracle, dev):
    B, N, Cc = 2, 1000, 80
    scores, deltas, props = synth.predictor_inputs(B, seed=4, N=N, Ccls=Cc)
    w = (10.0, 10.0, 5.0, 5.0)
    rs, rb, rc_ = oracle.predictor_decode(scores, deltas, props, 800, 1067, w)
    plug = P.PredictorDecodePlugin(N, 800, 1067, w, Cc)
    os_, ob, oc = torch.zeros((B, N), device=dev), torch.zeros((B, N, 4), device=dev), torch.zeros((B, N), device=dev)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in (scores, deltas, props)], [os_, ob, oc], _ws(256, dev)) == 0
    assert np.array_equal(os_.cpu().numpy(), rs)
    assert np.array_equal(oc.cpu().numpy(), rc_)
    np.testing.assert_allclose(ob.cpu().numpy(), rb, atol=ATOL, rtol=RTOL_EXP)


@pytest.mark.parametrize("method", [0, 1, 2])
def test_batched_nms_parity(oracle, dev, method):
    B, N, Cc = 3, 1000, 80
    scores, deltas, props = synth.predictor_inputs(B, seed=6 + method, N=N, Ccls=Cc)
    s, b, c = oracle.predictor_decode(scores, deltas, props, 800, 1067, (10.0, 10.0, 5.0, 5.0))
    rs, rb, rc_ = oracle.batched_nms(method, s, b, c, 100, 0.5)
    plug = P.BatchedNmsPlugin(method, 0.5, 100, N)
    os_, ob, oc = torch.zeros((B, 100), device=dev), torch.zeros((B, 100, 4), device=dev), torch.zeros((B, 100), device=dev)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in (s, b, c)], [os_, ob, oc], _ws(256, dev)) == 0
    got_s = os_.cpu().numpy()
    if method == 2:  # gaussian decay goes through expf
        np.testing.assert_allclose(got_s, rs, atol=1e-6, rtol=RTOL_EXP)
    else:
        assert np.array_equal(got_s, rs)
    assert np.array_equal(ob.cpu().numpy(), rb)
    assert np.array_equal(oc.cpu().numpy(), rc_)


def test_rcnn_workspace_idiom(dev):
    plug = P.BatchedNmsPlugin(1, 0.5, 100, 1000)
    assert plug.getWorkspaceSize(8) > 0        # null workspace -> required bytes (BatchedNmsPlugin.h:106-114)
    assert P.RpnNmsPlugin(0.7, 1000, 6000).getWorkspaceSize(8) > 0


def test_retina_full_config_b16(oracle, dev):
    """BASELINE configs[2]: RetinaFace batch 16 at 640x640 -- decode and NMS of every image against the oracle."""
    B = 16
    heads = synth.retina_heads(B, seed=21)
    ref, _ = oracle.retina_decode(heads, in_h=640, in_w=640, gate=0.02)
    plug = P.DecodePlugin(640, 640)
    out = torch.zeros((B, plug.output_elems()), dtype=torch.float32, device=dev)
    assert plug.enqueue(B, [torch.from_numpy(x).to(dev) for x in heads], [out], _ws(plug.getWorkspaceSize(B), dev)) == 0
    got = out.cpu().numpy()
    assert np.array_equal(got[:, 0], ref[:, 0]) and ref[:, 0].min() > 50
    comp, idx = P.batch_nms(out, B, plug.output_elems(), P.float_le_threshold(0.1), 0.4, box_format=L.BOX_RETINA, det_floats=15,
                            max_det=2048, extra_floats=10, extra_offset=5, return_index=True)
    comp, idx = comp.cpu().numpy(), idx.cpu().numpy()
    tp = oracle.retina_total_priors(640, 640)
    for b in range(B):
        n = int(ref[b, 0])
        np.testing.assert_allclose(got[b, 1:1 + n * 15], ref[b, 1:1 + n * 15], atol=ATOL, rtol=RTOL_EXP)
        res, src = oracle.nms(2, got[b], tp, 15, 0.1, 0.4)    # NMS of OUR rows: kept sets must agree bit for bit
        k = int(comp[b, 0])
        assert k == len(res) and np.array_equal(idx[b, :k], src)
        assert np.array_equal(comp[b, 1:1 + k * 17].reshape(k, 17)[:, :5], res[:, :5])


def test_rcnn_full_config_b8_chain(oracle, dev):
    """BASELINE configs[3]: Faster R-CNN batch 8 -- RpnDecode -> RpnNms -> PredictorDecode -> BatchedNms chained on the
    device, every stage of every image against the oracle fed with the SAME stage inputs."""
    B, A, H, W, pre, post, N, Cc = 8, 15, 50, 67, 6000, 1000, 1000, 80
    anchors = synth.rcnn_anchors()
    scores, deltas = synth.rpn_inputs(B, seed=31, A=A, H=H, W=W)
    d_s, d_b = torch.zeros((B, pre), device=dev), torch.zeros((B, pre, 4), device=dev)
    p1 = P.RpnDecodePlugin(pre, anchors, 16.0, 800, 1067, H, W)
    assert p1.enqueue(B, [torch.from_numpy(scores).to(dev), torch.from_numpy(deltas).to(dev)], [d_s, d_b],
                      _ws(p1.getWorkspaceSize(B), dev)) == 0
    r_s, r_b = oracle.rpn_decode(scores, deltas, 800, 1067, 16.0, anchors, pre)
    assert np.array_equal(d_s.cpu().numpy(), r_s)
    # x1 = ctr - w/2 with w = expf(..) * anchor up to ~1000 px: one ulp of CUDA-vs-glibc expf at that scale (1.2e-4) survives the
    # cancellation into a small coordinate, so the absolute slack is 5 ulp(1024) here (vs the reference KERNEL: <= 2 ulp,
    # tests/test_vs_reference_gpu.py::test_rcnn_vs_reference_functions)
    np.testing.assert_allclose(d_b.cpu().numpy(), r_b, atol=6e-4, rtol=RTOL_EXP)
    props = torch.zeros((B, post, 4), device=dev)
    assert P.RpnNmsPlugin(0.7, post, pre).enqueue(B, [d_s, d_b], [props], _ws(256, dev)) == 0
    assert np.array_equal(props.cpu().numpy(), oracle.rpn_nms(d_s.cpu().numpy(), d_b.cpu().numpy(), post, 0.7))
    cls_scores, box_deltas, _ = synth.predictor_inputs(B, seed=32, N=N, Ccls=Cc)
    w = (10.0, 10.0, 5.0, 5.0)
    os_, ob, oc = torch.zeros((B, N), device=dev), torch.zeros((B, N, 4), device=dev), torch.zeros((B, N), device=dev)
    assert P.PredictorDecodePlugin(N, 800, 1067, w, Cc).enqueue(
        B, [torch.from_numpy(cls_scores).to(dev), torch.from_numpy(box_deltas).to(dev), props], [os_, ob, oc], _ws(256, dev)) == 0
    rs, rb, rc_ = oracle.predictor_decode(cls_scores, box_deltas, props.cpu().numpy(), 800, 1067, w)
    assert np.array_equal(os_.cpu().numpy(), rs) and np.array_equal(oc.cpu().numpy(), rc_)
    np.testing.assert_allclose(ob.cpu().numpy(), rb, atol=6e-4, rtol=RTOL_EXP)
    for method in (0, 1):
        fs, fb, fc = torch.zeros((B, 100), device=dev), torch.zeros((B, 100, 4), device=dev), torch.zeros((B, 100), device=dev)
        assert P.BatchedNmsPlugin(method, 0.5, 100, N).enqueue(B, [os_, ob, oc], [fs, fb, fc], _ws(256, dev)) == 0
        es, eb, ec = oracle.batched_nms(method, os_.cpu().numpy(), ob.cpu().numpy(), oc.cpu().numpy(), 100, 0.5)
        assert np.array_equal(fs.cpu().numpy(), es) and np.array_equal(fb.cpu().numpy(), eb) and np.array_equal(fc.cpu().numpy(), ec)


# ------------------------------------------------------------------ pre-process ---------------
def _bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint16)


@pytest.mark.parametrize("h,w", [(640, 640), (1080, 1920), (517, 333), (64, 48), (640, 480), (400, 640), (640, 636)])
@pytest.mark.parametrize("odt", [torch.float32, torch.float16])
def test_letterbox_parity(oracle, dev, h, w, odt):
    B = 3
    fr = synth.frames(B, seed=h + w, h=h, w=w)
    dst = torch.zeros((B, 3, 640, 640), dtype=odt, device=dev)
    P.cuda_batch_preprocess([torch.from_numpy(f).to(dev) for f in fr], dst, 640, 640)
    got = dst.cpu().numpy()
    for b in range(B):
        # the exact model: fp32 bit for bit, fp16 its fp32 value rounded to nearest
        ref = oracle.warpaffine(fr[b], 640, 640, contracted=True)
        if odt == torch.float16:
            ref = ref.astype(np.float16)
        assert np.array_equal(_bits(got[b]), _bits(ref)), (h, w, b, int(np.sum(got[b] != ref)))


def test_letterbox_mixed_sizes_one_launch(oracle, dev):
    sizes = [(480, 640), (720, 1280), (1000, 300), (33, 47)]
    frs = [synth.frames(1, seed=i, h=h, w=w)[0] for i, (h, w) in enumerate(sizes)]
    dst = torch.zeros((len(sizes), 3, 416, 608), dtype=torch.float32, device=dev)
    P.cuda_batch_preprocess([torch.from_numpy(f).to(dev) for f in frs], dst, 608, 416)
    got = dst.cpu().numpy()
    for b, f in enumerate(frs):
        assert np.array_equal(_bits(got[b]), _bits(oracle.warpaffine(f, 608, 416, contracted=True))), (b, f.shape)


def test_pipeline_e2e_matches_oracle(oracle, dev):
    from tensorrtx_b200.pipeline import DetectionPipeline

    B = 4
    heads = synth.yolov8_heads(B, seed=90)
    fr = torch.from_numpy(synth.frames(B, seed=91)).pin_memory()
    pipe = DetectionPipeline(B, device=dev)
    hd = [torch.from_numpy(h).to(dev) for h in heads]
    out = pipe.run(fr, hd)
    torch.cuda.synchronize()
    out = out.numpy()
    ref, _ = oracle.yolov8_decode(heads)
    for b in range(B):
        res, _ = oracle.nms(0, ref[b], 1000, 90, 0.5, 0.45)
        n = int(out[b, 0])
        assert n == len(res)
        np.testing.assert_allclose(out[b, 1:1 + n * 7].reshape(n, 7)[:, :6], res[:, :6], atol=ATOL, rtol=0)
    assert np.array_equal(_bits(pipe.net_input[1].cpu().numpy()), _bits(oracle.warpaffine(fr[1].numpy(), 640, 640, contracted=True)))
    # graph replay gives the same bytes
    g = pipe.capture(lambda: pipe.run(fr, hd))
    first = out.copy()
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(pipe.out_host.numpy(), first)


@pytest.mark.parametrize("variant", [0, 1])
def test_process_mask_matches_oracle(oracle, dev, variant):
    """process_mask of the seg drivers (host code in the reference) as one fused GPU launch for the batch."""
    rng = np.random.default_rng(60 + variant)
    B, K, M, R = 3, 50, 12, 39
    proto = rng.standard_normal((B, 32, 160, 160)).astype(np.float32)
    dets = np.zeros((B, 1 + K * R), np.float32)
    counts = [12, 0, 5]
    for b in range(B):
        dets[b, 0] = counts[b]
        rows = dets[b, 1:].reshape(K, R)
        for i in range(counts[b]):
            if variant == 0:
                rows[i, :4] = [rng.uniform(-40, 600), rng.uniform(-40, 600), rng.uniform(1, 300), rng.uniform(1, 300)]
            else:
                rows[i, :4] = [rng.uniform(20, 620), rng.uniform(20, 620), rng.uniform(1, 300), rng.uniform(1, 300)]
            rows[i, 4:7] = [0.9, 3.0, 1.0]
            rows[i, 7:39] = rng.standard_normal(32) * 0.5
    sentinel = -7.0
    out = torch.full((B, M, 640, 640), sentinel, dtype=torch.float32, device=dev)
    got = P.process_mask(torch.from_numpy(proto).to(dev), torch.from_numpy(dets).to(dev), K, R, 7, M, 640, 640,
                         variant=variant, out=out)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    for b in range(B):
        rows = dets[b, 1:].reshape(K, R)
        n = min(counts[b], M)
        for i in range(n):
            ref = oracle.process_mask(variant, proto[b], rows[i, :4], rows[i, 7:39])
            assert np.abs(got[b, i] - ref).max() <= 2e-6   # CUDA expf vs glibc expf inside the sigmoid
            assert (got[b, i] > 0).sum() == (ref > 0).sum()
        assert np.all(got[b, n:] == sentinel)              # slots past the image's detections are not written



@pytest.mark.parametrize("img_w,img_h", [(1920, 1080), (1080, 1920), (640, 640), (500, 375), (333, 1001)])
def test_scale_mask_matches_oracle(oracle, dev, img_w, img_h):
    """scale_mask (yolov8/src/postprocess.cpp:207-226) for a stack of device masks: crop rectangle pinned to the reference's
    compiled code (tests/test_oracle_vs_ref_cpu.py), resize = OpenCV's float bilinear kernel (pinned to cv2 on the CPU)."""
    import ctypes as C
    rng = np.random.default_rng(img_w + img_h)
    n = 3
    masks = rng.uniform(0, 1, (n, 640, 640)).astype(np.float32)
    out = P.scale_mask(torch.from_numpy(masks).to(dev), img_w, img_h)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    r = (C.c_int * 4)()
    assert L.load().trtx_scale_mask_rect(640, 640, img_w, img_h, r) == 0
    x, y, w, h = list(r)
    for i in range(n):
        ref = oracle.resize_bilinear(np.ascontiguousarray(masks[i, y:y + h, x:x + w]), img_h, img_w)
        assert np.array_equal(got[i], ref)      # same operations in the same order, every product and sum rounded: bit-exact
