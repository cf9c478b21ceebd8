"""The YOLO instance-mask kernels (tensorrtx_b200/csrc/mask.cu) on every shape class: process_mask_kernel, scale_mask_kernel
and the fused segmentation post-process (seg_rows_kernel + seg_canvas_kernel), against the float64 reference and its error
bound of tests/test_mask_paths_cpu.py, the CPU oracle, and each other.

Shape classes: nets 640^2, 640 x 480 (partial tile rows), 544^2 (partial tiles on both axes), 1280^2, 64^2 (one tile) and
1024 x 256; 1, 32 and 64 coefficients; rows (39, 7), (38, 6) and the block at the end of a longer row.  Every call writes
into sentinel-filled buffers, and the bytes a call must not write are checked.  Each class prints the largest
|GPU - float64| next to its bound, and the fused post-process the number of canvas pixels excused because |S64 - 0.5| lies
within the bound of S (run with -s to see them)."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import seg_post as SP
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

from test_mask_paths_cpu import (NET_SHAPES, SHAPES, V5, V8, Shape, canvas64, downscale_cells, edge_boxes, excess,
                                 largest_seg_net, make_dets, make_proto, process_mask64, random_boxes, scale_mask64,
                                 undefined_boxes)

pytestmark = pytest.mark.gpu
SENTINEL, ROW_SENTINEL, CANVAS_SENTINEL = -7.0, -9.0, 77
TINY = [(1, 1), (2, 2), (4, 4), (8, 8)]
MIXED = [(1920, 1080), (333, 1001), (1282, 719)]


def _process_mask(shape, variant, proto, dets, K, M, out=None):
    R, off = shape.row
    return P.process_mask(torch.from_numpy(proto).cuda(), torch.from_numpy(dets).cuda(), K, R, off, M, shape.net_w,
                          shape.net_h, variant=variant, out=out)


def _check_mask(oracle, shape, variant, proto, row, got):
    """one process_mask slot against the float64 reference (bound) and the oracle (2e-6) -> (max |err|, max bound)"""
    R, off = shape.row
    c = row[off:off + shape.nm]
    ref, bound = process_mask64(variant, proto, row[:4], c, shape.net_w, shape.net_h)
    assert excess(got, ref, bound) <= 1.0, (shape.id, variant, row[:4])
    orc = oracle.process_mask(variant, proto, row[:4], c, shape.net_w, shape.net_h)
    assert np.abs(got - orc).max() <= 2e-6, (shape.id, variant, row[:4])   # CUDA expf vs glibc expf
    return float(np.abs(got - ref).max()), float(bound.max())


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s.id)
def test_process_mask(oracle, shape):
    """Tile-edge, 0- and 1-cell, whole-mask, half-outside, .5-cell (V5) and random boxes on one image, undefined and random
    ones on another; max_masks above both counts, so the last slots must keep the sentinel."""
    rng = np.random.default_rng(3000 + shape.net_w + shape.net_h + shape.nm + shape.row[0])
    R, off = shape.row
    for variant in (V8, V5):
        boxes = [edge_boxes(variant, shape.net_w, shape.net_h) + random_boxes(rng, variant, shape.net_w, shape.net_h, 6),
                 undefined_boxes(variant, shape.net_w, shape.net_h)[::2] + random_boxes(rng, variant, shape.net_w, shape.net_h, 2)]
        K = M = max(len(b) for b in boxes) + 2
        proto = make_proto(rng, shape, 2)
        dets = np.stack([make_dets(rng, shape, b, pad_rows=K - len(b)) for b in boxes])
        out = torch.full((2, M, shape.net_h, shape.net_w), SENTINEL, device="cuda")
        _process_mask(shape, variant, proto, dets, K, M, out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        worst = bound = 0.0
        for b in range(2):
            n = len(boxes[b])
            rows = dets[b, 1:].reshape(K, R)
            for k in range(n):
                e, q = _check_mask(oracle, shape, variant, proto[b], rows[k], got[b, k])
                worst, bound = max(worst, e), max(bound, q)
            assert np.all(got[b, n:] == SENTINEL)
        print(f"process_mask {shape.id} v{variant}: max |GPU - f64| {worst:.3e}, bound {bound:.3e}")


@pytest.mark.parametrize("offset", [4, 8, 12])
def test_process_mask_unaligned_out(oracle, offset):
    """An output based 4, 8 or 12 bytes past 16-byte alignment takes the scalar store on every pixel: equal bit for bit to
    the aligned call, and the floats around it keep their sentinel."""
    shape = Shape(544, 544)
    rng = np.random.default_rng(4000 + offset)
    boxes = edge_boxes(V5, 544, 544)[-12:] + random_boxes(rng, V5, 544, 544, 4)
    K = M = len(boxes)
    proto = make_proto(rng, shape)
    dets = make_dets(rng, shape, boxes)[None]
    aligned = _process_mask(shape, V5, proto, dets, K, M)
    n = M * 544 * 544
    buf = torch.full((n + 8,), SENTINEL, device="cuda")
    e = offset // 4
    assert buf[e:].data_ptr() % 16 == offset
    _process_mask(shape, V5, proto, dets, K, M, buf[e:e + n].view(1, M, 544, 544))
    torch.cuda.synchronize()
    assert torch.equal(buf[e:e + n].view(1, M, 544, 544), aligned)
    assert torch.all(buf[:e] == SENTINEL) and torch.all(buf[e + n:] == SENTINEL)
    rows = dets[0, 1:].reshape(K, shape.row[0])
    got = aligned.cpu().numpy()
    for k in (0, K - 1):
        _check_mask(oracle, shape, V5, proto[0], rows[k], got[0, k])


def test_process_mask_grid_limit(oracle):
    """batch * max_masks = 65 535 on a 64^2 net (one CTA per slot in grid z) runs; 65 536 is refused and writes nothing.
    Rows repeat 7 boxes, so every slot equals the first slot of its box, which is checked against the references."""
    shape = Shape(64, 64)
    rng = np.random.default_rng(65535)
    pattern = edge_boxes(V8, 64, 64)[:4] + random_boxes(rng, V8, 64, 64, 3)
    total = 65536
    out = torch.full((total, 64, 64), SENTINEL, device="cuda")   # 1.07 GB
    B, M = 4, 16384
    proto = make_proto(rng, shape, 5)
    dets = np.stack([make_dets(rng, shape, [pattern[i % 7] for i in range(M)]) for _ in range(5)])
    for b in range(5):
        base = dets[b, 1:].reshape(M, shape.row[0])
        base[:, :] = base[np.arange(M) % 7]
    with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
        _process_mask(shape, V8, proto[:B], dets[:B], M, M, out.view(B, M, 64, 64))
    torch.cuda.synchronize()
    assert torch.all(out == SENTINEL)
    B, M = 5, 13107   # 65 535
    _process_mask(shape, V8, proto, np.ascontiguousarray(dets[:, :1 + M * shape.row[0]]), M, M, out[:B * M].view(B, M, 64, 64))
    torch.cuda.synchronize()
    assert torch.all(out[B * M:] == SENTINEL)
    v = out[:B * M].view(B, M, 64, 64)
    for b in range(B):
        rows = dets[b, 1:].reshape(-1, shape.row[0])
        for p in range(7):
            first = v[b, p]
            assert torch.equal(v[b, p::7], first.expand_as(v[b, p::7]))
            _check_mask(oracle, shape, V8, proto[b], rows[p], first.cpu().numpy())


def test_undefined_boxes_give_zero_masks(oracle):
    """A box for which one of get_downscale_rect's conversions is undefined gets an all-zero mask from the kernel and the
    oracle alike; one whose conversions are defined is evaluated (e.g. V8 width +inf: right clamps to the net).  Named V5
    boxes: a defined left with a width past INT_MAX cells (a saturating width gave a full-width band), and defined rx, rw
    (ry, rh) both near -2e9, whose sum below INT_MIN must not wrap to a large positive end."""
    shape = Shape(640, 640)
    rng = np.random.default_rng(77)
    named = [[1e9, 320, 1e10, 100], [-1.2e10, 320, -8e9, 100], [320, -1.2e10, 100, -8e9]]
    for variant in (V8, V5):
        boxes = undefined_boxes(variant, 640, 640)
        K = len(boxes)
        proto = make_proto(rng, shape)
        dets = make_dets(rng, shape, boxes)[None]
        got = _process_mask(shape, variant, proto, dets, K, K).cpu().numpy()[0]
        rows = dets[0, 1:].reshape(K, 39)
        zero = 0
        for k in range(K):
            x0, x1, y0, y1 = downscale_cells(variant, rows[k, :4], 640, 640)
            orc = oracle.process_mask(variant, proto[0], rows[k, :4], rows[k, 7:39])
            if x0 >= x1 or y0 >= y1:
                assert not got[k].any() and not orc.any(), (variant, rows[k, :4])
                zero += 1
            else:
                assert got[k].any()
                _check_mask(oracle, shape, variant, proto[0], rows[k], got[k])
        assert zero >= 20
        if variant == V5:
            for box in named:
                k = next(i for i, b in enumerate(boxes) if b == box)
                assert not got[k].any(), box


SCALE_FRAMES = [(1, 1), (2, 3), (3, 640), (333, 1001), (1282, 719), (1919, 1080), (7680, 4320)]


@pytest.mark.parametrize("net", [s for s in NET_SHAPES], ids=lambda s: f"net{s.net_w}x{s.net_h}")
def test_scale_mask(oracle, net):
    """scale_mask at every net (crop from trtx_scale_mask_rect): bit for bit with the oracle, within the float64 bound,
    into an output based 4 bytes past alignment with sentinels around it; a frame whose crop is empty is refused."""
    rng = np.random.default_rng(5000 + net.net_w + net.net_h)
    n = 2
    masks = torch.from_numpy(rng.uniform(0, 1, (n, net.net_h, net.net_w)).astype(np.float32)).cuda()
    mh = masks.cpu().numpy()
    for w, h in SCALE_FRAMES:
        crop = SP.scale_mask_rect(w, h, net.net_w, net.net_h)
        size = n * w * h
        buf = torch.full((size + 2,), SENTINEL, device="cuda")
        out = buf[1:1 + size].view(n, h, w)
        if min(crop[2:]) <= 0:
            with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
                P.scale_mask(masks, w, h, out=out)
            torch.cuda.synchronize()
            assert torch.all(buf == SENTINEL)
            continue
        P.scale_mask(masks, w, h, out=out)
        torch.cuda.synchronize()
        assert buf[0] == SENTINEL and buf[-1] == SENTINEL
        got = out.cpu().numpy()
        x, y, cw, ch = crop
        rows = None if w * h <= 2_000_000 else np.unique(np.linspace(0, h - 1, 48).astype(int))
        worst = 0.0
        for i in range(n):
            assert np.array_equal(got[i], oracle.resize_bilinear(np.ascontiguousarray(mh[i, y:y + ch, x:x + cw]), h, w))
            ref, bound = scale_mask64(mh[i].astype(np.float64), np.zeros(mh[i].shape), crop, w, h, rows)
            g = got[i] if rows is None else got[i][rows]
            assert excess(g, ref, bound) <= 1.0, ((w, h), i)
            worst = max(worst, float(np.abs(g - ref).max()))
        print(f"scale_mask net{net.net_w}x{net.net_h} {w}x{h}: max |GPU - f64| {worst:.3e}, bound {bound.max():.3e}")


def _canvases(sizes, M):
    return [torch.full((M, h, w), CANVAS_SENTINEL, dtype=torch.uint8, device="cuda") for w, h in sizes]


def _seg(shape, variant, proto_d, dets_d, sizes, K, M, canvases):
    R, off = shape.row
    rows = torch.full((len(sizes), 1 + K * 6), ROW_SENTINEL, device="cuda")
    P.yolo_seg_postprocess(proto_d, dets_d, sizes, variant=variant, max_rows=K, row_floats=R, coeff_offset=off, max_masks=M,
                           net_w=shape.net_w, net_h=shape.net_h, rows_out=rows, canvases_out=canvases)
    torch.cuda.synchronize()
    return rows.cpu().numpy()


def _check_seg(shape, variant, proto, dets, sizes, K, M, canvases, rows_got, f64_rows=40):
    """The canvases against the library's process_mask -> scale_mask thresholded inside get_rect (array_equal, on the
    device) and against the float64 canvas except where |S64 - 0.5| is within S's bound -> (excused pixels, max |S err|,
    max bound)"""
    R, off = shape.row
    excused, worst, bound = 0, 0.0, 0.0
    for b, (w, h) in enumerate(sizes):
        masks = _process_mask(shape, variant, proto[b:b + 1], dets[b:b + 1], K, M)[0]
        assert rows_got[b, 0] == min(int(dets[b, 0]), K)
        n = min(int(dets[b, 0]), K, M)
        crop = SP.scale_mask_rect(w, h, shape.net_w, shape.net_h)
        src = dets[b, 1:].reshape(K, R)
        for k in range(n):
            rect = P.get_rect(w, h, src[k, :4], shape.net_w, shape.net_h, variant)
            assert tuple(int(v) for v in rows_got[b, 1 + 6 * k:5 + 6 * k]) == rect
            S = P.scale_mask(masks[k:k + 1].contiguous(), w, h)[0]
            x, y, rw, rh = rect
            x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + rw, w), min(y + rh, h)
            want = torch.zeros((h, w), dtype=torch.uint8, device="cuda")
            if x0 < x1 and y0 < y1:
                want[y0:y1, x0:x1] = torch.where(S[y0:y1, x0:x1] <= 0.5, 0, 255).to(torch.uint8)
            assert torch.equal(canvases[b][k], want), (shape.id, variant, (w, h), k)
            sel = None if w * h <= 300_000 else np.unique(np.linspace(0, h - 1, f64_rows).astype(int))
            c64, S64, sb = canvas64(variant, proto[b], src[k], shape, w, h, crop, rect, sel)
            got = canvases[b][k].cpu().numpy() if sel is None else canvases[b][k][torch.from_numpy(sel).cuda()].cpu().numpy()
            near = np.abs(S64 - 0.5) <= sb
            assert not np.any((got != c64) & ~near), (shape.id, variant, (w, h), k)
            excused += int(((got != c64) & near).sum())
            if rect[2] > 0 and rect[3] > 0 and x0 < x1 and y0 < y1:
                Sg = S.cpu().numpy() if sel is None else S[torch.from_numpy(sel).cuda()].cpu().numpy()
                assert excess(Sg, S64, sb) <= 1.0
                worst, bound = max(worst, float(np.abs(Sg - S64).max())), max(bound, float(sb.max()))
        assert torch.all(canvases[b][n:] == CANVAS_SENTINEL)   # slots at or past the count are not written
    return excused, worst, bound


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s.id)
def test_seg_postprocess(shape):
    """The fused post-process at every class: tiny frames (the caps at their hard limits 16 and 32) and mixed frames in one
    call, and (net classes) an 8K frame; both variants, with the edge, undefined and random boxes."""
    rng = np.random.default_rng(6000 + shape.net_w + shape.net_h + shape.nm + shape.row[0])
    sizes = [s for s in TINY + MIXED if min(SP.scale_mask_rect(*s, shape.net_w, shape.net_h)[2:]) > 0]
    for variant in (V8, V5):
        boxes = random_boxes(rng, variant, shape.net_w, shape.net_h, 8) + edge_boxes(variant, shape.net_w, shape.net_h)[-10:] + \
            undefined_boxes(variant, shape.net_w, shape.net_h)[::3]
        K = len(boxes)
        M = K - 2    # the last two rows have no canvas
        proto = make_proto(rng, shape, len(sizes))
        dets = np.stack([make_dets(rng, shape, boxes) for _ in sizes])
        canv = _canvases(sizes, M)
        rows = _seg(shape, variant, torch.from_numpy(proto).cuda(), torch.from_numpy(dets).cuda(), sizes, K, M, canv)
        excused, worst, bound = _check_seg(shape, variant, proto, dets, sizes, K, M, canv, rows)
        if shape in NET_SHAPES:
            big = [(7680, 4320)]
            d8 = make_dets(rng, shape, random_boxes(rng, variant, shape.net_w, shape.net_h, 4))[None]
            p8 = make_proto(rng, shape)
            c8 = _canvases(big, 4)
            r8 = _seg(shape, variant, torch.from_numpy(p8).cuda(), torch.from_numpy(d8).cuda(), big, 4, 4, c8)
            e8, w8, b8 = _check_seg(shape, variant, p8, d8, big, 4, 4, c8, r8)
            excused, worst, bound = excused + e8, max(worst, w8), max(bound, b8)
        print(f"seg {shape.id} v{variant}: max |S GPU - f64| {worst:.3e}, bound {bound:.3e}, {excused} canvas pixels "
              f"excused as near 0.5")


def test_seg_largest_net_and_refusal():
    """For a frame of a few pixels the canvas launch needs 96 bytes of shared memory per net column: 2408^2 is the largest
    square net that fits (and is bit-exact to the composition); 2412^2, and 2560^2 with a 4 x 4 frame (240 KB), are refused
    with TRTX_ERR_UNSUPPORTED before any launch and write nothing."""
    n = largest_seg_net()
    assert n == 2408
    rng = np.random.default_rng(2408)
    sizes = [(1, 1), (4, 4)]
    for net, ok in ((n, True), (n + 4, False), (2560, False)):
        shape = Shape(net, net)
        boxes = random_boxes(rng, V8, net, net, 3) + [[0, 0, net, net]]
        K = M = len(boxes)
        proto = make_proto(rng, shape, 2)
        dets = np.stack([make_dets(rng, shape, boxes) for _ in sizes])
        canv = _canvases(sizes, M)
        if ok:
            rows = _seg(shape, V8, torch.from_numpy(proto).cuda(), torch.from_numpy(dets).cuda(), sizes, K, M, canv)
            _check_seg(shape, V8, proto, dets, sizes, K, M, canv, rows)
            continue
        rows = torch.full((2, 1 + K * 6), ROW_SENTINEL, device="cuda")
        with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
            P.yolo_seg_postprocess(torch.from_numpy(proto).cuda(), torch.from_numpy(dets).cuda(), sizes, variant=V8,
                                   max_rows=K, max_masks=M, net_w=net, net_h=net, rows_out=rows, canvases_out=canv)
        torch.cuda.synchronize()
        assert torch.all(rows == ROW_SENTINEL) and all(torch.all(c == CANVAS_SENTINEL) for c in canv)
