"""The band pre-processes on the device along the shared template's seams: each of the 13 entry / variant cases against its
existing CPU oracle, bit for bit, at its widest rectangles (per slot count for the bicubic ones), at net sides of every
residue mod 4, at tiny nets, at dst offsets of 0, 4, 8 and 12 B, at letterbox rectangles that start and end at every row of
a band, at the bicubic vector / tail split, at bands that stage 4 ... 8 rows, across 64-frame launches, and through the
shared-memory opt-in in a fresh process.  Each store's byte table is checked against the driver's value formula in
float64.  Every output sits between sentinels, and the frames are checked unchanged after every call."""
from __future__ import annotations

import subprocess
import sys
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import cls as CL
from oracle import cubic as CO
from oracle import detr as DO
from oracle import linear as LO
from oracle import pyrunner as PO
from oracle import rcnn_pre as RP
from oracle import refinedet as RD
from oracle import ufld as UO
from oracle import yolop as YO
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

from test_band_paths_cpu import (BYTE_FRAME, CASES, CUBIC, LETTERBOX, LINEAR, MIXED, SLOT_GROUP_SIDES, TINY_FRAMES,
                                 cubic_slot_frame, cubic_slots, edge_frames, fill_width_frame, many_frames, rect,
                                 residue_nets, rw_mod8_frames, scale_y, spp_canvas, tiny_nets, widest)

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
SENTINEL = np.float32(-9999.0)  # no case's value


# ---- the case table ---------------------------------------------------------------------------------------------------
def _run(case, frames, net_w, net_h, max_size, out):
    if case == "rcnn":
        P.rcnn_preprocess(frames, net_w, net_h, out=out)
    elif case in ("cls_v8", "cls_v5"):
        P.cls_preprocess(frames, L.YOLO_V8 if case == "cls_v8" else L.YOLO_V5, net_w, net_h, out=out)
    elif case == "yolop":
        P.yolop_preprocess(frames, out=out, net_w=net_w, net_h=net_h)
    elif case == "detr":
        P.detr_preprocess(frames, out=out, net_w=net_w, net_h=net_h)
    elif case == "ufld":
        P.ufld_preprocess(frames, out=out, net_w=net_w, net_h=net_h)
    elif case == "refinedet":
        P.refinedet_preprocess(frames, out=out, net=net_w)
    elif case in CUBIC:
        P.cubic_preprocess(frames, _VARIANT[case], out=out, net_w=net_w, net_h=net_h)
    elif case == "linear_py":
        P.PyRunnerPreprocessPlan(frames, out=out, net_w=net_w, net_h=net_h).enqueue()
    else:
        P.linear_preprocess(frames, _VARIANT[case], out=out, net_w=net_w, net_h=net_h, max_size=max_size)


_VARIANT = {"cubic_yolov3_tiny": L.CUBIC_YOLOV3_TINY, "cubic_anticov": L.CUBIC_ANTICOV, "linear_yolov3": L.LINEAR_YOLOV3,
            "linear_retina": L.LINEAR_RETINA, "linear_yolov3_spp": L.LINEAR_YOLOV3_SPP}


def _first(r):
    return None if r is None else r[0]


def _oracle(case, img, net_w, net_h, max_size):
    """The case's oracle output for one frame, or None where the reference throws."""
    if case == "rcnn":
        return _first(RP.rcnn_preprocess(img, net_w, net_h))
    if case in ("cls_v8", "cls_v5"):
        return _first(CL.cls_preprocess(img, 0 if case == "cls_v8" else 1, net_w, net_h))
    if case == "yolop":
        return _first(YO.preprocess(img, net_w, net_h))
    if case == "detr":
        return DO.preprocess(img, net_w, net_h)
    if case == "ufld":
        return UO.preprocess(img, net_w, net_h)
    if case == "refinedet":
        return RD.preprocess(img, net_w)
    if case in CUBIC:
        return _first(CO.preprocess(img, _VARIANT[case], net_w, net_h))
    if case == "linear_py":
        return PO.preprocess(img, net_w, net_h) if rect(case, img.shape[1], img.shape[0], net_w, net_h) else None
    return _first(LO.preprocess(img, _VARIANT[case], net_w, net_h, max_size))


def _shape(case, net_w, net_h):
    return (net_h, net_w, 3) if case == "rcnn" else (3, net_h, net_w)


def _frame(rng, w, h, dev, extra=0, data=None):
    """A u8 BGR frame [h, w, 3] on the device (random, or `data`), read through a pitch of 3 * w + extra + 1 bytes from an odd
    base."""
    buf = rng.integers(0, 256, (h, 3 * w + extra + 1), dtype=np.uint8)
    if data is not None:
        buf[:, 1:1 + 3 * w] = data.reshape(h, 3 * w)
    t = torch.from_numpy(buf).to(dev)
    return t[:, 1:].as_strided((h, w, 3), (3 * w + extra + 1, 3, 1))


def _host(t):
    return np.ascontiguousarray(t.cpu().numpy())


def check(case, frames, net_w, net_h, max_size=0, offset=1, expect=None):
    """One call over `frames` into a float32 output that starts `offset` floats past a 16-byte boundary, between sentinels:
    bit for bit the oracle's (or `expect`'s) frames, or, where the oracle refuses any frame, TRTX_ERR_UNSUPPORTED and nothing
    written.  The frames are unchanged either way.  Returns the output."""
    dev = frames[0].device
    before = [_host(f) for f in frames]
    exp = expect if expect is not None else [_oracle(case, f, net_w, net_h, max_size) for f in before]
    shape = _shape(case, net_w, net_h)
    per = int(np.prod(shape))
    n = len(frames) * per
    big = torch.full((offset + n + 7,), float(SENTINEL), dtype=torch.float32, device=dev)
    out = big[offset:offset + n].view(len(frames), *shape)
    if any(e is None for e in exp):
        with pytest.raises(L.TrtxError, match="UNSUPPORTED"):
            _run(case, frames, net_w, net_h, max_size, out)
        torch.cuda.synchronize()
        assert (big == float(SENTINEL)).all()
        got = None
    else:
        _run(case, frames, net_w, net_h, max_size, out)
        b = big.cpu().numpy()
        got = b[offset:offset + n].reshape(len(frames), *shape)
        for i, e in enumerate(exp):
            assert np.array_equal(got[i].view(np.uint32), np.asarray(e, np.float32).view(np.uint32)), (
                case, (net_w, net_h), tuple(frames[i].shape[:2]), i, int((got[i] != e).sum()))
        assert (b[:offset] == SENTINEL).all() and (b[offset + n:] == SENTINEL).all()
    for f, h in zip(frames, before):
        assert np.array_equal(_host(f), h)
    return got


def _frames(rng, dev, sizes):
    return [_frame(rng, w, h, dev, extra=i % 5) for i, (w, h) in enumerate(sizes)]


def _split(case, sizes, net_w, net_h, max_size):
    """(the sizes whose rectangle the call accepts, the sizes it refuses as unsupported); a yolov3-spp frame whose canvas is
    another net is in neither (the call is TRTX_ERR_INVALID)."""
    ok = [s for s in sizes if rect(case, *s, net_w, net_h, max_size)]
    if case == "linear_yolov3_spp":
        return ok, [s for s in sizes if spp_canvas(*s, max_size) is None]
    return ok, [s for s in sizes if s not in ok]


# ---- widest rectangles ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in CASES if c not in CUBIC])
def test_widest_rectangle_bit_exact(dev, case):
    """The widest rectangle the case's budget admits (4 840 px for R-CNN, 4 757 px for the planar stores), shrunk from a frame
    1.5x its size; RefineDet's square net is 4 757 x 4 757 from a small frame."""
    rng = np.random.default_rng(11)
    W = widest(case)
    if case == "refinedet":
        check(case, [_frame(rng, 333, 250, dev, 3)], W, W)
        return
    fw, fh, nw, nh, mx = fill_width_frame(case, W)
    assert rect(case, fw, fh, nw, nh, mx)[2] == W
    sizes = [(fw, fh)] + ([] if case == "linear_yolov3_spp" else [(fw // 3, fh)])  # and a narrow frame beside it
    check(case, [_frame(rng, w, h, dev, 5) for w, h in sizes], nw, nh, mx)


@pytest.mark.parametrize("case", CUBIC)
def test_widest_cubic_rectangle_at_every_slot_count(dev, case):
    """At each slot count 6 ... 16, two frames at floor(228 352 / (12 * slots)) px, one on each side of the ceil(3 * scale)
    step's range; then one call with a 1 189 px frame at 6 slots beside a narrow one at 16."""
    rng = np.random.default_rng(12)
    for slots in range(6, 17):
        W = widest(case, slots)
        specs = [cubic_slot_frame(slots, side, W) for side in (0, 1)]
        nw, nh = specs[0][2:]
        check(case, [_frame(rng, w, h, dev, side) for side, (w, h, _, _) in enumerate(specs)], nw, nh)
    W = widest(case, 16)
    w, h, nw, nh = cubic_slot_frame(6, 1, W)
    assert cubic_slots(scale_y(nh, 160)) == 16 and rect(case, 80, 160, nw, nh)[2] < W
    check(case, [_frame(rng, w, h, dev, 1), _frame(rng, 80, 160, dev, 2)], nw, nh)


# ---- shapes -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_net_residues_and_dst_offsets(dev, case):
    """net_w and net_h mod 4 at 0 ... 3, each at dst offsets of 0, 4, 8 and 12 B, over frames that are enlarged, shrunk, 1 x N,
    N x 1 and 1 x 1; a frame whose rectangle is empty is refused alone."""
    rng = np.random.default_rng(13)
    for net_w, net_h, mx in residue_nets(case):
        ok, refused = _split(case, MIXED, net_w, net_h, mx)
        assert ok, (case, net_w, net_h)
        frames = _frames(rng, dev, ok)
        for offset in range(4):
            check(case, frames, net_w, net_h, mx, offset)
        for s in refused:
            check(case, _frames(rng, dev, [s]), net_w, net_h, mx)


@pytest.mark.parametrize("case", CASES)
def test_tiny_nets(dev, case):
    """Nets of 1 x 1, 2 x 3, 3 x 1, 1 x 7 and 5 x 5 (square ones for RefineDet and yolov3-spp): a band's run is shorter than its
    store's head.  The frames with a rectangle go in one call; each frame with an empty one is refused and writes nothing."""
    rng = np.random.default_rng(14)
    for k, (net_w, net_h, mx) in enumerate(tiny_nets(case)):
        ok, refused = _split(case, TINY_FRAMES, net_w, net_h, mx)
        assert ok, (case, net_w, net_h)
        check(case, _frames(rng, dev, ok), net_w, net_h, mx, k % 4)
        for s in refused:
            check(case, _frames(rng, dev, [s]), net_w, net_h, mx)


@pytest.mark.parametrize("case", LETTERBOX)
def test_letterbox_edges_at_every_band_row(dev, case):
    """Rectangles whose first row y0 and end y0 + rh are at every row of a band (all 16 pairs mod 4), with whole bands of
    padding above and below; one call per net."""
    rng = np.random.default_rng(15)
    groups = {}
    for w, h, nw, nh, mx in edge_frames(case):
        groups.setdefault((nw, nh, mx), []).append((w, h))
    for (nw, nh, mx), sizes in groups.items():
        check(case, _frames(rng, dev, sizes), nw, nh, mx)


@pytest.mark.parametrize("case", CUBIC)
def test_cubic_vector_tail_split_at_every_rw_mod_8(dev, case):
    """rw mod 8 at every value.  Each frame's rows are constant and alternate between two bytes p, p + 1 per channel; a 2x
    shrink weighs its 4 taps -192, 1216, 1216, -192 / 2048, so every inner output byte is the tie p + 0.5: the float loop
    rounds it to even (p), the integer tail up (p + 1).  An error in where a row's vector part ends moves bytes between them.
    Random frames at the same shapes follow."""
    rng = np.random.default_rng(16)
    net_w, net_h, sizes = rw_mod8_frames()
    frames = []
    for w, h in sizes:
        rows = np.array([[100, 40, 200], [101, 41, 201]], np.uint8)[np.arange(h) % 2]
        frames.append(_frame(rng, w, h, dev, 3, np.repeat(rows[:, None, :], w, axis=1)))
    got = check(case, frames, net_w, net_h)
    for i, (w, h) in enumerate(sizes):
        x0, y0, rw, _, _ = rect(case, w, h, net_w, net_h)
        nvec = (3 * rw) & ~7
        for c, (p, ch) in enumerate(((200, 2), (40, 1), (100, 0))):  # plane c, its BGR byte and that byte's lower value
            want = [CO.input_value(_VARIANT[case], p + (3 * x + ch >= nvec)) for x in range(rw)]
            assert np.array_equal(got[i][c, y0 + 5, x0:x0 + rw], np.array(want, np.float32)), (i, c)
    check(case, _frames(rng, dev, sizes), net_w, net_h)


def linear_band_rows(rh, sh, y0, net_h):
    """The distinct source rows LinearBand stages for each band of a rectangle rh rows high at row y0 over sh source rows."""
    sc = scale_y(rh, sh)
    counts = set()
    for b0 in range(0, net_h, 4):
        rows = set()
        for k in range(max(y0 - b0, 0), min(y0 + rh - b0, min(4, net_h - b0))):
            s = int(np.floor(np.float32((b0 + k - y0 + 0.5) * sc - 0.5)))
            rows |= {min(max(s + j, 0), sh - 1) for j in (0, 1)}
        if rows:
            counts.add(len(rows))
    return counts


@pytest.mark.parametrize("case", LINEAR)
def test_linear_bands_stage_4_to_8_rows(dev, case):
    """Square frames of 20 ... 80 px in a 40 x 40 net (scales 0.5 ... 2) give bands that stage every count of source rows from
    4 to 8: LinearBand's groups of 4 slot rows end exactly at 4 and part-way at 5 ... 7."""
    rng = np.random.default_rng(17)
    mx = 40 if case == "linear_yolov3_spp" else 0
    seen = set()
    groups = {}
    for s in SLOT_GROUP_SIDES:
        nw, nh = (40, 40) if case != "linear_yolov3_spp" else tuple(P.yolov3spp_letterbox(s, s, mx)[0])
        r = rect(case, s, s, nw, nh, mx)
        seen |= linear_band_rows(r[3], r[4], r[1], nh)
        groups.setdefault((nw, nh), []).append((s, s))
    assert {4, 5, 6, 7, 8} <= seen, seen
    for (nw, nh), sizes in groups.items():
        check(case, _frames(rng, dev, sizes), nw, nh, mx)


@pytest.mark.parametrize("case", ["rcnn", "cls_v5", "cubic_anticov", "linear_retina", "linear_py"])
def test_130_frames_widest_in_the_second_launch(dev, case):
    """130 frames take three launches; the widest rectangle, and so the call's stride, is frame 100's, in the second."""
    rng = np.random.default_rng(18)
    sizes = many_frames()
    rects = [rect(case, w, h, 200, 36) for w, h in sizes]
    assert max(range(130), key=lambda i: rects[i][2]) == 100
    check(case, _frames(rng, dev, sizes), 200, 36)


# ---- byte tables ------------------------------------------------------------------------------------------------------
def _f32(x):
    return np.float32(x)


def _fma_f32(a, b, c):
    """fmaf(a, b, c): the exact a * b + c rounded once to float (ties to even)."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    f = np.float32(float(x))
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.array(v).view(np.uint32)) & 1))


MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def byte_value(case, c, u):
    """The engine input value of byte u in plane c, from the driver's literals in float64 (each float step rounded as the
    driver's float does)."""
    u = float(u)
    if case in ("rcnn",):
        return _f32(u)
    if case in ("cls_v8", "linear_yolov3_spp"):  # convertTo / blobFromImage: (float)u * (float)(1 / 255.0)
        return _f32(u * float(_f32(1 / 255.0)))
    if case == "cls_v5":
        return _f32((u / 255.0 - MEAN[c]) / STD[c])
    if case in ("yolop", "detr"):  # u * (1.f / 255.f), minus (float)mean in float, over std in double
        t = _f32(u * float(_f32(1.0) / _f32(255.0)))
        s = _f32(float(t) - float(_f32(MEAN[c])))
        return _f32(float(s) / STD[c])
    if case == "ufld":
        mean, sd = float(_f32(MEAN[c])), float(_f32(STD[c]))
        return _fma_f32(_f32(u * float(_f32(1. / 255.))), _f32(1.0 / sd), _f32(-mean / sd))
    if case == "refinedet":
        return _f32(u - (123.0, 117.0, 104.0)[c])
    if case == "linear_retina":
        return _f32(u - (104.0, 117.0, 123.0)[c])
    if case == "cubic_anticov":
        return _f32((u - 127.5) * 0.0078125)
    return _f32(u / 255.0)  # yolov3-tiny, yolov3 / yolov4, the Python runners


CANVAS = {"rcnn": 128, "cls_v5": 128, "yolop": 114, "cubic_yolov3_tiny": 128, "cubic_anticov": 128, "linear_yolov3": 128,
          "linear_retina": 128, "linear_yolov3_spp": 128, "linear_py": 128}
BGR_PLANES = ("yolop", "linear_retina")  # plane c takes BGR byte c; every other planar store takes byte 2 - c (R first)


@pytest.mark.parametrize("case", CASES)
def test_byte_table_against_the_driver_formula(dev, case):
    """A 16 x 16 frame whose every channel holds all 256 bytes (B = i, G = i + 85, R = i + 170), at identity scale so the resize
    passes bytes through, equals the driver's value formula of each byte in float64, in the case's plane order; a
    letterbox's canvas rows take the canvas byte's value."""
    rng = np.random.default_rng(19)
    fw, fh = BYTE_FRAME
    i = np.arange(fw * fh).reshape(fh, fw)
    data = np.stack([i, (i + 85) % 256, (i + 170) % 256], axis=-1).astype(np.uint8)
    mx = 0
    if case == "linear_yolov3_spp":
        mx = fw + 8
        nw, nh = P.yolov3spp_letterbox(fw, fh, mx)[0]
    elif case in LETTERBOX:
        nw, nh = fw, fh + 8
    else:
        nw, nh = fw, fh
    x0, y0, rw, rh, sh = rect(case, fw, fh, nw, nh, mx)
    assert (rw, rh, sh) == (fw, fh, fh) and (case not in LETTERBOX or y0 >= 4)
    table = np.array([[byte_value(case, c, u) for u in range(256)] for c in range(3)], np.float32)
    exp = np.empty(_shape(case, nw, nh), np.float32)
    canvas = np.full((nh, nw, 3), CANVAS.get(case, 0), np.int64)
    canvas[y0:y0 + rh, x0:x0 + rw] = data
    if case == "rcnn":
        exp[:] = canvas.astype(np.float32)
    else:
        for c in range(3):
            exp[c] = table[c][canvas[:, :, c if case in BGR_PLANES else 2 - c]]
    check(case, [_frame(rng, fw, fh, dev, 7, data)], nw, nh, mx, expect=[exp])
    if case != "rcnn":  # the oracle agrees, as a cross-check of the formula
        check(case, [_frame(rng, fw, fh, dev, 7, data)], nw, nh, mx)


# ---- shared-memory opt-in, in a fresh process -------------------------------------------------------------------------
def opt_in_child(dev="cuda"):
    """Calls whose dynamic shared memory crosses 48 KiB, each on a kernel instantiation that no earlier call of the process
    opted in: a 65-frame call whose second launch alone needs more than 48 KiB, and calls at exactly 49 152 B and one column
    past it, each against its oracle.  49 152 B needs the opt-in too: the limit without it is 48 KiB less the kernel's static
    shared memory.  Raises on a mismatch."""
    rng = np.random.default_rng(20)
    # LinearBand stages 8 rows of 3 * rw int16: 48 * rw bytes, 48 KiB at rw = 1024
    sizes = [(40 + i, 48) for i in range(64)] + [(2300, 40)]  # rectangles of <= 32 px, then one of 1100 px
    assert max(rect("linear_retina", w, h, 1100, 24)[2] for w, h in sizes[:64]) * 48 <= 48 * 1024
    assert rect("linear_retina", *sizes[64], 1100, 24)[2] * 48 > 48 * 1024
    check("linear_retina", _frames(rng, dev, sizes), 1100, 24)
    print("ok 65 frames")
    for W, smem in ((1024, 49152), (1025, 49200)):
        fw, fh, nw, nh, _ = fill_width_frame("linear_yolov3", W, net_h=16, frame_h=24)
        assert 48 * rect("linear_yolov3", fw, fh, nw, nh)[2] == smem
        check("linear_yolov3", _frames(rng, dev, [(fw, fh)]), nw, nh)
        print("ok linear", smem)
    for W, smem in ((256, 49152), (257, 49344)):  # 16 slots of 3 * rw int: 192 * rw bytes
        fw, fh, nw, nh = cubic_slot_frame(16, 0, W)
        assert 16 * 12 * rect("cubic_yolov3_tiny", fw, fh, nw, nh)[2] == smem
        check("cubic_yolov3_tiny", _frames(rng, dev, [(fw, fh)]), nw, nh)
        print("ok cubic", smem)


_CHILD = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_band_paths_gpu as T; T.opt_in_child()"


def test_opt_in_in_a_fresh_process(dev):
    """cudaFuncSetAttribute lasts as long as the process, so these calls run in a child process of their own, which ends
    with the test."""
    r = subprocess.run([sys.executable, "-c", _CHILD, str(ROOT)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.split("\n")[:5] == ["ok 65 frames", "ok linear 49152", "ok linear 49200", "ok cubic 49152",
                                        "ok cubic 49344"], r.stdout
