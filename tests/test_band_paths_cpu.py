"""The band pre-processes' shared template (band_preprocess_kernel<Resize, Store> and band_preprocess in preprocess.cu) along its
own seams, without a GPU:
  * a model of CubicBand's row geometry checks that CubicBand::slots(scale_y) bounds the source rows every band stages;
  * one budget table gives each of the 13 entry / variant cases its widest rectangle (per slot count for the bicubic ones),
    derived from the stores' shared-memory constants, and a call one pixel wider is refused before any launch;
  * the static shared memory cuobjdump reports for each instantiation, plus its store's dynamic budget, fits the opt-in.
The frame and net tables the GPU file (test_band_paths_gpu.py) runs live here, so the slot model covers every shape it uses.
The pointers of every call here are fake: every call is refused before a launch."""
from __future__ import annotations

import ctypes as C
import math
import os
import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

from tensorrtx_b200 import _lib as L

# ---- the cases and their rectangles -----------------------------------------------------------------------------------
CASES = ["rcnn", "cls_v8", "cls_v5", "yolop", "detr", "ufld", "refinedet", "cubic_yolov3_tiny", "cubic_anticov", "linear_yolov3",
         "linear_retina", "linear_yolov3_spp", "linear_py"]
CUBIC = ["cubic_yolov3_tiny", "cubic_anticov"]
LINEAR = [c for c in CASES if c not in CUBIC]            # the LinearBand instantiations' cases
STRETCH = ["detr", "ufld", "refinedet"]                  # the whole frame over the whole net
LETTERBOX = [c for c in CASES if c not in STRETCH + ["cls_v8"]]  # a rectangle on a canvas
ENTRY = {  # case: (entry, the arguments before the descriptors)
    "rcnn": ("trtx_rcnn_preprocess_enqueue", ()),
    "cls_v8": ("trtx_cls_preprocess_enqueue", (L.YOLO_V8,)),
    "cls_v5": ("trtx_cls_preprocess_enqueue", (L.YOLO_V5,)),
    "yolop": ("trtx_yolop_preprocess_enqueue", ()),
    "detr": ("trtx_detr_preprocess_enqueue", ()),
    "ufld": ("trtx_ufld_preprocess_enqueue", ()),
    "refinedet": ("trtx_refinedet_preprocess_enqueue", ()),
    "cubic_yolov3_tiny": ("trtx_cubic_preprocess_enqueue", (L.CUBIC_YOLOV3_TINY,)),
    "cubic_anticov": ("trtx_cubic_preprocess_enqueue", (L.CUBIC_ANTICOV,)),
    "linear_yolov3": ("trtx_linear_preprocess_enqueue", (L.LINEAR_YOLOV3,)),
    "linear_retina": ("trtx_linear_preprocess_enqueue", (L.LINEAR_RETINA,)),
    "linear_yolov3_spp": ("trtx_linear_preprocess_enqueue", (L.LINEAR_YOLOV3_SPP,)),
    "linear_py": ("trtx_linear_preprocess_enqueue", (L.LINEAR_PY,)),
}


def trailing(case, net_w, net_h, max_size=0):
    """The entry's arguments after the frame count."""
    if case == "refinedet":
        assert net_w == net_h
        return (net_w,)
    if case.startswith("linear"):
        return (net_w, net_h, max_size)
    return (net_w, net_h)


def spp_canvas(w, h, max_size):
    """yolov3-spp's canvas (w, h) of a w x h frame, or None where its rectangle is empty."""
    g = (C.c_int * 6)()
    return (g[0], g[1]) if L.load().trtx_yolov3spp_letterbox(w, h, max_size, g) == L.OK else None


def rect(case, w, h, net_w, net_h, max_size=0):
    """(x0, y0, rw, rh, sh): the rectangle the band driver resizes frame w x h into and the source height it reads (the centre
    crop's for cls V8), from the library's own host geometry; None where the call is refused (an empty rectangle, one off
    the canvas, or a yolov3-spp canvas that is not the net)."""
    lib = L.load()
    r = (C.c_int * 6)()
    if case in STRETCH:
        return 0, 0, net_w, net_h, h
    if case == "cls_v8":
        return 0, 0, net_w, net_h, min(w, h)
    if case == "rcnn":
        lib.trtx_rcnn_letterbox_pads(w, h, net_w, net_h, r)
        rw, rh = net_w - r[0] - r[1], net_h - r[2] - r[3]
        return (r[0], r[2], rw, rh, h) if rw > 0 and rh > 0 and r[0] >= 0 and r[2] >= 0 else None
    if case == "linear_yolov3_spp":
        if lib.trtx_yolov3spp_letterbox(w, h, max_size, r) or (r[0], r[1]) != (net_w, net_h):
            return None
        return r[2], r[3], r[4], r[5], h
    if case == "linear_py":
        lib.trtx_pyrunner_letterbox_rect(w, h, net_w, net_h, r)
        return (r[0], r[1], r[2], r[3], h) if r[2] > 0 and r[3] > 0 else None
    lib.trtx_calib_letterbox_rect(w, h, net_w, net_h, r)
    x0, y0, rw, rh = r[0], r[1], r[2], r[3]
    ok = rw > 0 and rh > 0 and x0 >= 0 and y0 >= 0 and x0 + rw <= net_w and y0 + rh <= net_h
    return (x0, y0, rw, rh, h) if ok else None


def scale_y(rh, sh):
    """BandImage::scale_y, as the host computes it."""
    return 1. / (rh / sh)


# ---- the budget table -------------------------------------------------------------------------------------------------
OPT_IN = 227 * 1024        # the most dynamic + static shared memory a block may opt in to on an H100 (232 448 B)
RESERVED = 1024            # the per-block system reservation cuobjdump counts in a kernel's static shared memory
BAND_ROWS = 4              # kBandRows
LINEAR_SLOTS = 2 * BAND_ROWS
BUDGET = {  # Store::kMaxDynamicSmem
    "rcnn": OPT_IN - 128,                    # RcnnHwcStore: LinearBand's 128 B of static arrays
    "planar": OPT_IN - 3 * 256 * 4 - 1024,   # PlanarStore: its 3 x 256 float table and the band's other static arrays
}
STAGED = {"linear": 2, "cubic": 4}  # bytes per staged element: int16 rows (LinearBand), int rows (CubicBand)


PREPROCESS_CU = Path(__file__).resolve().parents[1] / "tensorrtx_b200" / "csrc" / "preprocess.cu"


def source_constants():
    """The constants the library is compiled from, read from preprocess.cu: each store's kMaxDynamicSmem in bytes, and the
    k of CubicBand::slots = min(16, ceil(3 * scale) + k)."""
    src = PREPROCESS_CU.read_text()
    got = {}
    for store, expr in re.findall(r"struct (\w+) \{\n(?:\s*//[^\n]*\n)*\s*static constexpr size_t kMaxDynamicSmem = ([^;]+);", src):
        assert re.fullmatch(r"[\d\s*+()-]+", expr.replace("sizeof(float)", "4")), expr
        got[store] = eval(expr.replace("sizeof(float)", "4"))
    m = re.search(r"static int slots\(double scale\) \{ return \(int\)fmin\(\(double\)kCubicMaxSlots, "
                  r"ceil\(\(kBandRows - 1\) \* scale\) \+ (\d+)\); \}", src)
    assert m and set(got) == {"RcnnHwcStore", "PlanarStore"}, got
    got["slots_k"] = int(m.group(1))
    return got


def test_source_constants_are_the_budget_table():
    """The stores' budgets and CubicBand::slots in preprocess.cu are the ones the table above is derived from."""
    c = source_constants()
    assert (c["RcnnHwcStore"], c["PlanarStore"], c["slots_k"]) == (BUDGET["rcnn"], BUDGET["planar"], 5)


def cubic_slots(scale):
    """CubicBand::slots: min(16, ceil(3 * scale) + 5)."""
    return int(min(16.0, math.ceil((BAND_ROWS - 1) * scale) + 5))


def widest(case, slots=None):
    """The widest rectangle the case accepts: its store's budget over the bytes of one staged column, 3 elements per slot."""
    budget = BUDGET["rcnn" if case == "rcnn" else "planar"]
    if case in CUBIC:
        return budget // (slots * 3 * STAGED["cubic"])
    return budget // (LINEAR_SLOTS * 3 * STAGED["linear"])


def test_budget_table_matches_the_documented_limits():
    """The derived table is the one the store comments state: 4 840 px (R-CNN), 4 757 px (every planar bilinear store), and
    for the bicubic stores floor(228 352 / (12 * slots)) at 6 ... 16 slots."""
    assert widest("rcnn") == 4840
    assert all(widest(c) == 4757 for c in LINEAR if c != "rcnn")
    assert [widest(CUBIC[0], s) for s in range(6, 17)] == [3171, 2718, 2378, 2114, 1902, 1729, 1585, 1463, 1359, 1268, 1189]
    assert BUDGET["planar"] == 228352


def _descs(*sizes):
    d = (L.ImageDesc * len(sizes))()
    for i, (w, h) in enumerate(sizes):
        d[i].data_dev, d[i].width, d[i].height, d[i].pitch = 4096, w, h, 3 * w
    return d


def fill_width_frame(case, W, net_h=20, frame_h=30):
    """(frame w, frame h, net w, net h, max_size): a frame about 1.5x the net, whose rectangle is exactly W pixels wide."""
    if case in STRETCH or case == "cls_v8":
        return (3 * W) // 2, frame_h, W, net_h, 0
    for w in range((3 * W) // 2 - 2, (3 * W) // 2 + 40):
        if case == "linear_yolov3_spp":
            canvas = spp_canvas(w, frame_h, W)
            if canvas and canvas[0] == W and rect(case, w, frame_h, *canvas, W)[2] == W:
                return w, frame_h, canvas[0], canvas[1], W
        else:
            r = rect(case, w, frame_h, W, net_h)
            if r and r[2] == W:
                return w, frame_h, W, net_h, 0
    raise AssertionError((case, W))


def cubic_slot_sh(slots, side, rh=31):
    """A source height whose scale over rh rows gives `slots` slots: side 0 just above the scale where the count steps up
    to `slots`, side 1 at the top of that range (just below the next step, or 5x for 16 slots)."""
    k = slots - 5  # ceil(3 * scale) over (k - 1) / 3 < scale <= k / 3
    if side == 0:
        return (rh * (k - 1)) // 3 + 1
    return 5 * rh if slots == 16 else (rh * k) // 3


def cubic_slot_frame(slots, side, W, net_h=40, rh=31):
    """(frame w, frame h, net w, net h): a frame whose letterbox rectangle fills the W-pixel-wide net over rh of its net_h rows
    (whole padding bands above and below), at a scale with `slots` slots."""
    sh = cubic_slot_sh(slots, side, rh)
    for w in range((W * sh) // rh + 2, (W * sh) // rh - 40, -1):
        r = rect(CUBIC[0], w, sh, W, net_h)
        if r and r[2] == W and r[3] == rh:
            assert cubic_slots(scale_y(rh, sh)) == slots, (slots, side, sh)
            return w, sh, W, net_h
    raise AssertionError((slots, side, W))


@pytest.mark.parametrize("case", [c for c in CASES if c not in CUBIC])
def test_one_pixel_past_the_widest_rectangle_is_refused(case):
    """A rectangle one pixel wider than the table's is TRTX_ERR_UNSUPPORTED; so, for the planar stores, is a net that wide."""
    W = widest(case) + 1
    fw, fh, nw, nh, mx = fill_width_frame(case, W)
    assert rect(case, fw, fh, nw, nh, mx)[2] == W
    entry, lead = ENTRY[case]
    fn = getattr(L.load(), entry)
    if case == "refinedet":
        nh = nw
    assert fn(*lead, _descs((fw, fh)), 1, *trailing(case, nw, nh, mx), 4096, None) == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("case", CUBIC)
@pytest.mark.parametrize("slots", range(6, 17))
def test_one_pixel_past_the_widest_cubic_rectangle_is_refused(case, slots):
    """At each slot count, on both sides of the ceil(3 * scale) step that reaches it, a rectangle one pixel wider than
    floor(228 352 / (12 * slots)) is refused; a wide frame with few slots and a narrow one with many are budgeted together."""
    entry, lead = ENTRY[case]
    fn = getattr(L.load(), entry)
    W = widest(case, slots) + 1
    for side in (0, 1):
        fw, fh, nw, nh = cubic_slot_frame(slots, side, W)
        assert fn(*lead, _descs((fw, fh)), 1, nw, nh, 4096, None) == L.ERR_UNSUPPORTED, side
    if slots < 16:  # widest(slots) is past widest(16): a 16-slot frame beside it takes the launch over the budget
        fw, fh, nw, nh = cubic_slot_frame(slots, 1, widest(case, slots))
        tall = (40, 4 * nh)
        assert rect(case, *tall, nw, nh)[2] < nw and cubic_slots(scale_y(nh, tall[1])) == 16
        assert fn(*lead, _descs((fw, fh), tall), 2, nw, nh, 4096, None) == L.ERR_UNSUPPORTED


# ---- CubicBand's slot bound -------------------------------------------------------------------------------------------
def cubic_staged(rh, sh):
    """The most source rows CubicBand stages for any band of a rectangle rh rows high that resizes sh source rows, for each
    sh of the 1-D sequence `sh`: every window of min(4, rh) consecutive destination rows d (a band may start at any row of
    the rectangle) reads taps s - 1 .. s + 2 clamped into the image, s = floor((float)((d + 0.5) * scale - 0.5)) with the
    host's double scale.  s is non-decreasing in d, so the distinct rows of a window are the first row's 4 taps plus, for
    each next row, its taps above the previous row's last.  torch on the CPU, for its threads."""
    sh = torch.as_tensor(sh, dtype=torch.float64)[:, None]
    scale = 1. / (rh / sh)
    s = ((torch.arange(rh, dtype=torch.float64)[None, :] + 0.5) * scale - 0.5).float().floor_()  # exact small integers
    last = (sh - 1).float()
    lo = torch.minimum((s - 1).clamp_(min=0), last)
    hi = torch.minimum((s + 2).clamp_(min=0), last)
    del s
    first = hi - lo + 1
    new = (hi[:, 1:] - torch.maximum(lo[:, 1:], hi[:, :-1] + 1) + 1).clamp_(min=0)
    w = min(BAND_ROWS, rh)
    total = first[:, :rh - w + 1].clone()
    for j in range(1, w):
        total += new[:, j - 1:rh - w + j]
    return total.amax(dim=1).to(torch.int64)


def _margins(rh, sh):
    """(staged - slots, staged - ceil(3 * scale)) for each sh."""
    staged = cubic_staged(rh, sh)
    step = torch.ceil((BAND_ROWS - 1) * (1. / (rh / torch.as_tensor(sh, dtype=torch.float64)))).to(torch.int64)
    return staged - torch.clamp(step + _SLOTS_K, max=16), staged - step


_SLOTS_K = source_constants()["slots_k"]


def test_cubic_slot_bound_model_sees_the_known_cases():
    """The model's own check: 7 rows at rh = sh = 7 (ceil(3 * scale) + 4, which ceil(3 * scale) + 3 would miss), the one row
    of a 1-row image, and no band past 16 rows however far the rectangle shrinks."""
    assert int(cubic_staged(7, [7])[0]) == 7
    assert int(cubic_staged(1, [1])[0]) == 1
    assert int(cubic_staged(40, [1000])[0]) == 16
    assert int(cubic_staged(31, [155])[0]) == 16


def test_cubic_slots_bound_every_band_up_to_rh_1200_sh_5000(capsys):
    """For every rectangle height rh <= 1 200 and source height sh <= 5 000 with scale <= 11 / 3 (where slots() is below its
    cap of 16), no band stages more rows than slots(scale), as preprocess.cu states it.  Prints the tightest bound
    ceil(3 * scale) + m that holds."""
    tight = -99
    for rh in range(1, 1201):
        sh = torch.arange(1, min(5000, (11 * rh) // 3) + 1)
        over, m = _margins(rh, sh)
        assert int(over.max()) <= 0, (rh, int(sh[int(over.argmax())]))
        tight = max(tight, int(m.max()))
    with capsys.disabled():
        print(f"\n[cubic slots] every band stages at most ceil(3 * scale) + {tight} rows; slots() allows + 5")
    assert tight == 4


def gpu_cubic_shapes():
    """Every (rh, sh) a bicubic frame of the GPU file resizes."""
    shapes = {(31, cubic_slot_sh(s, side)) for s in range(6, 17) for side in (0, 1)}  # cubic_slot_frame's, at every width
    for net_w, net_h, frames in cubic_gpu_calls():
        for w, h in frames:
            r = rect(CUBIC[0], w, h, net_w, net_h)
            if r:
                shapes.add((r[3], r[4]))
    return shapes


def test_cubic_slots_bound_every_shape_of_the_gpu_file():
    """The same bound at every bicubic shape the GPU file runs, 16-slot ones past scale 11 / 3 included."""
    by_rh = {}
    for rh, sh in gpu_cubic_shapes():
        by_rh.setdefault(rh, []).append(sh)
    assert len(by_rh) > 20
    for rh, shs in by_rh.items():
        over, _ = _margins(rh, torch.tensor(sorted(shs)))
        assert int(over.max()) <= 0, (rh, shs)


# ---- static shared memory ---------------------------------------------------------------------------------------------
def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_static_plus_dynamic_shared_memory_fits_the_opt_in():
    """For each of the 11 band_preprocess_kernel instantiations, its static shared memory less the system's 1 024 B
    reservation plus its store's kMaxDynamicSmem (as preprocess.cu states it) is at most the 232 448 B a block may opt in
    to: the widest accepted rectangle can launch."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    budget = source_constants()
    out = subprocess.run([tool, "-res-usage", str(L.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*band_preprocess_kernel\S*):\s*\n\s*REG:\d+ STACK:\d+ SHARED:(\d+)", out)
    assert len(found) == 11, found
    stores = set()
    for name, shared in found:
        store = "RcnnHwcStore" if "RcnnHwcStore" in name else "PlanarStore"
        assert store in name, name
        stores.add(name.split("band_preprocess_kernel")[1])
        assert int(shared) - RESERVED + budget[store] <= OPT_IN, (name, int(shared))
    assert len(stores) == 11


# ---- the GPU file's frames and nets -----------------------------------------------------------------------------------
MIXED = [(64, 48), (31, 77), (100, 9), (1, 13), (13, 1), (7, 7), (120, 130), (1, 1)]  # up, down, 1 x N, N x 1, 1 x 1
RESIDUE_NETS = [(37, 41), (38, 42), (39, 43), (41, 38), (44, 39), (42, 37)]  # (net_w, net_h) mod 4 at 1, 2, 3 and 0
TINY_NETS = [(1, 1), (2, 3), (3, 1), (1, 7), (5, 5)]
TINY_FRAMES = [(1, 1), (1, 9), (9, 1), (2, 3), (6, 4), (13, 11), (40, 30)]
SLOT_GROUP_SIDES = [20, 30, 32, 40, 50, 60, 70, 80]  # square frames in a 40 x 40 net: scales 0.5 ... 2
BYTE_FRAME = (16, 16)


def residue_nets(case):
    """(net_w, net_h, max_size) with net_h and net_w mod 4 at 0 ... 3; square for RefineDet, and for yolov3-spp each
    max_size whose canvases are those nets."""
    if case in ("refinedet", "linear_yolov3_spp"):
        return [(n, n, n) for n in (37, 38, 39, 44)]
    return [(w, h, 0) for w, h in RESIDUE_NETS]


def tiny_nets(case):
    if case in ("refinedet", "linear_yolov3_spp"):
        return [(n, n, n) for n in (1, 2, 3, 5, 7)]
    return [(w, h, 0) for w, h in TINY_NETS]


def edge_frames(case):
    """[(frame w, frame h, net w, net h, max_size)]: for every pair (y0 mod 4, (y0 + rh) mod 4) a frame whose rectangle
    starts and ends there, most of them shrunk from a frame about twice its size, with whole padding bands above and below it
    where the pair allows.  A centred rectangle has y0 + (y0 + rh) = net_h or net_h - 1, so the pairs take two net heights,
    0 and 2 mod 4 (yolov3-spp's canvases below 32 are max_size square)."""
    nets = [(24, 24, 24), (26, 26, 26)] if case == "linear_yolov3_spp" else [(24, 60, 0), (24, 62, 0)]
    got = {}
    for nw, nh, mx in nets:
        for h in range(2, 4 * nh):
            for w in (2 * nw, 2 * nw - 3, nw):
                r = rect(case, w, h, nw, nh, mx)
                if r is None:
                    continue
                key = (r[1] % 4, (r[1] + r[3]) % 4)
                pad = r[1] >= 4 and nh - r[1] - r[3] >= 4
                if key not in got or (pad and not got[key][1]):
                    got[key] = ((w, h, nw, nh, mx), pad)
    assert len(got) == 16, (case, sorted(got))
    assert sum(p for _, p in got.values()) >= 8, case
    return [f for f, _ in got.values()]


def rw_mod8_frames(net_w=61, net_h=23):
    """Frames (w, 2 * net_h): each letterbox rectangle is net_h rows of a 2x vertical shrink (bicubic weights -192, 1216,
    1216, -192 at fraction 0.5) and rw = w // 2 pixels, rw mod 8 at every value."""
    frames = [(2 * rw, 2 * net_h) for rw in range(net_w - 8, net_w)]
    assert sorted(rect(CUBIC[0], w, h, net_w, net_h)[2] % 8 for w, h in frames) == list(range(8))
    return net_w, net_h, frames


def many_frames(n=130, net_w=200, net_h=36, wide_at=100):
    """n frames: narrow rectangles (tall frames) but for frame wide_at, whose rectangle fills the net."""
    return [(2 * net_w + 10, net_h) if i == wide_at else (20 + (i * 7) % 90, 3 * net_h + i % 5) for i in range(n)]


def cubic_gpu_calls():
    """(net_w, net_h, frames) of every bicubic call in the GPU file but the widest-rectangle ones."""
    calls = [(w, h, MIXED) for w, h, _ in residue_nets(CUBIC[0])]
    calls += [(w, h, TINY_FRAMES) for w, h, _ in tiny_nets(CUBIC[0])]
    calls += [(nw, nh, [(w, h)]) for w, h, nw, nh, _ in edge_frames(CUBIC[0])]
    calls.append(rw_mod8_frames())
    calls.append((200, 36, many_frames()))
    calls.append((BYTE_FRAME[0], BYTE_FRAME[1] + 8, [BYTE_FRAME]))
    calls.append((1189, 40, [(80, 160)]))  # the 16-slot frame of the mixed widest call
    return calls
