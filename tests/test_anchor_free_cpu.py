"""yolov9, yolov10 and yolov13 on the CPU: their host post-processes, their YoloLayer_TRT creators, and yolov13's device
post-process defect.

* The oracle (oracle/anchor_free.py) equals each driver's own compiled code bit for bit (oracle/_ref/libref_af_<driver>_host.so;
  where it was not built, the digests in tests/golden/ref_af_host.npz): yolov9's nms() and get_rect, yolov10's get_topk and
  get_rect, and yolov13's nms() equals the library's yolov8 NMS semantics (oracle_nms variant 0).  The rows are seeded
  clusters plus crafted ones: pairs whose IoU falls on the other side of 0.45f only after yolov9's corner -> centre
  conversion, confidences at and beside 0.1f / 0.5f, equal confidences whose box[0] order is not their row order, NaN
  confidences (yolov10, yolov13), more rows than kMaxNumOutputBbox, and frames of mixed sizes.
* tests/trt_adapter_anchor_free_check.cpp: registry -> createPlugin -> serialize -> deserializePlugin for both creators and
  adapters, refused fields and blobs; its blobs equal the Python mirrors' and those the drivers' compiled plugins write.
* yolov13's postprocess.cu strides its 7-float rows by bbox_element = 4 (include/types.h:11-16): a restatement of its
  decode_kernel shows every row's conf, class and keep landing on the next row's box."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import anchor_free as A
from oracle.golden import RefOutputs
from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

ROOT = Path(__file__).resolve().parents[1]
G = RefOutputs("ref_af_host")
F = np.float32
SIZES = ((1280, 720), (640, 640), (480, 853), (333, 1000), (1920, 1080))


def _buf(rows, det_floats, count=None, cap=None):
    rows = np.asarray(rows, np.float32).reshape(-1, det_floats)
    cap = max(len(rows), 1) if cap is None else cap
    b = np.zeros(1 + cap * det_floats, np.float32)
    b[0] = len(rows) if count is None else count
    b[1:1 + rows.size] = rows.reshape(-1)
    return b


def _f32_iou_ltrb(a, b):
    l, r = max(a[0], b[0]), min(a[2], b[2])
    t, bo = max(a[1], b[1]), min(a[3], b[3])
    if t > bo or l > r:
        return F(0)
    inter = F(F(r - l) * F(bo - t))
    return F(inter / F(F(F(F(a[2] - a[0]) * F(a[3] - a[1])) + F(F(b[2] - b[0]) * F(b[3] - b[1]))) - inter))


def _f32_v9(a):
    return [F(F(a[0] + a[2]) / F(2)), F(F(a[1] + a[3]) / F(2)), F(a[2] - a[0]), F(a[3] - a[1])]


def _f32_iou_cxcywh(a, b):
    h = lambda v: F(v / F(2))  # noqa: E731
    l, r = max(F(a[0] - h(a[2])), F(b[0] - h(b[2]))), min(F(a[0] + h(a[2])), F(b[0] + h(b[2])))
    t, bo = max(F(a[1] - h(a[3])), F(b[1] - h(b[3]))), min(F(a[1] + h(a[3])), F(b[1] + h(b[3])))
    if t > bo or l > r:
        return F(0)
    inter = F(F(r - l) * F(bo - t))
    return F(inter / F(F(F(a[2] * a[3]) + F(b[2] * b[3])) - inter))


def straddling_pairs(k=6, seed=901):
    """k pairs of l, t, r, b boxes whose `iou > 0.45f` verdict on the corners differs from the verdict on yolov9's converted
    boxes (float32 arithmetic of both nms() functions)."""
    rng = np.random.default_rng(seed)
    thr, out = F(0.45), []
    for _ in range(2000):
        l, t = F(rng.uniform(100, 4000)), F(rng.uniform(100, 4000))
        w, h = F(rng.uniform(1, 60)), F(rng.uniform(1, 60))
        a = [l, t, F(l + w), F(t + h)]
        s0 = F(w * F(0.55 / 1.45))  # a copy shifted by s0 along x has IoU (w - s0) / (w + s0) = 0.45
        for j in range(-30, 31):
            s = F(s0 + F(j) * np.spacing(s0) * F(64))
            b = [F(l + s), t, F(a[2] + s), a[3]]
            if (_f32_iou_ltrb(a, b) > thr) != (_f32_iou_cxcywh(_f32_v9(a), _f32_v9(b)) > thr):
                out.append((a, b))
                break
        if len(out) == k:
            return out
    raise AssertionError("no straddling pairs found")


def v9_rows(seed, n_clusters=60, seg=True):
    """38-float yolov9 rows: seeded clusters over 6 classes, straddling pairs, confidences at and beside 0.1f, equal
    confidences in a small class whose box[0] order is the reverse of their row order."""
    rng = np.random.default_rng(seed)
    rows = []

    def row(box, conf, cls):
        r = np.zeros(38, np.float32)
        r[:4], r[4], r[5] = box, conf, cls
        if seg:
            r[6:] = rng.normal(0, 1, 32)
        rows.append(r)
    for _ in range(n_clusters):
        cx, cy, w, h = rng.uniform(50, 600, 2).tolist() + rng.uniform(10, 150, 2).tolist()
        c = float(rng.integers(0, 6))
        for _ in range(int(rng.integers(1, 6))):
            x, y = cx + rng.normal(0, 6), cy + rng.normal(0, 6)
            ww, hh = w * rng.uniform(0.8, 1.2), h * rng.uniform(0.8, 1.2)
            row([x - ww / 2, y - hh / 2, x + ww / 2, y + hh / 2], rng.uniform(0.1, 1.0), c)
    for i, (a, b) in enumerate(straddling_pairs()):
        row(a, 0.9, 7.0 + i)
        row(b, 0.8, 7.0 + i)
    for i, c in enumerate((F(0.1), np.nextafter(F(0.1), F(0)), np.nextafter(F(0.1), F(1)))):
        row([5000 + 100 * i, 10, 5050 + 100 * i, 60], c, 20.0)
    for i in range(4):  # tied confidences: row order != box[0] order, disjoint boxes
        row([9000 - 200 * i, 10, 9050 - 200 * i, 60], 0.75, 30.0)
    rows = np.asarray(rows, np.float32)
    tail = rows[-4:]
    rows = rows[:-4][rng.permutation(len(rows) - 4)]
    return np.concatenate([rows, tail])


def _rows_of(lib, buf, det_floats, conf, nms, cap):
    out = np.zeros((cap, det_floats), np.float32)
    n = lib.ref_af_rows(buf.ctypes.data_as(C.c_void_p), C.c_float(conf), C.c_float(nms), out.ctypes.data_as(C.c_void_p), cap)
    return out[:n]


def test_v9_oracle_equals_driver_nms():
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    lib = G.lib("libref_af_yolov9_host.so")
    if lib is not None:
        c = (C.c_int * 4)()
        lib.ref_af_consts(c)
        assert tuple(c) == (640, 640, d["max_out"], d["det_floats"])
        t = (C.c_float * 2)()
        lib.ref_af_thresh(t)
        assert (t[0], t[1]) == (F(d["conf_thresh"]), F(d["nms_thresh"]))
    for seed in (910, 911, 912):
        buf = _buf(v9_rows(seed, seg=seed != 912), 38)
        got, _ = A.v9_nms(buf, d["max_out"], 38, d["conf_thresh"], d["nms_thresh"])
        ref = None if lib is None else _rows_of(lib, buf, 38, d["conf_thresh"], d["nms_thresh"], 4000)
        G.equal(f"v9.nms.{seed}", got, ref)
        # what each crafted row claims: 0.1f itself is dropped, the float above kept; the tied rows keep their row order
        assert F(0.1) not in got[:, 4] and np.nextafter(F(0.1), F(1)) in got[:, 4]
        tied = got[got[:, 5] == 30.0]
        assert len(tied) == 4 and (np.diff(tied[:, 0]) < 0).all()
        # the straddling pairs: the oracle's kept count differs from an LTRB NMS of the same pairs
        from oracle import oracle as O
        pairs = np.concatenate([r for r in buf[1:].reshape(-1, 38) if 7.0 <= r[5] < 20.0]).reshape(-1, 38)
        ltrb, _ = O.nms(0, _buf(pairs, 38), len(pairs), 38, d["conf_thresh"], d["nms_thresh"])
        v9, _ = A.v9_nms(_buf(pairs, 38), len(pairs), 38, d["conf_thresh"], d["nms_thresh"])
        assert len(ltrb) != len(v9)


def test_v9_reads_at_most_max_out_rows():
    d = P.ANCHOR_FREE_DRIVERS["yolov9"]
    rng = np.random.default_rng(913)
    n = d["max_out"] + 150
    rows = np.zeros((n, 38), np.float32)
    xy = rng.uniform(0, 3000, (n, 2)).astype(np.float32)
    rows[:, :2], rows[:, 2:4] = xy, xy + rng.uniform(5, 40, (n, 2)).astype(np.float32)
    rows[:, 4], rows[:, 5] = rng.uniform(0.05, 1, n), rng.integers(0, 3, n)
    buf = _buf(rows, 38)
    got, src = A.v9_nms(buf, d["max_out"], 38, d["conf_thresh"], d["nms_thresh"])
    assert src.max() < d["max_out"] and len(got) > 100
    lib = G.lib("libref_af_yolov9_host.so")
    G.equal("v9.nms.over_max_out", got, None if lib is None else _rows_of(lib, buf, 38, d["conf_thresh"], d["nms_thresh"], n))


def _boxes_for_rect(rng, n, center_size):
    """Boxes in network pixels, a fifth of them reaching past the letterboxed area (clamped by yolov8's get_rect)."""
    x, y = rng.uniform(-60, 700, n), rng.uniform(-60, 700, n)
    w, h = rng.uniform(1, 300, n), rng.uniform(1, 300, n)
    return np.stack([x, y, w, h] if center_size else [x, y, x + w, y + h], 1).astype(np.float32)


@pytest.mark.parametrize("driver", ["yolov9", "yolov10"])
def test_get_rect_equals_driver(oracle, driver):
    d = P.ANCHOR_FREE_DRIVERS[driver]
    lib = G.lib(f"libref_af_{driver}_host.so")
    rng = np.random.default_rng(920)
    variant = d["rect"]
    for w, h in SIZES:
        boxes = _boxes_for_rect(rng, 200, variant == L.YOLO_V5)
        got = np.stack([oracle.get_rect(variant, w, h, b) for b in boxes])
        ref = None
        if lib is not None:
            ref = np.zeros((len(boxes), 4), np.int32)
            for i, b in enumerate(boxes):
                bb = np.ascontiguousarray(b)
                lib.ref_af_get_rect(w, h, bb.ctypes.data_as(C.c_void_p), ref[i].ctypes.data_as(C.c_void_p))
        G.equal(f"{driver}.rect.{w}x{h}", got, ref)
        if variant == L.YOLO_V8:
            assert (got >= 0).all() and ((got[:, 0] + got[:, 2] <= w) | (got[:, 2] == 0)).all()   # clamped to the frame
        else:
            assert (got[:, :2] < 0).any()                                           # yolov5's: not clamped


def v10_rows(seed, n=300):
    rng = np.random.default_rng(seed)
    rows = np.zeros((n, 6), np.float32)
    rows[:, :4] = _boxes_for_rect(rng, n, False)
    rows[:, 4] = rng.uniform(0.1, 1.0, n)
    rows[:, 5] = rng.integers(0, 80, n)
    rows[3:6, 4] = (F(0.5), np.nextafter(F(0.5), F(0)), np.nextafter(F(0.5), F(1)))
    rows[10, 4] = np.nan
    return rows


def test_v10_oracle_topk_equals_driver():
    d = P.ANCHOR_FREE_DRIVERS["yolov10"]
    lib = G.lib("libref_af_yolov10_host.so")
    for seed in (930, 931):
        rows = v10_rows(seed)
        buf = _buf(rows, 6)
        for w, h in SIZES:
            got = A.topk(buf, len(rows), 6, d["conf_thresh"], w, h, variant=d["rect"])
            assert np.isnan(got[:, 4]).sum() == 1 and F(0.5) not in got[:, 4] and np.nextafter(F(0.5), F(1)) in got[:, 4]
            ref = None
            if lib is not None:
                sel = _rows_of(lib, buf, 6, d["conf_thresh"], 0.0, len(rows))
                ref = np.zeros((len(sel), 6), np.float32)
                for i, r in enumerate(sel):
                    rr = np.zeros(4, np.int32)
                    bb = np.ascontiguousarray(r[:4])
                    lib.ref_af_get_rect(w, h, bb.ctypes.data_as(C.c_void_p), rr.ctypes.data_as(C.c_void_p))
                    ref[i, :4], ref[i, 4:] = rr, r[4:6]
            G.equal(f"v10.topk.{seed}.{w}x{h}", got, ref, nan_ok=True)


def test_v10_topk_takes_the_first_max_rows():
    """A count past max_rows: the first max_rows rows, what get_topk reads when the count is the plugin's capacity."""
    d = P.ANCHOR_FREE_DRIVERS["yolov10"]
    rows = v10_rows(932, n=d["max_out"] + 100)
    got = A.topk(_buf(rows, 6), d["max_out"], 6, d["conf_thresh"], 1280, 720)
    clamped = A.topk(_buf(rows[:d["max_out"]], 6), d["max_out"], 6, d["conf_thresh"], 1280, 720)
    assert np.array_equal(got, clamped, equal_nan=True) and len(got) < len(A.topk(_buf(rows, 6), len(rows), 6, 0.5, 1280, 720))
    lib = G.lib("libref_af_yolov10_host.so")
    ref = None
    if lib is not None:
        ref = _rows_of(lib, _buf(rows, 6, count=d["max_out"], cap=len(rows)), 6, d["conf_thresh"], 0.0, len(rows))[:, 4:6]
    G.equal("v10.topk.first_max_rows", got[:, 4:6], ref, nan_ok=True)


def v13_rows(seed, n_clusters=60):
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_clusters):
        cx, cy, w, h = rng.uniform(50, 600, 2).tolist() + rng.uniform(10, 150, 2).tolist()
        c = float(rng.integers(0, 5))
        for _ in range(int(rng.integers(1, 6))):
            x, y = cx + rng.normal(0, 6), cy + rng.normal(0, 6)
            rows.append([x - w / 2, y - h / 2, x + w / 2, y + h / 2, rng.uniform(0.3, 1.0), c])
    for i in range(4):  # tied confidences: yolov8's cmp orders them by box[0]
        rows.append([9000 - 200 * i, 10, 9050 - 200 * i, 60, 0.75, 30.0])
    rows.append([100, 100, 200, 200, np.nan, 1.0])
    rows.append([100, 100, 200, 200, 0.5, 2.0])
    rows = np.asarray(rows, np.float32)
    return rows[rng.permutation(len(rows))]


def test_v13_nms_is_the_library_ltrb_nms(oracle):
    d = P.ANCHOR_FREE_DRIVERS["yolov13"]
    assert (d["box_format"], d["mode"], d["tie_break_x0"]) == (L.BOX_LTRB, L.NMS_GREEDY, True)
    lib = G.lib("libref_af_yolov13_host.so")
    for seed in (940, 941):
        buf = _buf(v13_rows(seed), 6)
        got, _ = oracle.nms(0, buf, int(buf[0]), 6, d["conf_thresh"], d["nms_thresh"])
        assert not np.isnan(got[:, 4]).any() and F(0.5) not in got[:, 4]
        tied = got[got[:, 5] == 30.0]
        assert len(tied) == 4 and (np.diff(tied[:, 0]) > 0).all()
        G.equal(f"v13.nms.{seed}", got, None if lib is None else _rows_of(lib, buf, 6, d["conf_thresh"], d["nms_thresh"], 1000))


def test_v13_device_post_process_overwrites_rows():
    """yolov13/src/postprocess.cu:16-49 with bbox_element = sizeof(AffineMatrix{float value[3]}) / 4 + 1 = 4: row k is written
    at 1 + 4k with 7 floats, so its conf, class and keep become row k + 1's l, t, r (in arrival order), and nms_kernel
    reads every row at that stride.  The library's one-shot NMS on 6-float rows is the semantics the code intends."""
    bbox_element = 3 * 4 // 4 + 1
    assert bbox_element == 4
    rows = np.array([[10, 20, 30, 40, 0.9, 3], [50, 60, 70, 80, 0.8, 5], [90, 100, 110, 120, 0.7, 7]], np.float32)
    parray = np.zeros(1 + 3 * 7, np.float32)
    for k, r in enumerate(rows):  # arrival order = row order
        parray[1 + k * bbox_element:1 + k * bbox_element + 7] = [*r[:4], r[4], r[5], 1.0]
    parray[0] = len(rows)
    read = [parray[1 + k * bbox_element:1 + k * bbox_element + 7] for k in range(len(rows))]
    for k in range(len(rows) - 1):
        assert list(read[k][:4]) == list(rows[k][:4])                 # its own box survives
        assert list(read[k][4:7]) == list(rows[k + 1][:3])            # conf, class, keep = the next row's l, t, r
    assert list(read[-1][4:7]) == [rows[-1][4], rows[-1][5], 1.0]     # only the last row is whole


# ------------------------------------------------------------------ TensorRT creators ----------------------------------
def _build_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda = Path(nvcc).resolve().parents[1]
    exe = tmp_path / "trt_adapter_anchor_free_check"
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-I", str(ROOT / "include"), "-I", str(ROOT / "tests" / "mock_trt"),
           "-I", str(cuda / "include"), str(ROOT / "tests" / "trt_adapter_anchor_free_check.cpp"), "-o", str(exe),
           str(L.LIB_PATH), f"-Wl,-rpath,{L.LIB_PATH.parent}", "-L", str(cuda / "lib64"), "-lcudart", f"-Wl,-rpath,{cuda / 'lib64'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_creators_blobs_and_refusals(tmp_path):
    r = subprocess.run([str(_build_check(tmp_path)), "--dump"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "anchor-free adapter check ok" in r.stdout
    blobs = {ln.split()[1]: bytes.fromhex(ln.split()[2]) for ln in r.stdout.splitlines() if ln.startswith("blob ")}
    assert set(blobs) == {"yolov9", "yolov9-seg", "yolov10"}
    mirrors = {"yolov9": P.YoloLayerPluginV9(80, 640, 640, 2000, False), "yolov9-seg": P.YoloLayerPluginV9(80, 640, 640, 2000, True),
               "yolov10": P.YoloLayerPluginV10(80, 640, 640, 1000, (8, 16, 32))}
    for name, m in mirrors.items():
        assert blobs[name] == m.serialize() and len(blobs[name]) == m.getSerializationSize()
        q = type(m).deserialize(blobs[name])
        assert q.serialize() == blobs[name] and q.output_elems() == m.output_elems()
    # the drivers' compiled plugins write the same bytes (yolov13's class is yolov10's)
    for driver, name, seg in (("yolov9", "yolov9", 0), ("yolov9", "yolov9-seg", 1), ("yolov10", "yolov10", 0),
                              ("yolov13", "yolov10", 0)):
        lib = G.lib(f"libref_af_{driver}.so")
        ref = None
        if lib is not None:
            buf = (C.c_ubyte * 64)()
            st = (C.c_int * 3)(8, 16, 32)
            n = lib.ref_af_serialize(80, 640, 640, 2000 if driver == "yolov9" else 1000, seg, st, 3, buf, 64)
            ref = np.frombuffer(bytes(buf[:n]), np.uint8)
        G.equal(f"blob.{driver}.{name}", np.frombuffer(blobs[name], np.uint8), ref)


def test_mirror_refuses_other_lengths():
    b = P.YoloLayerPluginV10(80, 640, 640, 1000, (8, 16, 32)).serialize()
    for blob in (b[:-4], b + b"\0\0\0\0", b[:20]):
        with pytest.raises(L.TrtxError):
            P.YoloLayerPluginV10.deserialize(blob)
    b9 = P.YoloLayerPluginV9(80, 640, 640, 2000, True).serialize()
    for blob in (b9[:-1], b9 + b"\0", b9[:20] + b"\x02"):
        with pytest.raises(L.TrtxError):
            P.YoloLayerPluginV9.deserialize(blob)


def test_abi_and_box_constant():
    lib = L.load()
    assert lib.trtx_abi_sizeof(15) == C.sizeof(L.YoloTopkParams) == 20
    assert L.BOX_V9 == 4
