"""CPU oracle of the Python runners' pre- and post-process (the *_trt.py scripts), and a loader that runs the reference
runners' own methods where the reference tree is present.

letterbox_rect / preprocess / postprocess are our numpy statement of what the runners compute, with the two rules the library adds where the runners leave
the result open: equal confidences are ordered by ascending row, and a front row of the greedy NMS is consumed after it is
kept (the runner's `while` never ends where that row does not suppress itself).  reference_runner() parses a runner file and
executes only its module constants and the five methods preprocess_image, xywh2xyxy, bbox_iou, non_max_suppression and
post_process, bound to a stand-in object holding input_w / input_h; tensorrt and pycuda are never imported and nothing of
the file is kept in this repository.  pre_frames() and post_cases() build the seeded inputs that the CPU and GPU tests share, so that the GPU
tests compare the device with the reference's digests in tests/golden/ref_pyrunner_host.npz.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ast
import os
import types
from pathlib import Path

import numpy as np

# The reference tree, as oracle/Makefile finds it.
REF_TREE = Path(os.environ.get("TRTX_REFERENCE", "/root/reference"))

# runner key (tensorrtx_b200.plugins.PYRUNNER_PRESETS) -> its file in the reference tree
RUNNER_FILES = {
    "yolov8_det_trt": "yolov8/yolov8_det_trt.py",
    "yolov8_5u_det_trt": "yolov8/yolov8_5u_det_trt.py",
    "yolo11_det_trt": "yolo11/yolo11_det_trt.py",
    "yolov12_det_trt": "yolov12-tubro/yolov12_det_trt.py",
    "yolov9_trt": "yolov9/yolov9_trt.py",
    "yolov10_det_trt": "yolov10/yolov10_det_trt.py",
    "yolov13_det_trt": "yolov13/yolov13_det_trt.py",
    "yolov7_trt": "yolov7/yolov7_trt.py",
    "yolov5_det_trt": "yolov5/yolov5_det_trt.py",
    "yolov5_det_cuda_python": "yolov5/yolov5_det_cuda_python.py",
    "yolov3_trt": "yolov3/yolov3_trt.py",
}
METHODS = ("preprocess_image", "xywh2xyxy", "bbox_iou", "non_max_suppression", "post_process")


# ---- restatement ------------------------------------------------------------------------------------------------------

def letterbox_rect(w: int, h: int, net_w: int, net_h: int) -> tuple[int, int, int, int]:
    """(x, y, w, h) of the resized frame: the ratio of the tighter side in double, the other side truncated, centred."""
    sx, sy = net_w / w, net_h / h
    if sy > sx:
        rh = int(sx * h)
        return 0, (net_h - rh) // 2, net_w, rh
    rw = int(sy * w)
    return (net_w - rw) // 2, 0, rw, net_h


def preprocess(frame: np.ndarray, net_w: int, net_h: int) -> np.ndarray:
    """[3, net_h, net_w] float32 planes R, G, B: the frame resized by cv2's INTER_LINEAR into letterbox_rect on 128."""
    import cv2

    x, y, rw, rh = letterbox_rect(frame.shape[1], frame.shape[0], net_w, net_h)
    canvas = np.full((net_h, net_w, 3), 128, np.uint8)
    canvas[y:y + rh, x:x + rw] = cv2.resize(np.ascontiguousarray(frame), (rw, rh))
    return np.ascontiguousarray(canvas[:, :, ::-1].transpose(2, 0, 1)).astype(np.float32) / np.float32(255.0)


def _frame_boxes(xyxy_or_cxcywh: np.ndarray, cxcywh: bool, w: int, h: int, net_w: int, net_h: int) -> np.ndarray:
    """The rows' boxes as corners at the frame's size, clipped to it; float32 throughout, the pad and ratio rounded once."""
    v = xyxy_or_cxcywh.astype(np.float32)
    if cxcywh:
        half_w, half_h = v[:, 2] / np.float32(2), v[:, 3] / np.float32(2)
        v = np.stack([v[:, 0] - half_w, v[:, 1] - half_h, v[:, 0] + half_w, v[:, 1] + half_h], 1)
    else:
        v = v.copy()
    sx, sy = net_w / w, net_h / h
    if sy > sx:
        v[:, [1, 3]] -= np.float32((net_h - sx * h) / 2)
        v /= np.float32(sx)
    else:
        v[:, [0, 2]] -= np.float32((net_w - sy * w) / 2)
        v /= np.float32(sy)
    lim = np.array([w - 1, h - 1, w - 1, h - 1], np.float32)
    return np.clip(v, np.float32(0), lim)


def _overlap(front: np.ndarray, rest: np.ndarray) -> np.ndarray:
    """Pixel IoU of one box with many: +1 on every side length, 1e-16 in the denominator, NaN corners give NaN."""
    one = np.float32(1)
    iw = np.clip(np.minimum(front[2], rest[:, 2]) - np.maximum(front[0], rest[:, 0]) + one, 0, None)
    ih = np.clip(np.minimum(front[3], rest[:, 3]) - np.maximum(front[1], rest[:, 1]) + one, 0, None)
    inter = iw * ih
    a0 = (front[2] - front[0] + one) * (front[3] - front[1] + one)
    a1 = (rest[:, 2] - rest[:, 0] + one) * (rest[:, 3] - rest[:, 1] + one)
    return inter / (a0 + a1 - inter + np.float32(1e-16))


def postprocess(buf: np.ndarray, w: int, h: int, preset: tuple, net_w: int = 640, net_h: int = 640,
                conf_thresh: float = 0.5, nms_thresh: float = 0.4) -> np.ndarray:
    """One frame's plugin buffer [1 + max_rows * F] -> kept rows [K, 6] float32 (x1, y1, x2, y2, conf, row[5])."""
    box_format, F, label_col, conf_col = preset
    buf = np.asarray(buf, np.float32)
    table = buf[1:].reshape(-1, F)
    c = float(buf[0])
    n = 0 if not c >= 1 else (len(table) if c >= len(table) else int(c))  # the device's reading of the count
    table = table[:n]
    conf = table[:, 4] * table[:, conf_col] if conf_col >= 0 else table[:, 4].copy()
    pick = np.nonzero(conf >= np.float32(conf_thresh))[0]
    order = pick[np.lexsort((pick, -conf[pick]))]
    boxes = _frame_boxes(table[order, :4], box_format == 1, w, h, net_w, net_h)
    labels = table[order, label_col]
    out, alive = [], np.ones(len(order), bool)
    for k in range(len(order)):
        if not alive[k]:
            continue
        out.append(k)
        later = np.arange(k + 1, len(order))
        hit = (_overlap(boxes[k], boxes[later]) > np.float32(nms_thresh)) & (labels[later] == labels[k])
        alive[later[hit]] = False
    kept = np.array(out, np.int64)
    rows = np.concatenate([boxes[kept], conf[order[kept], None], table[order[kept], 5:6]], 1)
    return rows.astype(np.float32).reshape(-1, 6)


def canonical(frames_rows) -> np.ndarray:
    """One float32 vector of a call's result: per frame its count, then its rows."""
    return np.concatenate([np.concatenate([[len(r)], np.asarray(r, np.float32).reshape(-1)]) for r in frames_rows]).astype(
        np.float32)


def device_rows(rows: np.ndarray) -> list[np.ndarray]:
    """The device's [B, 1 + max_rows * 6] -> per frame its [K, 6] kept rows."""
    return [r[1:1 + 6 * int(r[0])].reshape(-1, 6) for r in rows]


# ---- the reference runners -----------------------------------------------------------------------------------------------

def reference_available() -> bool:
    return all((REF_TREE / f).exists() for f in RUNNER_FILES.values())


def reference_runner(key: str, input_w: int = 640, input_h: int = 640):
    """The runner's own five methods, bound to a stand-in with input_w / input_h, or None without the reference tree."""
    path = REF_TREE / RUNNER_FILES[key]
    if not path.exists():
        return None
    tree = ast.parse(path.read_text())
    ns: dict = {"np": np, "__name__": "reference_runner"}
    try:
        import cv2

        ns["cv2"] = cv2
    except ImportError:  # preprocess_image then raises NameError; the post-process needs numpy only
        pass
    consts = [n for n in tree.body if isinstance(n, ast.Assign) and all(isinstance(t, ast.Name) and t.id.isupper()
                                                                         for t in n.targets)
              and not any(isinstance(x, ast.Call) for x in ast.walk(n.value))]
    funcs = [f for c in tree.body if isinstance(c, ast.ClassDef) for f in c.body
             if isinstance(f, ast.FunctionDef) and f.name in METHODS]
    assert sorted(f.name for f in funcs) == sorted(METHODS), (key, [f.name for f in funcs])
    exec(compile(ast.Module(body=consts + funcs, type_ignores=[]), str(path), "exec"), ns)
    runner = types.SimpleNamespace(input_w=input_w, input_h=input_h)
    for name in METHODS:
        setattr(runner, name, types.MethodType(ns[name], runner))
    return runner


def reference_rows(runner, buf: np.ndarray, w: int, h: int) -> np.ndarray:
    """The runner's post_process of one frame's buffer as [K, 6] float32 rows (boxes, scores, class ids)."""
    boxes, scores, classid = runner.post_process(np.array(buf, np.float32), h, w)
    if len(boxes) == 0:
        return np.zeros((0, 6), np.float32)
    return np.concatenate([boxes, scores[:, None], classid[:, None]], 1).astype(np.float32)


# ---- seeded cases --------------------------------------------------------------------------------------------------------

# frame sizes of the post-process cases: landscape, portrait, square, tiny, the 592 x 333 frame, 4K
POST_SIZES = [(1920, 1080), (1280, 720), (592, 333), (333, 592), (640, 640), (480, 640), (97, 301), (3840, 2160)]
# frames of the pre-process cases: (w, h, extra pitch bytes)
PRE_FRAMES = [(592, 333, 7), (1920, 1080, 0), (1, 300, 3), (400, 1, 0), (640, 640, 0), (1280, 720, 5), (333, 592, 1),
              (97, 301, 2)]
PRE_NETS = [(640, 640), (640, 384)]


def frame(rng, w: int, h: int) -> np.ndarray:
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def pre_frames(net: tuple[int, int]) -> list[np.ndarray]:
    rng = np.random.default_rng(net[0] * 7 + net[1])
    return [frame(rng, w, h) for w, h, _ in PRE_FRAMES]


def plugin_rows(rng, preset: tuple, count: int, max_rows: int, net_w: int, net_h: int, labels: str) -> np.ndarray:
    """One frame's plugin buffer: `count` rows with distinct confidences around the threshold, clustered boxes (some past
    the net's edge), class ids in column 5; the label column equal across rows (labels="equal") or the class
    (labels="distinct"); a few NaN confidences below and above the threshold."""
    box_format, F, label_col, conf_col = preset
    buf = np.zeros(1 + max_rows * F, np.float32)
    t = buf[1:].reshape(max_rows, F)
    k = min(count, max_rows) if count > 0 else 0
    t[:, 6:] = rng.standard_normal((max_rows, F - 6)).astype(np.float32)
    centres = rng.uniform(-40, [net_w + 40, net_h + 40], (6, 2))
    c = centres[rng.integers(0, 6, k)] + rng.normal(0, 25, (k, 2))
    wh = rng.uniform(8, 260, (k, 2))
    if box_format == 1:
        t[:k, :4] = np.concatenate([c, wh], 1)
    else:
        t[:k, :4] = np.concatenate([c - wh / 2, c + wh / 2], 1)
    conf = rng.permutation(np.linspace(0.2, 0.99, max(k, 1)))[:k]
    if conf_col >= 0:  # conf = row[4] * row[conf_col], still distinct
        t[:k, conf_col] = rng.uniform(0.5, 1.0, k).astype(np.float32)
        t[:k, 4] = (conf / t[:k, conf_col]).astype(np.float32)
    else:
        t[:k, 4] = conf
    t[:k, 5] = rng.integers(0, 4, k)
    if label_col != 5:
        t[:, label_col] = t[:, 5] if labels == "distinct" else 0.0
    elif labels == "equal":
        t[:k, 5] = 1.0
    if k > 4:
        t[rng.choice(k, 2, replace=False), 4] = np.nan  # above and below the threshold alike: never kept
    buf[0] = count
    return buf


def post_cases(presets: dict, max_rows: int = 1000, batch: int = 32):
    """(key, runner, dets [batch, 1 + max_rows * F], sizes) per preset and label mode: counts from 0 to past max_rows."""
    out = []
    for ri, (runner, preset) in enumerate(sorted(presets.items())):
        for mode in ("distinct", "equal"):
            rng = np.random.default_rng(1000 + 10 * ri + (mode == "equal"))
            counts = [int(x) for x in rng.integers(1, 400, batch)]
            counts[0], counts[1], counts[2] = 0, max_rows + 500, 1
            sizes = [POST_SIZES[(i + ri) % len(POST_SIZES)] for i in range(batch)]
            dets = np.stack([plugin_rows(rng, preset, c, max_rows, 640, 640, mode) for c in counts])
            out.append((f"post-{runner}-{mode}", runner, dets, sizes))
    return out
