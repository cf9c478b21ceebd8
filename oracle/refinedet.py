"""ctypes/numpy wrapper around oracle/librefinedet_oracle.so, the CPU oracle of the RefineDet pre- and post-process
(base_transform, PriorBox, the two decode steps, the ARM filter, nms() and the driver's rectangles), and a line-by-line
transcription of the reference's libtorch post-process (refinedet/refinedet.cpp:600-791) in torch float64.

The transcription runs on any torch device.  On CUDA it runs the reference's own ATen kernels and CUDA's double exp, so it
is the reference's arithmetic; on the CPU its exp is torch's CPU exp.  Its order among tied scores is torch.sort's, which
the reference leaves open: compare it on tie-free heads.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: imported by tests/ and tools/, never by the product package.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import torch

from . import oracle as _base


HERE = Path(__file__).resolve().parent
LIB = HERE / "librefinedet_oracle.so"
NET = 320
NUM_CLASSES = 25
TOP_K = 1000
INT_MAX, INT_MIN = 2147483647, -2147483648
F32 = lambda v: float(np.float32(v))  # noqa: E731  a C++ float literal as the double a Scalar holds
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    _lib = _base.build_and_open(LIB)
    _lib.oracle_refinedet_input_value.restype = C.c_float
    _lib.oracle_refinedet_postprocess.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                                                     C.c_int, C.c_int, C.c_void_p]
    _lib.oracle_refinedet_rows.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]
    return _lib


def _vp(a):
    return C.c_void_p(a.ctypes.data)


def num_priors(net: int = NET) -> int:
    return 3 * sum((net >> s) ** 2 for s in (3, 4, 5, 6))


def input_value(c: int, u: int) -> np.float32:
    """The engine input value of byte u in plane c (0 = R, 1 = G, 2 = B)."""
    return np.float32(load().oracle_refinedet_input_value(int(c), int(u)))


def preprocess(img, net: int = NET) -> np.ndarray:
    """base_transform for one u8 HWC BGR image [h, w, 3] (rows may be pitched) -> [3, net, net] float32 planes."""
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and a.strides[2] == 1 and a.strides[1] == 3
    out = np.empty((3, net, net), np.float32)
    load().oracle_refinedet_preprocess(C.c_void_p(a.ctypes.data), int(a.shape[1]), int(a.shape[0]), C.c_size_t(a.strides[0]),
                                       int(net), _vp(out))
    return out


def priors(net: int = NET, double_sqrt: bool = False) -> np.ndarray:
    """PriorBox at a square net -> [P, 4] float64 (cx, cy, w, h), clamped to [0, 1]; sqrt(ar) the float (default) or double
    overload."""
    out = np.empty((num_priors(net), 4), np.float64)
    assert load().oracle_refinedet_priors(int(net), int(double_sqrt), _vp(out)) == out.shape[0]
    return out


def postprocess(arm_loc, arm_conf, odm_loc, odm_conf, net: int = NET, obj_thresh=0.01, conf_thresh=0.01, nms_thresh=0.45,
                top_k: int = TOP_K, max_det: int | None = None) -> np.ndarray:
    """doInference's post-process for one frame (heads [P, 4], [P, 2], [P, 4], [P, C] float32) with the library's tie rule
    -> dets [1 + max_det * 6]: the count, the rows (x1, y1, x2, y2, score, label), zeros."""
    heads = [np.ascontiguousarray(h, np.float32) for h in (arm_loc, arm_conf, odm_loc, odm_conf)]
    Cn = heads[3].shape[1]
    max_det = (Cn - 1) * top_k if max_det is None else max_det
    out = np.empty(1 + max_det * 6, np.float32)
    load().oracle_refinedet_postprocess(*[_vp(h) for h in heads], int(net), Cn, obj_thresh, conf_thresh, nms_thresh,
                                        int(top_k), int(max_det), _vp(out))
    return out


def rows(dets, cols: int, rows_: int, score_thresh: float = 0.2) -> np.ndarray:
    """The driver loop (:957-993) over dets [1 + max_det * 6] of a cols x rows frame -> [1 + max_det * 6]: the count, then
    (x, y, w, h, score, label) after `score < TH` and RoiCorrect, zeros."""
    d = np.ascontiguousarray(dets, np.float32)
    out = np.empty_like(d)
    load().oracle_refinedet_rows(_vp(d), (d.shape[0] - 1) // 6, int(cols), int(rows_), score_thresh, _vp(out))
    return out


# ------------------------------------------------------------------ the reference in torch ------------------------------
def prior_box(net: int = NET, device="cpu") -> torch.Tensor:
    """PriorBox (:553-597): the float vector, from_blob, .cuda(), clamp(0, 1), toType(kFloat64)."""
    mean = []
    for k, (step, min_size) in enumerate(zip((8, 16, 32, 64), (32, 64, 128, 256))):
        f = net // step
        for i in range(f):
            for j in range(f):
                f_k = F32(net * 1.0 / step)
                cx, cy, s_k = F32((j + 0.5) / f_k), F32((i + 0.5) / f_k), F32(min_size * 1.0 / net)
                sq = F32(np.sqrt(np.float32(2)))
                mean += [cx, cy, s_k, s_k, cx, cy, F32(s_k * 1.0 * sq), F32(s_k * 1.0 / sq), cx, cy, F32(s_k * 1.0 / sq),
                         F32(s_k * 1.0 * sq)]
    m = torch.tensor(mean, dtype=torch.float32).view(-1, 4).to(device)
    return m.clamp(0, 1).to(torch.float64)


def decode(_loc, _prior, b_form_pt=False):
    variance = [F32(0.1), F32(0.2)]
    top_2 = torch.tensor([0, 1], device=_loc.device)
    bottom_2 = torch.tensor([2, 3], device=_loc.device)
    c1 = _prior.index_select(1, top_2) + _loc.index_select(1, top_2).mul(variance[0]) * _prior.index_select(1, bottom_2)
    c2 = _prior.index_select(1, bottom_2) * torch.exp(_loc.index_select(1, bottom_2) * variance[1])
    _retv = torch.cat([c1, c2], 1)
    if b_form_pt:
        c3 = _retv.index_select(1, top_2) - _retv.index_select(1, bottom_2).div(2)
        c4 = c3 + _retv.index_select(1, bottom_2)
        return torch.cat([c3, c4], 1)
    return _retv


def nms(boxes, scores, overlap, top_k):
    count = 0
    keep = torch.zeros(scores.size(0), dtype=torch.long, device=scores.device)
    if boxes.numel() == 0:
        return keep, count
    x1, y1, x2, y2 = (boxes.select(1, k).clone() for k in range(4))
    area = (x2 - x1) * (y2 - y1)
    v, idx = torch.sort(scores.unsqueeze(1), 0, False)
    idx = idx.squeeze(1)
    num_ = idx.size(0)
    if num_ > top_k:
        idx = idx[num_ - top_k:num_].clone()
    while idx.numel() > 0:
        i = idx[-1]
        keep[count] = i
        count += 1
        if idx.size(0) == 1:
            break
        idx = idx[:idx.size(0) - 1].clone()
        xx1, yy1, xx2, yy2 = (t.index_select(0, idx) for t in (x1, y1, x2, y2))
        # x1[i].item().toFloat(): the double rounded to float, widened again as a Scalar
        xx1 = xx1.clamp(float(x1[i].to(torch.float32).item()), INT_MAX * 1.0)
        yy1 = yy1.clamp(float(y1[i].to(torch.float32).item()), INT_MAX * 1.0)
        xx2 = xx2.clamp(INT_MIN * 1.0, float(x2[i].to(torch.float32).item()))
        yy2 = yy2.clamp(INT_MIN * 1.0, float(y2[i].to(torch.float32).item()))
        w = (xx2 - xx1).clamp(0, INT_MAX)
        h = (yy2 - yy1).clamp(0, INT_MAX)
        inter = w * h
        rem_areas = area.index_select(0, idx)
        union_ = (rem_areas - inter) + area[i]
        iou = inter * 1.0 / union_
        mask_idx = torch.nonzero(iou < overlap).squeeze()
        idx = idx.index_select(0, mask_idx)
    return keep, count


def reference_postprocess(arm_loc, arm_conf, odm_loc, odm_conf, net: int = NET, device="cpu", obj_thresh=0.01,
                          conf_thresh=0.01, nms_thresh=0.45, top_k: int = TOP_K, prior=None) -> np.ndarray:
    """doInference (:730-815) for one frame, statement by statement, on `device` -> [N, 6] float32, the driver's
    std::vector<float> rows (x1, y1, x2, y2, score, label)."""
    num_class = int(odm_conf.shape[1])
    m_prior = prior_box(net, device) if prior is None else prior
    arm_loc, arm_conf, odm_loc, odm_conf = (torch.as_tensor(np.asarray(h, np.float32)).to(device).to(torch.float64)
                                            .unsqueeze(0) for h in (arm_loc, arm_conf, odm_loc, odm_conf))
    arm_object_conf = arm_conf.squeeze(0).select(1, 1)
    object_index = (arm_object_conf > F32(obj_thresh)).unsqueeze(1)
    object_index_1 = object_index.expand_as(odm_conf.squeeze(0)).to(torch.float64)
    filter_odm_conf = odm_conf.squeeze(0).to(torch.float64) * object_index_1
    conf_preds = filter_odm_conf.clone().transpose(1, 0)
    default_m = decode(arm_loc[0], m_prior)
    decode_boxes_m = decode(odm_loc[0], default_m, True)
    result = []
    for i in range(1, num_class):
        c_mask_m = conf_preds[i] > F32(conf_thresh)
        nonzero_index = torch.nonzero(c_mask_m)
        score_m = torch.index_select(conf_preds[i], 0, nonzero_index.squeeze(1))
        boxes_m = torch.index_select(decode_boxes_m, 0, nonzero_index.squeeze(1))
        keep, count = nms(boxes_m, score_m, F32(nms_thresh), top_k)
        if count == 0:
            continue
        keep = keep[:count].clone()
        score_my = score_m.index_select(0, keep)
        boxes_my = boxes_m.index_select(0, keep)
        if np.float32(score_my[0].item()) < np.float32(conf_thresh):
            continue
        label = torch.full_like(score_my.unsqueeze(1), i)
        result.append(torch.cat([boxes_my, score_my.unsqueeze(1), label], 1))
    if not result:
        return np.zeros((0, 6), np.float32)
    return torch.cat(result, 0).cpu().numpy().astype(np.float32)


def as_dets(result: np.ndarray, max_det: int) -> np.ndarray:
    """[N, 6] rows -> the device layout [1 + max_det * 6]: min(N, max_det), the first rows, zeros."""
    out = np.zeros(1 + max_det * 6, np.float32)
    n = min(len(result), max_det)
    out[0] = n
    out[1:1 + 6 * n] = result[:n].ravel()
    return out


# ------------------------------------------------------------------ test inputs ----------------------------------------
def heads(B: int = 1, net: int = NET, C_: int = NUM_CLASSES, seed: int = 0, objects: int = 50, dense: int = 0,
          always=()):
    """Seeded engine heads [B, P, 4], [B, P, 2], [B, P, 4], [B, P, C] float32 with no tied candidate scores in a class:
    per class `objects` planted objects, each a prior with a high score and its anchors and neighbours with lower ones
    (overlapping boxes for the NMS), about one prior in 20 failing the ARM filter, and with `dense` > 0 that many extra
    candidates in classes 1 and 2 (above top_k: the cut).  The priors in `always` are candidates of every class.  Scores
    are distinct floats drawn from a permutation."""
    rng = np.random.default_rng(seed)
    P = num_priors(net)
    arm_loc = rng.normal(0, 0.5, (B, P, 4)).astype(np.float32)
    odm_loc = rng.normal(0, 0.5, (B, P, 4)).astype(np.float32)
    arm_conf = np.empty((B, P, 2), np.float32)
    arm_conf[..., 1] = rng.uniform(0.02, 1, (B, P)).astype(np.float32)
    arm_conf[..., 1][rng.random((B, P)) < 0.05] = np.float32(0.005)
    arm_conf[..., 0] = 1 - arm_conf[..., 1]
    odm_conf = rng.uniform(0, 0.009, (B, P, C_)).astype(np.float32)
    for b in range(B):
        for c in range(1, C_):
            picks = set()
            for p in rng.choice(P, objects, replace=False):
                base = p - p % 3
                picks.update(q for q in (base, base + 1, base + 2, base + 3, base + 4, base + 5, base - 3) if 0 <= q < P)
            if dense and c <= 2:
                picks.update(rng.choice(P, dense, replace=False).tolist())
            picks.update(int(q) for q in always)
            picks = np.array(sorted(picks))
            vals = np.linspace(0.0101, 0.99, len(picks), dtype=np.float32)
            odm_conf[b, picks, c] = rng.permutation(vals)
    return arm_loc, arm_conf, odm_loc, odm_conf
