"""Host-side mirror of the reference's plugin / helper interface for the hot path.

Same names, argument meaning and error behaviour as the reference classes, so the parity tests read
like the reference's call sites:

  YoloLayerPlugin        yolov8/plugin/yololayer.h:7-85      (IPluginV2IOExt; "YoloLayer_TRT" v1)
  YoloLayerPluginV5      yolov5/plugin/yololayer.h:10-82
  YoloPluginCreator      yolov8/plugin/yololayer.h:87-109    (field "combinedInfo", block.cpp:264-296)
  DecodePlugin           retinaface/decode.h:22-83           ("Decode_TRT" v1)
  RpnDecodePlugin / RpnNmsPlugin / PredictorDecodePlugin / BatchedNmsPlugin   rcnn/*Plugin.h
  batch_nms / cuda_decode+cuda_nms / cuda_batch_preprocess   yolov8/include/postprocess.h, preprocess.h

All compute goes through the C ABI of libtrtx_hot.so (include/trtx_hot.h); torch is used only for
device memory and streams.  There is no CPU fallback: without the library these classes raise.
"""
from __future__ import annotations

import ctypes as C
import math
import struct
from typing import Sequence

import torch

from . import _lib as L


def _ptr(t) -> int:
    if isinstance(t, torch.Tensor):
        if not t.is_cuda:
            raise L.TrtxError("expected a CUDA tensor (device pointer); host buffers are not accepted here")
        if not t.is_contiguous():
            raise L.TrtxError("tensor must be contiguous (TensorFormat::kLINEAR)")
        return t.data_ptr()
    return int(t)


def _elem_dtype(tensors, what: str, only=None) -> int:
    """TRTX_F32 / TRTX_F16 of tensors that share one element type: the tensors' dtype is the selector, no option to set.  A raw
    integer address carries no dtype and means fp32.  Another dtype, a mix, or a dtype other than `only` raises TrtxError,
    before the library is called with a pointer it would read as the wrong type."""
    codes = set()
    for t in tensors:
        if not isinstance(t, torch.Tensor):
            codes.add(L.F32)
        elif t.dtype == torch.float32:
            codes.add(L.F32)
        elif t.dtype == torch.float16:
            codes.add(L.F16)
        else:
            raise L.TrtxError(f"{what}: {t.dtype} tensors are not accepted (torch.float32 or torch.float16)")
    if len(codes) != 1:
        raise L.TrtxError(f"{what}: tensors of mixed dtypes (all torch.float32 or all torch.float16)")
    code = codes.pop()
    if only is not None and code != only:
        raise L.TrtxError(f"{what}: must be torch.float32")
    return code


def _stream(stream=None) -> int:
    if stream is None:
        return torch.cuda.current_stream().cuda_stream
    if isinstance(stream, torch.cuda.Stream):
        return stream.cuda_stream
    return int(stream)


def _nbytes(workspace: torch.Tensor) -> int:
    return workspace.numel() * workspace.element_size()


def _out_tensor(t, shape: tuple, dtype, device, what: str, alloc=torch.empty, contiguous: bool = True) -> torch.Tensor:
    """`t`, or a new tensor from alloc (torch.empty or torch.zeros) when t is None.  A given t of another shape or dtype
    raises ValueError(what), and so does a non-contiguous one when `contiguous` (else _ptr rejects it with TrtxError)."""
    if t is None:
        return alloc(shape, dtype=dtype, device=device)
    if tuple(t.shape) != tuple(shape) or t.dtype != dtype or (contiguous and not t.is_contiguous()):
        raise ValueError(what)
    return t


def float_le_threshold(x: float) -> float:
    """Largest fp32 t with t <= x: `(double)conf <= x`  <=>  `conf <= t` in fp32 (retinaface 0.1 / 0.02 literals)."""
    t = struct.unpack("f", struct.pack("f", x))[0]
    if t > x:
        t = float(torch.nextafter(torch.tensor(t, dtype=torch.float32), torch.tensor(-math.inf)).item())
    return t


def float_ge_threshold(x: float) -> float:
    """Smallest fp32 t with t >= x: `(double)conf < x`  <=>  `conf < t` in fp32 (retinaface's CONF_THRESH literal)."""
    t = struct.unpack("f", struct.pack("f", x))[0]
    if t < x:
        t = float(torch.nextafter(torch.tensor(t, dtype=torch.float32), torch.tensor(math.inf)).item())
    return t


# --------------------------------------------------------------------------------------------------
# YoloLayer_TRT: what every variant's mirror shares
# --------------------------------------------------------------------------------------------------
class _YoloLayerBase:
    """The YoloLayer_TRT surface common to all variants: one output of 1 + rows*DET_FLOATS floats per image, the workspace
    trtx_yolo_workspace_size asks for, and the trtx_yolo_decode_enqueue call on the subclass' `params` block."""
    PLUGIN_TYPE = "YoloLayer_TRT"
    PLUGIN_VERSION = "1"
    mThreadCount = 256  # serialized by the reference (yololayer.cu:80); unused here
    mPluginNamespace = ""

    @property
    def _max_rows(self) -> int:
        return self.mMaxOutObject

    def getNbOutputs(self) -> int:
        return 1

    def output_elems(self) -> int:
        return 1 + self._max_rows * self.DET_FLOATS

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return int(self._lib.trtx_yolo_workspace_size(C.byref(self.params), int(maxBatchSize)))

    def getPluginType(self) -> str:
        return self.PLUGIN_TYPE

    def getPluginVersion(self) -> str:
        return self.PLUGIN_VERSION

    def _decode(self, batch: int, inputs, output, workspace, stream, ws_bytes: int | None = None) -> int:
        """trtx_yolo_decode_enqueue of `inputs` (device tensors, one per level) into `output`; ws_bytes defaults to the size
        of the workspace tensor.  Returns the library's status, 0 on success."""
        ptrs = L.ptr_array([_ptr(t) for t in inputs])
        return int(self._lib.trtx_yolo_decode_enqueue(C.byref(self.params), int(batch), ptrs, _ptr(output), _ptr(workspace),
                                                      _nbytes(workspace) if ws_bytes is None else ws_bytes, _stream(stream)))


class _TunableYoloLayer(_YoloLayerBase):
    """The YoloLayer mirrors with tune(): all but YoloLayerPlugin26."""

    def tune(self, *, slices: int = 0, rows: int = 0, box: int = 0):
        """Per-plugin launch tuning of the scan kernel (trtx_yolo_params.tune_*; 0 = default).  Plain data inside the
        plugin's own parameter block -- nothing global, clones / other plugins are unaffected."""
        p = self.params
        p.tune_class_slices, p.tune_rows_in_flight, p.tune_box_prefetch = int(slices), int(rows), int(box)
        return self


# --------------------------------------------------------------------------------------------------
# YoloLayer_TRT, anchor-free (yolov8 / yolo11 / yolov12 / yolov13 ...)
# --------------------------------------------------------------------------------------------------
class YoloLayerPlugin(_TunableYoloLayer):
    DET_FLOATS = 90  # sizeof(Detection)/4, yolov8/include/types.h:4-12

    def __init__(self, classCount: int, numberofpoints: int, confthreshkeypoints: float, netWidth: int,
                 netHeight: int, maxOut: int, is_segmentation: bool, is_pose: bool, is_obb: bool,
                 strides: Sequence[int], in_dtype: int = L.F32):
        self.mClassCount = int(classCount)
        self.mNumberofpoints = int(numberofpoints)
        self.mConfthreshkeypoints = float(confthreshkeypoints)
        self.mYoloV8NetWidth = int(netWidth)
        self.mYoloV8netHeight = int(netHeight)
        self.mMaxOutObject = int(maxOut)
        self.is_segmentation_ = bool(is_segmentation)
        self.is_pose_ = bool(is_pose)
        self.is_obb_ = bool(is_obb)
        self.mStrides = [int(s) for s in strides]
        self.in_dtype = in_dtype
        self._lib = L.load()
        p = L.YoloParams()
        arr = (C.c_int * len(self.mStrides))(*self.mStrides)
        L.check(self._lib.trtx_yolo_params_init_v8(C.byref(p), self.mClassCount, self.mYoloV8NetWidth,
                                                  self.mYoloV8netHeight, self.mMaxOutObject, arr, len(self.mStrides)),
                "trtx_yolo_params_init_v8")
        p.det_floats = self.DET_FLOATS
        p.is_seg, p.is_pose, p.is_obb = int(self.is_segmentation_), int(self.is_pose_), int(self.is_obb_)
        p.num_kpts = self.mNumberofpoints
        p.kpt_thresh = self.mConfthreshkeypoints
        p.gate = 0.1  # literal of yololayer.cu:203
        p.in_dtype = in_dtype
        self.params = p

    # ---- IPluginV2 surface ----
    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        total = self.mMaxOutObject * self.DET_FLOATS  # yololayer.cu:107-111
        return (total + 1, 1, 1)

    def initialize(self) -> int:
        return 0

    def terminate(self) -> None:
        pass

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        """inputs: one device tensor per stride [B, C, g]; outputs[0]: [B, 1+maxOut*90] fp32; workspace: a device tensor or
        a raw pointer to getWorkspaceSize(batchSize) bytes; returns 0 on success."""
        ws_bytes = None if isinstance(workspace, torch.Tensor) else self.getWorkspaceSize(batchSize)
        return self._decode(batchSize, inputs, outputs[0], workspace, stream, ws_bytes)

    def supportsFormatCombination(self, pos, inOut, nbInputs, nbOutputs) -> bool:
        fmt, dtype = inOut[pos]
        if pos < nbInputs:
            return fmt == "kLINEAR" and dtype in (("kFLOAT",) if self.in_dtype == L.F32 else ("kHALF",))
        return fmt == "kLINEAR" and dtype == "kFLOAT"

    def getOutputDataType(self, index, inputTypes, nbInputs) -> str:
        return "kFLOAT"

    def setPluginNamespace(self, ns: str) -> None:
        self.mPluginNamespace = ns

    def getPluginNamespace(self) -> str:
        return self.mPluginNamespace

    def destroy(self) -> None:
        pass

    def clone(self) -> "YoloLayerPlugin":
        p = YoloLayerPlugin(self.mClassCount, self.mNumberofpoints, self.mConfthreshkeypoints, self.mYoloV8NetWidth,
                            self.mYoloV8netHeight, self.mMaxOutObject, self.is_segmentation_, self.is_pose_,
                            self.is_obb_, self.mStrides, self.in_dtype)
        p.setPluginNamespace(self.mPluginNamespace)
        return p

    # ---- serialization: byte layout of yololayer.cu:75-101 ----
    def getSerializationSize(self) -> int:
        return 4 * 8 + 4 * len(self.mStrides) + 3

    def serialize(self) -> bytes:
        d = struct.pack("<iifiiiii", self.mClassCount, self.mNumberofpoints, self.mConfthreshkeypoints,
                        self.mThreadCount, self.mYoloV8NetWidth, self.mYoloV8netHeight, self.mMaxOutObject,
                        len(self.mStrides))
        d += struct.pack(f"<{len(self.mStrides)}i", *self.mStrides)
        d += struct.pack("<???", self.is_segmentation_, self.is_pose_, self.is_obb_)
        assert len(d) == self.getSerializationSize()
        return d

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPlugin":
        cc, nk, kt, tc, w, h, mo, ns = struct.unpack_from("<iifiiiii", data, 0)
        strides = struct.unpack_from(f"<{ns}i", data, 32)
        seg, pose, obb = struct.unpack_from("<???", data, 32 + 4 * ns)
        if 32 + 4 * ns + 3 != len(data):
            raise L.TrtxError("YoloLayerPlugin.deserialize: length mismatch")  # assert(d == a + length)
        p = cls(cc, nk, kt, w, h, mo, seg, pose, obb, strides)
        p.mThreadCount = tc
        return p


class YoloPluginCreator:
    """yolov8/plugin/yololayer.cu:318-369."""

    def __init__(self):
        self.mNamespace = ""

    def getPluginName(self) -> str:
        return "YoloLayer_TRT"

    def getPluginVersion(self) -> str:
        return "1"

    def getFieldNames(self):
        return []

    def setPluginNamespace(self, ns: str) -> None:
        self.mNamespace = ns

    def getPluginNamespace(self) -> str:
        return self.mNamespace

    def createPlugin(self, name: str, fc: dict) -> YoloLayerPlugin:
        if len(fc) != 1 or "combinedInfo" not in fc:  # assert(fc->nbFields == 1), assert(strcmp(...)==0)
            raise L.TrtxError("YoloPluginCreator.createPlugin expects exactly one field 'combinedInfo'")
        ci = [int(v) for v in fc["combinedInfo"]]
        if len(ci) < 10:
            raise L.TrtxError("combinedInfo needs 9 net-info ints + at least one stride")
        obj = YoloLayerPlugin(ci[0], ci[1], float(ci[2]), ci[3], ci[4], ci[5], bool(ci[6]), bool(ci[7]), bool(ci[8]), ci[9:])
        obj.setPluginNamespace(self.mNamespace)
        return obj

    def deserializePlugin(self, name: str, data: bytes) -> YoloLayerPlugin:
        obj = YoloLayerPlugin.deserialize(data)
        obj.setPluginNamespace(self.mNamespace)
        return obj


# --------------------------------------------------------------------------------------------------
# YoloLayer_TRT, anchor-based (yolov5 / yolov7 ...)
# --------------------------------------------------------------------------------------------------
class YoloKernel:
    """yolov5/src/types.h:5-9."""

    def __init__(self, width: int, height: int, anchors: Sequence[float]):
        self.width, self.height = int(width), int(height)
        self.anchors = [float(a) for a in anchors]
        assert len(self.anchors) == 6


class YoloLayerPluginV5(_TunableYoloLayer):
    DET_FLOATS = 38  # yolov5/src/types.h:11-16

    def __init__(self, classCount: int, netWidth: int, netHeight: int, maxOut: int, is_segmentation: bool,
                 vYoloKernel: Sequence[YoloKernel], in_dtype: int = L.F32):
        self.mClassCount, self.mYoloV5NetWidth, self.mYoloV5NetHeight = int(classCount), int(netWidth), int(netHeight)
        self.mMaxOutObject = int(maxOut)
        self.is_segmentation_ = bool(is_segmentation)
        self.mYoloKernel = list(vYoloKernel)
        self.mKernelCount = len(self.mYoloKernel)
        self._lib = L.load()
        p = L.YoloParams()
        p.variant = L.YOLO_V5
        p.num_classes = self.mClassCount
        p.net_w, p.net_h = self.mYoloV5NetWidth, self.mYoloV5NetHeight
        p.max_out = self.mMaxOutObject
        p.det_floats = self.DET_FLOATS
        p.num_levels = self.mKernelCount
        for i, k in enumerate(self.mYoloKernel):
            p.grid_w[i], p.grid_h[i] = k.width, k.height
            for j in range(6):
                p.anchors[i][j] = k.anchors[j]
        p.is_seg = int(self.is_segmentation_)
        p.gate = 0.1  # kIgnoreThresh, yolov5/src/config.h:38
        p.in_dtype = in_dtype
        self.params = p

    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        return (self.mMaxOutObject * self.DET_FLOATS + 1, 1, 1)

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        return self._decode(batchSize, inputs, outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPluginV5":
        p = YoloLayerPluginV5(self.mClassCount, self.mYoloV5NetWidth, self.mYoloV5NetHeight, self.mMaxOutObject,
                              self.is_segmentation_, self.mYoloKernel, self.params.in_dtype)
        p.mPluginNamespace = self.mPluginNamespace
        return p

    # byte layout of yolov5/plugin/yololayer.cu:48-83
    def serialize(self) -> bytes:
        d = struct.pack("<iiiiii?", self.mClassCount, self.mThreadCount, self.mKernelCount, self.mYoloV5NetWidth,
                        self.mYoloV5NetHeight, self.mMaxOutObject, self.is_segmentation_)
        for k in self.mYoloKernel:
            d += struct.pack("<ii6f", k.width, k.height, *k.anchors)
        return d

    def getSerializationSize(self) -> int:
        return 25 + 32 * self.mKernelCount

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPluginV5":
        cc, tc, kc, w, h, mo, seg = struct.unpack_from("<iiiiii?", data, 0)
        ks = []
        for i in range(kc):
            v = struct.unpack_from("<ii6f", data, 25 + 32 * i)
            ks.append(YoloKernel(v[0], v[1], v[2:]))
        if 25 + 32 * kc != len(data):
            raise L.TrtxError("YoloLayerPluginV5.deserialize: length mismatch")
        p = cls(cc, w, h, mo, seg, ks)
        p.mThreadCount = tc
        return p


class YoloLayerPluginV7(YoloLayerPluginV5):
    """yolov7/plugin/yololayer.h:9-73 (same kernel arithmetic as yolov5, yolov7/plugin/yololayer.cu:152-200, but
    Detection = 6 floats, yolov7/include/types.h:11-16; also yolov10 / yolov13 style rows).  No segmentation flag:
    ctor (classCount, netWidth, netHeight, maxOut, vYoloKernel), serialization without the bool.  YOLOP's plugin
    (yolop/yololayer.h) is this one with YOLOP's arguments: (1, 640, 384, 1000, kernels with the stride-32 one first)."""
    DET_FLOATS = 6

    def __init__(self, classCount: int, netWidth: int, netHeight: int, maxOut: int, vYoloKernel: Sequence[YoloKernel],
                 in_dtype: int = L.F32):
        super().__init__(classCount, netWidth, netHeight, maxOut, False, vYoloKernel, in_dtype)

    def clone(self) -> "YoloLayerPluginV7":
        p = YoloLayerPluginV7(self.mClassCount, self.mYoloV5NetWidth, self.mYoloV5NetHeight, self.mMaxOutObject,
                              self.mYoloKernel, self.params.in_dtype)
        p.mPluginNamespace = self.mPluginNamespace
        return p

    def serialize(self) -> bytes:  # yolov7/plugin/yololayer.cu:62-77
        d = struct.pack("<iiiiii", self.mClassCount, self.mThreadCount, self.mKernelCount, self.mYoloV5NetWidth,
                        self.mYoloV5NetHeight, self.mMaxOutObject)
        for k in self.mYoloKernel:
            d += struct.pack("<ii6f", k.width, k.height, *k.anchors)
        return d

    def getSerializationSize(self) -> int:
        return 24 + 32 * self.mKernelCount

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPluginV7":
        cc, tc, kc, w, h, mo = struct.unpack_from("<iiiiii", data, 0)
        if 24 + 32 * kc != len(data):
            raise L.TrtxError("YoloLayerPluginV7.deserialize: length mismatch")
        ks = []
        for i in range(kc):
            v = struct.unpack_from("<ii6f", data, 24 + 32 * i)
            ks.append(YoloKernel(v[0], v[1], v[2:]))
        p = cls(cc, w, h, mo, ks)
        p.mThreadCount = tc
        return p


class YoloKernelV3:
    """Yolo::YoloKernel of yolov3-spp/yololayer.h:20-26: width, height (dynamic, -1 until enqueue), stride, anchors."""

    def __init__(self, width: int, height: int, stride: int, anchors: Sequence[float]):
        self.width, self.height, self.stride = int(width), int(height), int(stride)
        self.anchors = [float(a) for a in anchors]
        assert len(self.anchors) == 6


# yolo1..3 of yolov3-spp/yololayer.h:27-44 (the plugin's level order: stride 32, 16, 8)
YOLOV3_KERNELS = (YoloKernelV3(-1, -1, 32, (116, 90, 156, 198, 373, 326)),
                  YoloKernelV3(-1, -1, 16, (30, 61, 62, 45, 59, 119)),
                  YoloKernelV3(-1, -1, 8, (10, 13, 16, 30, 33, 23)))


class YoloLayerPluginV3(_TunableYoloLayer):
    """yolov3-spp/yololayer.h:58-121 (IPluginV2DynamicExt "YoloLayer_TRT" v1).  yolov3, yolov4, scaled-yolov4 and yolov3-tiny
    carry another plugin with other box arithmetic: YoloLayerPluginV3Net.
    The reference compiles CLASS_NUM, the kernels and MAX_OUTPUT_BBOX_COUNT in; here they are constructor arguments with
    the reference's values as defaults.  enqueue() takes the grids from the input tensors like the reference
    (yololayer.cu:207-216)."""
    DET_FLOATS = 7  # x,y,w,h, det_confidence, class_id, class_confidence (yololayer.h:47-53)

    def __init__(self, classCount: int = 80, kernels: Sequence[YoloKernelV3] = YOLOV3_KERNELS, maxOut: int = 1000,
                 in_dtype: int = L.F32):
        self.mClassCount, self.mYoloKernel, self.mMaxOutObject = int(classCount), list(kernels), int(maxOut)
        self.mKernelCount = len(self.mYoloKernel)
        self._lib = L.load()
        p = L.YoloParams()
        p.variant = L.YOLO_V3
        p.num_classes, p.max_out, p.det_floats, p.num_levels = self.mClassCount, self.mMaxOutObject, self.DET_FLOATS, self.mKernelCount
        for i, k in enumerate(self.mYoloKernel):
            p.strides[i] = k.stride
            p.grid_w[i], p.grid_h[i] = max(k.width, 1), max(k.height, 1)
            for j in range(6):
                p.anchors[i][j] = k.anchors[j]
        p.gate = 0.1  # IGNORE_THRESH, yololayer.h:15
        p.in_dtype = in_dtype
        self.params = p

    def configure(self, inputs) -> None:
        """grid = dims 2, 3 of every input tensor [B, 3*(5+nc), gh, gw] (yololayer.cu:209-212)."""
        for i, t in enumerate(inputs):
            self.params.grid_h[i], self.params.grid_w[i] = int(t.shape[2]), int(t.shape[3])

    def enqueue(self, inputs, outputs, workspace=None, stream=None) -> int:
        """IPluginV2DynamicExt::enqueue: batch = inputs[0].shape[0]."""
        self.configure(inputs)
        batch = int(inputs[0].shape[0])
        if workspace is None:
            workspace = torch.empty(self.getWorkspaceSize(batch), dtype=torch.uint8, device=inputs[0].device)
        return self._decode(batch, inputs, outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPluginV3":
        p = YoloLayerPluginV3(self.mClassCount, self.mYoloKernel, self.mMaxOutObject, self.params.in_dtype)
        p.mPluginNamespace = self.mPluginNamespace
        return p

    # byte layout of yolov3-spp/yololayer.cu:36-71: classCount, threadCount, kernelCount, kernels {w, h, stride, anchors[6]}
    def serialize(self) -> bytes:
        d = struct.pack("<iii", self.mClassCount, self.mThreadCount, self.mKernelCount)
        for k in self.mYoloKernel:
            d += struct.pack("<iii6f", k.width, k.height, k.stride, *k.anchors)
        return d

    def getSerializationSize(self) -> int:
        return 12 + 36 * self.mKernelCount

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPluginV3":
        cc, tc, kc = struct.unpack_from("<iii", data, 0)
        if 12 + 36 * kc != len(data):
            raise L.TrtxError("YoloLayerPluginV3.deserialize: length mismatch")
        ks = []
        for i in range(kc):
            v = struct.unpack_from("<iii6f", data, 12 + 36 * i)
            ks.append(YoloKernelV3(v[0], v[1], v[2], v[3:]))
        p = cls(cc, ks)
        p.mThreadCount = tc
        return p


class YoloLayerPluginV3Net(_TunableYoloLayer):
    """The YoloLayer_TRT of yolov3, yolov4, scaled-yolov4 and yolov3-tiny (yolov4/yololayer.h:52-121, IPluginV2IOExt): grids,
    anchors, the net size and MAX_OUTPUT_BBOX_COUNT are compile-time constants of each driver's yololayer.h, and its blob,
    classCount, threadCount, kernelCount, YoloKernel{int width, height; float anchors[6]}[n] (yolov4/yololayer.cu:58-70), does
    not say which box formula applies.  So the net size and `variant` (YOLO_V3_NET: yolov3, yolov3-tiny; YOLO_V4: yolov4;
    YOLO_V4_CSP: scaled-yolov4) are constructor arguments; V3_FAMILY_DRIVERS holds each driver's values."""
    DET_FLOATS = 7  # x,y,w,h, det_confidence, class_id, class_confidence (yolov4/yololayer.h:41-48)

    def __init__(self, classCount: int, kernels: Sequence[YoloKernel], netWidth: int, netHeight: int, variant: int,
                 maxOut: int = 1000, in_dtype: int = L.F32):
        if variant not in (L.YOLO_V3_NET, L.YOLO_V4, L.YOLO_V4_CSP):
            raise ValueError("variant must be YOLO_V3_NET, YOLO_V4 or YOLO_V4_CSP")
        self.mClassCount, self.mYoloKernel, self.mMaxOutObject = int(classCount), list(kernels), int(maxOut)
        self.mKernelCount = len(self.mYoloKernel)
        self.net_w, self.net_h, self.variant = int(netWidth), int(netHeight), int(variant)
        self._lib = L.load()
        p = L.YoloParams()
        p.variant = self.variant
        p.num_classes, p.max_out, p.det_floats, p.num_levels = self.mClassCount, self.mMaxOutObject, self.DET_FLOATS, self.mKernelCount
        p.net_w, p.net_h = self.net_w, self.net_h
        for i, k in enumerate(self.mYoloKernel):
            p.grid_w[i], p.grid_h[i] = k.width, k.height
            for j in range(6):
                p.anchors[i][j] = k.anchors[j]
        p.gate = 0.1  # IGNORE_THRESH, yolov4/yololayer.h:11
        p.in_dtype = in_dtype
        self.params = p

    @classmethod
    def for_driver(cls, driver: str, in_dtype: int = L.F32) -> "YoloLayerPluginV3Net":
        """The plugin a driver's YoloPluginCreator::createPlugin builds: its yololayer.h constants (V3_FAMILY_DRIVERS)."""
        d = V3_FAMILY_DRIVERS[driver]
        return cls(d["classes"], [YoloKernel(w, h, a) for w, h, a in d["kernels"]], d["net"][0], d["net"][1], d["variant"],
                   d["max_out"], in_dtype)

    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        return (self.mMaxOutObject * self.DET_FLOATS + 1, 1, 1)  # yolov4/yololayer.cu:82-86

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        return self._decode(batchSize, inputs, outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPluginV3Net":
        p = YoloLayerPluginV3Net(self.mClassCount, self.mYoloKernel, self.net_w, self.net_h, self.variant, self.mMaxOutObject,
                                 self.params.in_dtype)
        p.mPluginNamespace = self.mPluginNamespace
        return p

    def serialize(self) -> bytes:
        d = struct.pack("<iii", self.mClassCount, self.mThreadCount, self.mKernelCount)
        for k in self.mYoloKernel:
            d += struct.pack("<ii6f", k.width, k.height, *k.anchors)
        return d

    def getSerializationSize(self) -> int:
        return 12 + 32 * self.mKernelCount

    @classmethod
    def deserialize(cls, data: bytes, netWidth: int, netHeight: int, variant: int, maxOut: int = 1000) -> "YoloLayerPluginV3Net":
        """The blob does not hold the net size, the box formula or maxOut: the caller supplies them, as the driver's
        compiled-in constants do."""
        if len(data) < 12:
            raise L.TrtxError("YoloLayerPluginV3Net.deserialize: length mismatch")
        cc, tc, kc = struct.unpack_from("<iii", data, 0)
        if kc <= 0 or 12 + 32 * kc != len(data):
            raise L.TrtxError("YoloLayerPluginV3Net.deserialize: length mismatch")
        ks = []
        for i in range(kc):
            v = struct.unpack_from("<ii6f", data, 12 + 32 * i)
            ks.append(YoloKernel(v[0], v[1], v[2:]))
        p = cls(cc, ks, netWidth, netHeight, variant, maxOut)
        p.mThreadCount = tc
        return p


# Each driver's compiled-in constants (its yololayer.h: CLASS_NUM, INPUT_W x INPUT_H, the YoloKernel table in the plugin's
# level order, MAX_OUTPUT_BBOX_COUNT), its decode variant, and its NMS as library parameters: nms() drops
# `det_confidence <= BBOX_CONF_THRESH` (a double literal; conf_thresh is the float with the same verdict) and erases on
# `iou > NMS_THRESH`.
_V4_ANCHORS = ((12, 16, 19, 36, 40, 28), (36, 75, 76, 55, 72, 146), (142, 110, 192, 243, 459, 401))
V3_FAMILY_DRIVERS = {
    "yolov3": dict(variant=L.YOLO_V3_NET, net=(608, 608), classes=80, max_out=1000,
                   kernels=((19, 19, (116, 90, 156, 198, 373, 326)), (38, 38, (30, 61, 62, 45, 59, 119)),
                            (76, 76, (10, 13, 16, 30, 33, 23))), conf_thresh=0.5, nms_thresh=0.4),
    "yolov4": dict(variant=L.YOLO_V4, net=(608, 608), classes=80, max_out=1000,
                   kernels=tuple((608 // s, 608 // s, a) for s, a in zip((8, 16, 32), _V4_ANCHORS)), conf_thresh=0.5,
                   nms_thresh=0.4),
    "scaled-yolov4": dict(variant=L.YOLO_V4_CSP, net=(512, 512), classes=80, max_out=1000,
                          kernels=tuple((512 // s, 512 // s, a) for s, a in zip((8, 16, 32), _V4_ANCHORS)), conf_thresh=0.5,
                          nms_thresh=0.4),
    # yolov3-tiny.cpp:27-28: BBOX_CONF_THRESH 0.4 compared as a double with `<=`, so the float just below 0.4f
    "yolov3-tiny": dict(variant=L.YOLO_V3_NET, net=(608, 608), classes=80, max_out=1000,
                        kernels=((19, 19, (81, 82, 135, 169, 344, 319)), (38, 38, (23, 27, 37, 58, 81, 82))),
                        conf_thresh=float_le_threshold(0.4), nms_thresh=0.5),
}


class YoloLayerPluginV9(_TunableYoloLayer):
    """yolov9/plugin/yololayer.h ("YoloLayer_TRT" v1 of yolov9, IPluginV2IOExt): ctor (classCount, netWidth, netHeight,
    maxOut, is_segmentation).  The strides 8, 16, 32 and grids net / stride are compiled in (yololayer.cu:185-187); yolov8's
    decode into 38-float rows (box l, t, r, b, conf, class, 32 mask coefficients when is_segmentation).  Blob: classCount,
    threadCount, netWidth, netHeight, maxOut, is_segmentation = 21 bytes (yololayer.cu:48-60).  TensorRT creator:
    trtx::YoloV9PluginCreator (include/trtx_plugins.h)."""
    DET_FLOATS = 38  # yolov9/include/types.h
    STRIDES = (8, 16, 32)

    def __init__(self, classCount: int, netWidth: int, netHeight: int, maxOut: int, is_segmentation: bool,
                 in_dtype: int = L.F32):
        self.mClassCount, self.mYoloV8NetWidth, self.mYoloV8netHeight = int(classCount), int(netWidth), int(netHeight)
        self.mMaxOutObject, self.is_segmentation_ = int(maxOut), bool(is_segmentation)
        self._lib = L.load()
        self.params = _anchor_free_params(self._lib, self.mClassCount, self.mYoloV8NetWidth, self.mYoloV8netHeight,
                                          self.mMaxOutObject, self.STRIDES, self.DET_FLOATS, self.is_segmentation_, in_dtype)

    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        return (self.mMaxOutObject * self.DET_FLOATS + 1, 1, 1)  # yololayer.cu:70-73

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        return self._decode(batchSize, inputs, outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPluginV9":
        p = YoloLayerPluginV9(self.mClassCount, self.mYoloV8NetWidth, self.mYoloV8netHeight, self.mMaxOutObject,
                              self.is_segmentation_, self.params.in_dtype)
        p.mPluginNamespace, p.mThreadCount = self.mPluginNamespace, self.mThreadCount
        return p

    def serialize(self) -> bytes:
        return struct.pack("<iiiii?", self.mClassCount, self.mThreadCount, self.mYoloV8NetWidth, self.mYoloV8netHeight,
                           self.mMaxOutObject, self.is_segmentation_)

    def getSerializationSize(self) -> int:
        return 21

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPluginV9":
        if len(data) != 21 or data[20] > 1:
            raise L.TrtxError("YoloLayerPluginV9.deserialize: not a 21-byte yolov9 blob")
        cc, tc, w, h, mo, seg = struct.unpack("<iiiii?", data)
        p = cls(cc, w, h, mo, seg)
        p.mThreadCount = tc
        return p


class YoloLayerPluginV10(_TunableYoloLayer):
    """yolov10/plugin/yololayer.h and yolov13's, the same class ("YoloLayer_TRT" v1, IPluginV2IOExt): ctor (classCount,
    netWidth, netHeight, maxOut, strides).  yolov8's decode into 6-float rows (box l, t, r, b, conf, class).  Blob: classCount,
    threadCount, netWidth, netHeight, maxOut, len(strides), strides = 24 + 4n bytes (yololayer.cu:64-84).  TensorRT creator:
    trtx::YoloV10PluginCreator (include/trtx_plugins.h)."""
    DET_FLOATS = 6  # yolov10/include/types.h, yolov13/include/types.h

    def __init__(self, classCount: int, netWidth: int, netHeight: int, maxOut: int, strides: Sequence[int],
                 in_dtype: int = L.F32):
        self.mClassCount, self.mYoloV10NetWidth, self.mYoloV10netHeight = int(classCount), int(netWidth), int(netHeight)
        self.mMaxOutObject, self.mStrides = int(maxOut), [int(s) for s in strides]
        self._lib = L.load()
        self.params = _anchor_free_params(self._lib, self.mClassCount, self.mYoloV10NetWidth, self.mYoloV10netHeight,
                                          self.mMaxOutObject, self.mStrides, self.DET_FLOATS, False, in_dtype)

    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        return (self.mMaxOutObject * self.DET_FLOATS + 1, 1, 1)  # yololayer.cu:90-94

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        return self._decode(batchSize, inputs, outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPluginV10":
        p = YoloLayerPluginV10(self.mClassCount, self.mYoloV10NetWidth, self.mYoloV10netHeight, self.mMaxOutObject,
                               self.mStrides, self.params.in_dtype)
        p.mPluginNamespace, p.mThreadCount = self.mPluginNamespace, self.mThreadCount
        return p

    def serialize(self) -> bytes:
        n = len(self.mStrides)
        return struct.pack(f"<6i{n}i", self.mClassCount, self.mThreadCount, self.mYoloV10NetWidth, self.mYoloV10netHeight,
                           self.mMaxOutObject, n, *self.mStrides)

    def getSerializationSize(self) -> int:
        return 24 + 4 * len(self.mStrides)

    @classmethod
    def deserialize(cls, data: bytes) -> "YoloLayerPluginV10":
        if len(data) < 24:
            raise L.TrtxError("YoloLayerPluginV10.deserialize: length mismatch")
        cc, tc, w, h, mo, n = struct.unpack_from("<6i", data, 0)
        if not 1 <= n <= L.MAX_LEVELS or len(data) != 24 + 4 * n:
            raise L.TrtxError("YoloLayerPluginV10.deserialize: length mismatch")
        p = cls(cc, w, h, mo, struct.unpack_from(f"<{n}i", data, 24))
        p.mThreadCount = tc
        return p


def _anchor_free_params(lib, nc, w, h, max_out, strides, det_floats, seg, in_dtype) -> L.YoloParams:
    """TRTX_YOLO_V8 parameters for yolov9 / yolov10 / yolov13: each one's CalDetection is yolov8's arithmetic."""
    p = L.YoloParams()
    arr = (C.c_int * len(strides))(*strides)
    L.check(lib.trtx_yolo_params_init_v8(C.byref(p), nc, w, h, max_out, arr, len(strides)), "trtx_yolo_params_init_v8")
    p.det_floats, p.is_seg, p.in_dtype = det_floats, int(seg), in_dtype
    return p


# Each driver's compiled-in constants (config.h) and its host post-process as library parameters:
#   yolov9: nms() (src/postprocess.cpp:48-83) on rows i < kMaxNumOutputBbox, `conf <= kConfThresh` dropped, boxes converted to
#     cx, cy, w, h (BOX_V9), `iou > kNmsThresh` erased, conf-only sort (no box[0] tie-break); get_rect is yolov5's, unclamped;
#   yolov10: get_topk (:35-44), no NMS: yolo_topk_postprocess with yolov8's clamped get_rect (YOLO_V8);
#   yolov13: yolov8's nms() (isnan guard, box[0] tie-break) on l, t, r, b rows, and yolov8's get_rect.  Its device post-process
#     (postprocess.cu) strides 7-float rows by bbox_element = 4 and is not followed (DESIGN.md section 2).
ANCHOR_FREE_DRIVERS = {
    "yolov9": dict(plugin=YoloLayerPluginV9, net=(640, 640), classes=80, max_out=2000, det_floats=38, conf_thresh=0.1,
                   nms_thresh=0.45, box_format=L.BOX_V9, mode=L.NMS_GREEDY, tie_break_x0=False, rect=L.YOLO_V5),
    "yolov10": dict(plugin=YoloLayerPluginV10, net=(640, 640), classes=80, max_out=1000, det_floats=6, conf_thresh=0.5,
                    nms_thresh=None, box_format=None, mode=None, tie_break_x0=None, rect=L.YOLO_V8),
    "yolov13": dict(plugin=YoloLayerPluginV10, net=(640, 640), classes=80, max_out=1000, det_floats=6, conf_thresh=0.5,
                    nms_thresh=0.45, box_format=L.BOX_LTRB, mode=L.NMS_GREEDY, tie_break_x0=True, rect=L.YOLO_V8),
}


class YoloLayerPlugin26(_YoloLayerBase):
    """yolo26/plugin/yololayer.h:10-77 ("YoloLayer_TRT" v1 of the NMS-free yolo26 heads): ctor (classCount, numberOfPoints,
    maxDetections, isDetection, isSegmentation, isPose, isObb, anchor_count); setPluginDeviceParams(confThreshold) of the
    reference is the `conf_thresh` argument here (no device global).  One input [B, anchor_count, 4+nc(+1)]."""
    DET_FLOATS = 90  # yolo26/include/types.h

    def __init__(self, classCount: int, numberOfPoints: int, maxDetections: int, isDetection: bool, isSegmentation: bool,
                 isPose: bool, isObb: bool, anchor_count: int, conf_thresh: float = 0.4):
        self.mClassCount, self.mNumberOfPoints, self.mMaxDetections = int(classCount), int(numberOfPoints), int(maxDetections)
        self.mIsDetection, self.mIsSegmentation, self.mIsPose, self.mIsObb = bool(isDetection), bool(isSegmentation), bool(isPose), bool(isObb)
        self.mAnchorCount = int(anchor_count)
        self._lib = L.load()
        p = L.YoloParams()
        p.variant = L.YOLO_V26
        p.num_classes, p.max_out, p.det_floats, p.num_levels = self.mClassCount, self.mMaxDetections, self.DET_FLOATS, 1
        p.grid_h[0], p.grid_w[0] = 1, self.mAnchorCount
        p.is_seg, p.is_pose, p.is_obb = int(self.mIsSegmentation), int(self.mIsPose), int(self.mIsObb)
        p.num_kpts = self.mNumberOfPoints
        p.gate = float(conf_thresh)  # d_confThreshold, yololayer.cu:9 / setPluginDeviceParams :31-33
        p.in_dtype = L.F32
        self.params = p

    @property
    def _max_rows(self) -> int:
        return self.mMaxDetections

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        return self._decode(batchSize, (inputs[0],), outputs[0], workspace, stream)

    def clone(self) -> "YoloLayerPlugin26":
        p = YoloLayerPlugin26(self.mClassCount, self.mNumberOfPoints, self.mMaxDetections, self.mIsDetection, self.mIsSegmentation,
                              self.mIsPose, self.mIsObb, self.mAnchorCount, self.params.gate)
        p.mPluginNamespace = self.mPluginNamespace
        return p

    # byte layout of yolo26/plugin/yololayer.cu:68-100 (4 ints, 4 bools, 1 int)
    def serialize(self) -> bytes:
        return struct.pack("<iiii????i", self.mClassCount, self.mNumberOfPoints, self.mThreadCount, self.mMaxDetections,
                           self.mIsDetection, self.mIsSegmentation, self.mIsPose, self.mIsObb, self.mAnchorCount)

    def getSerializationSize(self) -> int:
        return 24

    @classmethod
    def deserialize(cls, data: bytes, conf_thresh: float = 0.4) -> "YoloLayerPlugin26":
        if len(data) != 24:
            raise L.TrtxError("YoloLayerPlugin26.deserialize: length mismatch")
        cc, nk, tc, md, d, sg, po, ob, ac = struct.unpack("<iiii????i", data)
        p = cls(cc, nk, md, d, sg, po, ob, ac, conf_thresh)
        p.mThreadCount = tc
        return p


# --------------------------------------------------------------------------------------------------
# NMS helpers (postprocess.h)
# --------------------------------------------------------------------------------------------------
def nms_params(box_format=L.BOX_LTRB, mode=L.NMS_GREEDY, conf_thresh=0.5, nms_thresh=0.45, max_det=1000,
               class_aware=True, tie_break_x0=None, extra_floats=0, extra_offset=0) -> L.NmsParams:
    q = L.NmsParams()
    q.box_format, q.mode = box_format, mode
    q.conf_thresh, q.nms_thresh = conf_thresh, nms_thresh
    q.max_det = max_det
    q.class_aware = int(class_aware)
    q.tie_break_x0 = int(box_format in (L.BOX_LTRB, L.BOX_OBB) if tie_break_x0 is None else tie_break_x0)  # v8 cmp, postprocess.cpp:87-92
    q.extra_floats, q.extra_offset = extra_floats, extra_offset
    return q


def batch_nms(output: torch.Tensor, batch_size: int, output_size: int, conf_thresh: float, nms_thresh: float = 0.5,
              box_format: int = L.BOX_LTRB, det_floats: int = 90, max_det: int | None = None, mode: int = L.NMS_GREEDY,
              extra_floats: int = 0, extra_offset: int = 0, return_index: bool = False, stream=None):
    """GPU drop-in for batch_nms() (yolov8/src/postprocess.cpp:123-129): `output` is the plugin buffer
    [batch, output_size] on the device; returns the compact buffer [batch, 1 + max_det*(7+extra)]."""
    lib = L.load()
    max_rows = (output_size - 1) // det_floats
    max_det = max_det or max_rows
    q = nms_params(box_format, mode, conf_thresh, nms_thresh, max_det, box_format != L.BOX_RETINA,
                   extra_floats=extra_floats, extra_offset=extra_offset)
    R = 7 + extra_floats
    out = torch.empty((batch_size, 1 + max_det * R), dtype=torch.float32, device=output.device)
    idx = torch.empty((batch_size, max_det), dtype=torch.int32, device=output.device) if return_index else None
    ws_bytes = int(lib.trtx_nms_workspace_size(C.byref(q), batch_size, max_rows))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=output.device)
    L.check(lib.trtx_nms_enqueue(C.byref(q), batch_size, _ptr(output), max_rows, det_floats, _ptr(out),
                                 _ptr(idx) if idx is not None else None, _ptr(ws), ws_bytes, _stream(stream)),
            "trtx_nms_enqueue")
    return (out, idx) if return_index else out


def batch_nms_obb(output: torch.Tensor, batch_size: int, output_size: int, conf_thresh: float, nms_thresh: float = 0.5,
                  max_det: int | None = None, mode: int = L.NMS_GREEDY, return_index: bool = False, stream=None):
    """GPU drop-in for batch_nms_obb() (yolov8/src/postprocess.cpp:387-393; mode=NMS_ONESHOT: cuda_decode_obb +
    cuda_nms_obb, postprocess.cu:7-40,147-193): oriented boxes, ProbIoU.  Returns [batch, 1 + max_det*8] rows
    (cx, cy, w, h, conf, cls, keep, angle) -- the 8-float element decode_kernel_obb writes."""
    return batch_nms(output, batch_size, output_size, conf_thresh, nms_thresh, box_format=L.BOX_OBB, det_floats=90,
                     max_det=max_det, mode=mode, extra_floats=1, extra_offset=89, return_index=return_index, stream=stream)


def process_mask(proto: torch.Tensor, dets: torch.Tensor, max_rows: int, row_floats: int = 39, coeff_offset: int = 7,
                 max_masks: int = 100, net_w: int = 640, net_h: int = 640, variant: int = L.YOLO_V8, out=None, stream=None):
    """GPU drop-in for process_mask() (yolov8/yolov8_seg.cpp:36-60, yolov5/src/postprocess.cpp:106-125) for the whole
    batch: proto [B, 32, net_h/4, net_w/4]; dets [B, 1 + max_rows*row_floats] (count, rows; e.g. batch_nms(...,
    extra_floats=32, extra_offset=6) output) -> masks [B, max_masks, net_h, net_w]; slots >= count are not written."""
    lib = L.load()
    B, nm, mh, mw = proto.shape
    q = L.MaskParams(variant, net_w, net_h, mw, mh, nm, row_floats, coeff_offset, max_masks)
    if out is None:
        out = torch.zeros((B, max_masks, net_h, net_w), dtype=torch.float32, device=proto.device)
    L.check(lib.trtx_process_mask_enqueue(C.byref(q), B, _ptr(proto), _ptr(dets), max_rows, _ptr(out), _stream(stream)),
            "trtx_process_mask_enqueue")
    return out


def _frames(sizes: Sequence[tuple[int, int]], canvases: Sequence[torch.Tensor] | None, max_masks: int, device,
            with_canvases: bool):
    """trtx_frame descriptors for frames of sizes[b] = (img_w, img_h) and, with_canvases, their u8 canvases
    [max_masks, img_h, img_w]: the caller's `canvases` (any u8 tensors with contiguous rows and slots, e.g. views
    [..., :img_w] of pitched buffers) or new zeroed ones.  -> (descriptors, list of canvases or None)"""
    B = len(sizes)
    if not with_canvases:
        canvases = None
    elif canvases is None:
        canvases = [torch.zeros((max_masks, h, w), dtype=torch.uint8, device=device) for w, h in sizes]
    elif len(canvases) != B:
        raise ValueError(f"expected {B} canvases")
    descs = (L.Frame * B)()
    for b, (w, h) in enumerate(sizes):
        descs[b].img_w, descs[b].img_h = int(w), int(h)
        if canvases is not None:
            c = canvases[b]
            if c.dtype != torch.uint8 or tuple(c.shape) != (max_masks, h, w) or c.stride(2) != 1 or \
                    c.stride(0) != h * c.stride(1):
                raise ValueError(f"canvas {b} must be u8 [{max_masks}, {h}, {w}] with contiguous rows and slots")
            descs[b].masks_dev = c.data_ptr()
            descs[b].pitch = int(c.stride(1))
    return descs, (list(canvases) if canvases is not None else None)


def _f32_rows(dets: torch.Tensor) -> None:
    """Per-row entries read dets [B, 1 + rows*F] as dense float32 rows."""
    if dets.dtype != torch.float32 or dets.stride(1) != 1 or dets.stride(0) != dets.shape[1]:
        raise ValueError("dets must be contiguous float32")


def _frame_wh(image_sizes: Sequence[tuple[int, int]]):
    """The per-row entries' host int32 array (img_w, img_h) of every frame."""
    return (C.c_int32 * (2 * len(image_sizes)))(*[int(v) for s in image_sizes for v in s])


def yolo_seg_postprocess(proto: torch.Tensor | None, dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *,
                         variant: int, max_rows: int, row_floats: int = 39, coeff_offset: int = 7, max_masks: int,
                         net_w: int = 640, net_h: int = 640, masks: bool = True, rows_out: torch.Tensor | None = None,
                         canvases_out: Sequence[torch.Tensor] | None = None, stream=None):
    """GPU drop-in for the segmentation models' post-process after NMS: process_mask + scale_mask + draw_mask_bbox's mask
    selection (yolov8/src/postprocess.cpp:228-248, yolov5/src/postprocess.cpp:148-167) for a batch of frames of any sizes.
    proto [B, 32, net_h/4, net_w/4] (may be None with masks=False); dets [B, 1 + max_rows*row_floats] (count, rows);
    image_sizes[b] = (img_w, img_h) of frame b ->
    (rows [B, 1 + max_rows*6] fp32: count, then (x, y, w, h, conf, class) with x, y, w, h = get_rect(img, bbox);
    variant YOLO_V3 or RECT_YOLOV3_SPP, with masks=False, maps the NMS rows of yolov3 / yolov4 / scaled-yolov4 /
    yolov3-tiny or yolov3-spp (net_w = net_h = MAX_INPUT_SIZE) by their get_rect;
     per-image u8 canvases [max_masks, img_h, img_w]: 255 where draw_mask_bbox would colour the pixel, or None with masks=False).
    `canvases_out[b]` may be any u8 cuda tensor [max_masks, img_h, img_w] with contiguous rows and slots (e.g. a view
    [..., :img_w] of a pitched buffer);
    canvases at or past an image's count are not written (new ones start zeroed).  Two launches per 64 images."""
    lib = L.load()
    B = len(image_sizes)
    if dets.dim() != 2 or dets.shape[0] != B or dets.shape[1] < 1 + max_rows * row_floats:
        raise ValueError(f"dets must be [{B}, >= {1 + max_rows * row_floats}]")
    nm, mh, mw = (proto.shape[1], proto.shape[2], proto.shape[3]) if proto is not None else (32, net_h // 4, net_w // 4)
    q = L.MaskParams(variant, net_w, net_h, mw, mh, nm, row_floats, coeff_offset, max_masks)
    if rows_out is None:
        rows_out = torch.empty((B, 1 + max_rows * 6), dtype=torch.float32, device=dets.device)
    descs, canvases_out = _frames(image_sizes, canvases_out, max_masks, dets.device, masks)
    L.check(lib.trtx_yolo_seg_postprocess_enqueue(C.byref(q), descs, B, None if proto is None else _ptr(proto), _ptr(dets),
                                                  max_rows, _ptr(rows_out), _stream(stream)),
            "trtx_yolo_seg_postprocess_enqueue")
    return rows_out, canvases_out


def yolo_seg_launch_caps(image_sizes: Sequence[tuple[int, int]], *, net_w: int = 640, net_h: int = 640) -> tuple[int, ...]:
    """The shared memory yolo_seg_postprocess's canvas launches would use for frames of image_sizes[b] = (img_w, img_h), from
    the host alone: (M rows, low-resolution rows, M columns, low-resolution columns, dynamic shared-memory bytes), each the
    largest over the call's launches.  Raises TrtxError (UNSUPPORTED) where the enqueue would refuse these frames."""
    descs, _ = _frames(image_sizes, None, 0, None, False)
    q = L.MaskParams(L.YOLO_V8, net_w, net_h, net_w // 4, net_h // 4, 32, 39, 7, 1)
    caps = (C.c_int32 * 5)()
    L.check(L.load().trtx_yolo_seg_launch_caps(C.byref(q), descs, len(image_sizes), caps), "trtx_yolo_seg_launch_caps")
    return tuple(caps)


def yolo_pose_obb_postprocess(dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *, task: int, max_rows: int,
                              row_floats: int | None = None, extra_offset: int | None = None, num_kpts: int = 17,
                              net_w: int = 640, net_h: int = 640, rows_out: torch.Tensor | None = None,
                              stream=None) -> torch.Tensor:
    """GPU drop-in for the pose and oriented-box models' geometry after NMS: get_rect_adapt_landmark of
    draw_bbox_keypoints_line (task TASK_POSE, yolov8/src/postprocess.cpp:173-205) or get_corner of draw_bbox_obb (task
    TASK_OBB, :474-507; yolo11-obb: net_w = net_h = 1024) for a batch of frames of any sizes.
    dets [B, 1 + max_rows*row_floats]: count, then (box4, conf, class, keep, extras...) rows -- the compact NMS output (pose:
    extra_floats 51, row_floats 58; OBB: batch_nms_obb, row_floats 8); only rows with (int)keep == 1 are used.
    Task TASK_OBB_NMS_FREE: dets is yolo26-obb's NMS-free plugin output (YoloLayerPlugin26 with is_obb, row_floats 90, the
    angle last; net_w = net_h = 1024) and every row is used, as yolo26's batch_decode_obb + draw_bbox_obb do.
    extra_offset defaults to 7 (the first keypoint, or the angle of a compact OBB row), and to row_floats - 1 for
    TASK_OBB_NMS_FREE.
    image_sizes[b] = (img_w, img_h) of frame b -> rows [B, 1 + max_rows*F] fp32: the kept count, then per kept row (input
    order) pose (x, y, w, h, conf, class, kx, ky, kc, ...), F = 6 + 3*num_kpts, or OBB (x0, y0, ..., x3, y3, conf, class),
    F = 10; rows past the count are zero.  One launch per 64 frames, no workspace."""
    lib = L.load()
    B = len(image_sizes)
    if row_floats is None:
        row_floats = {L.TASK_POSE: 7 + 3 * num_kpts, L.TASK_OBB_NMS_FREE: YoloLayerPlugin26.DET_FLOATS}.get(task, 8)
    if extra_offset is None:
        extra_offset = row_floats - 1 if task == L.TASK_OBB_NMS_FREE else 7
    if dets.dim() != 2 or dets.shape[0] != B or dets.shape[1] < 1 + max_rows * row_floats:
        raise ValueError(f"dets must be [{B}, >= {1 + max_rows * row_floats}]")
    _f32_rows(dets)
    F = 6 + 3 * num_kpts if task == L.TASK_POSE else 10
    q = L.PoseObbParams(task, net_w, net_h, row_floats, extra_offset, num_kpts)
    rows_out = _out_tensor(rows_out, (B, 1 + max_rows * F), torch.float32, dets.device,
                           f"rows_out must be contiguous float32 [{B}, {1 + max_rows * F}]")
    L.check(lib.trtx_yolo_pose_obb_postprocess_enqueue(C.byref(q), _frame_wh(image_sizes), B, _ptr(dets), max_rows,
                                                       _ptr(rows_out), _stream(stream)), "trtx_yolo_pose_obb_postprocess_enqueue")
    return rows_out


def yolo_topk_postprocess(dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *, max_rows: int,
                          conf_thresh: float = 0.5, row_floats: int = 6, variant: int = L.YOLO_V8, net_w: int = 640,
                          net_h: int = 640, rows_out: torch.Tensor | None = None, stream=None) -> torch.Tensor:
    """GPU drop-in for yolov10's host post-process: batch_topk / get_topk (yolov10/src/postprocess.cpp:35-52: every plugin row
    with !(conf <= conf_thresh), a NaN conf included, in plugin order, no NMS) and draw_bbox's get_rect (yolov8's, clamped:
    variant YOLO_V8) for a batch of frames of any sizes.  dets [B, 1 + max_rows*row_floats]: the YoloLayerPluginV10 output
    (row_floats 6).  image_sizes[b] = (img_w, img_h) -> rows [B, 1 + max_rows*6] fp32: the used count, then (x, y, w, h,
    conf, class) per used row; rows past the count are zero.  One launch per 64 frames, no workspace."""
    lib = L.load()
    B = len(image_sizes)
    if dets.dim() != 2 or dets.shape[0] != B or dets.shape[1] < 1 + max_rows * row_floats:
        raise ValueError(f"dets must be [{B}, >= {1 + max_rows * row_floats}]")
    _f32_rows(dets)
    q = L.YoloTopkParams(variant, net_w, net_h, row_floats, conf_thresh)
    rows_out = _out_tensor(rows_out, (B, 1 + max_rows * 6), torch.float32, dets.device,
                           f"rows_out must be contiguous float32 [{B}, {1 + max_rows * 6}]")
    L.check(lib.trtx_yolo_topk_postprocess_enqueue(C.byref(q), _frame_wh(image_sizes), B, _ptr(dets), max_rows, _ptr(rows_out),
                                                   _stream(stream)), "trtx_yolo_topk_postprocess_enqueue")
    return rows_out


def retina_postprocess(dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *, variant: int, max_rows: int,
                       conf_thresh: float, in_w: int, in_h: int, row_floats: int | None = None, lmk_offset: int = 7,
                       rows_out: torch.Tensor | None = None, stream=None) -> torch.Tensor:
    """GPU drop-in for RetinaFace's last host stage after NMS: retinaface/retina_r50.cpp:373-388 (skip a face with
    class_confidence < CONF_THRESH, then get_rect_adapt_landmark; in_w x in_h = decodeplugin::INPUT_W x INPUT_H) and
    retinafaceAntiCov/retinafaceAntiCov.cpp:540-552 (variant RETINA_ANTICOV, no threshold: conf_thresh = -math.inf, 640 x 640)
    for a batch of frames of any sizes.
    dets [B, 1 + max_rows*row_floats]: count, then (x1, y1, x2, y2, conf, class, keep, landmarks[, mask_conf]) rows -- the
    output of batch_nms(..., box_format=BOX_RETINA, extra_floats=10 (AntiCov 11), extra_offset=5); row_floats defaults to
    17 (AntiCov 18).  Rows with (int)keep == 1 and !(conf < conf_thresh) are used (a NaN conf is kept); conf_thresh is the
    reference's double literal, passed to the library as the smallest float >= it, which selects the same faces.
    image_sizes[b] = (img_w, img_h) of frame b -> rows [B, 1 + max_rows*F] fp32, F = 15 (AntiCov 16): the used count, then
    per used row (input order) (x, y, w, h, conf, lx0, ly0, ..., lx4, ly4[, mask_conf]) = retina_get_rect_adapt_landmark;
    rows past the count are zero.  One launch per 64 frames, no workspace."""
    lib = L.load()
    B = len(image_sizes)
    extras = 11 if variant == L.RETINA_ANTICOV else 10
    if row_floats is None:
        row_floats = 7 + extras
    if dets.dim() != 2 or tuple(dets.shape) != (B, 1 + max_rows * row_floats):
        raise ValueError(f"dets must be [{B}, {1 + max_rows * row_floats}]")
    _f32_rows(dets)
    F = 5 + extras
    q = L.FacePostParams(variant, in_w, in_h, row_floats, lmk_offset, float_ge_threshold(conf_thresh))
    rows_out = _out_tensor(rows_out, (B, 1 + max_rows * F), torch.float32, dets.device,
                           f"rows_out must be contiguous float32 [{B}, {1 + max_rows * F}]")
    L.check(lib.trtx_retina_postprocess_enqueue(C.byref(q), _frame_wh(image_sizes), B, _ptr(dets), max_rows, _ptr(rows_out),
                                                _stream(stream)), "trtx_retina_postprocess_enqueue")
    return rows_out


class FusedYoloDecodeNms:
    """YoloLayer inputs -> compact detections in two launches (scan + NMS), no plugin-format round trip.
    Owns its workspace/output buffers (allocated once; enqueue itself allocates nothing)."""

    def __init__(self, plugin, max_batch: int, conf_thresh=0.5, nms_thresh=0.45, max_det=None, mode=L.NMS_GREEDY,
                 device="cuda", return_index=True, box_format=None):
        """box_format: the NMS box format (e.g. BOX_V9 for yolov9); by default the one the decode variant's rows have."""
        self.plugin = plugin
        self.max_batch = max_batch
        v5 = plugin.params.variant in (L.YOLO_V5, L.YOLO_V3, L.YOLO_V3_NET, L.YOLO_V4, L.YOLO_V4_CSP)  # rows are cx, cy, w, h
        if box_format is None:
            box_format = L.BOX_CXCYWH if v5 else L.BOX_LTRB
        self.max_det = max_det or plugin.mMaxOutObject
        self.q = nms_params(box_format, mode, conf_thresh, nms_thresh, self.max_det, True)
        self._lib = L.load()
        self.ws_bytes = plugin.getWorkspaceSize(max_batch)
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=device)
        self.out = torch.empty((max_batch, 1 + self.max_det * 7), dtype=torch.float32, device=device)
        self.idx = torch.empty((max_batch, self.max_det), dtype=torch.int32, device=device) if return_index else None

    def enqueue(self, batch: int, inputs, stream=None, out=None, idx=None, gather=None):
        """gather: an L.Gather descriptor (pipeline.PeerGather.desc) -> the NMS kernel also stores its rows into every
        rank's gathered buffer (trtx_yolo_decode_nms_gather_enqueue)."""
        ptrs = L.ptr_array([_ptr(t) for t in inputs])
        out = self.out if out is None else out
        idx = self.idx if idx is None else idx
        if gather is not None:
            L.check(self._lib.trtx_yolo_decode_nms_gather_enqueue(C.byref(self.plugin.params), C.byref(self.q), int(batch), ptrs,
                                                                  _ptr(out), _ptr(idx) if idx is not None else None, _ptr(self.ws),
                                                                  self.ws_bytes, C.byref(gather), _stream(stream)),
                    "trtx_yolo_decode_nms_gather_enqueue")
            return out[:batch], (idx[:batch] if idx is not None else None)
        L.check(self._lib.trtx_yolo_decode_nms_enqueue(C.byref(self.plugin.params), C.byref(self.q), int(batch), ptrs,
                                                       _ptr(out), _ptr(idx) if idx is not None else None,
                                                       _ptr(self.ws), self.ws_bytes, _stream(stream)),
                "trtx_yolo_decode_nms_enqueue")
        return out[:batch], (idx[:batch] if idx is not None else None)

    def enqueue_scan(self, batch: int, inputs, stream=None) -> None:
        """Split form, first half: the HBM-bound scan kernel only."""
        ptrs = L.ptr_array([_ptr(t) for t in inputs])
        L.check(self._lib.trtx_yolo_scan_enqueue(C.byref(self.plugin.params), int(batch), ptrs, _ptr(self.ws),
                                                 self.ws_bytes, _stream(stream)), "trtx_yolo_scan_enqueue")

    def enqueue_nms(self, batch: int, inputs, stream=None, out=None):
        """Split form, second half: NMS over the tiles left by enqueue_scan (out: another [max_batch, 1 + max_det*7] buffer,
        e.g. the second of a double buffer whose first half is still being gathered)."""
        ptrs = L.ptr_array([_ptr(t) for t in inputs])
        out = self.out if out is None else out
        L.check(self._lib.trtx_yolo_nms_after_scan_enqueue(C.byref(self.plugin.params), C.byref(self.q), int(batch), ptrs,
                                                           _ptr(out), _ptr(self.idx) if self.idx is not None else None,
                                                           _ptr(self.ws), self.ws_bytes, _stream(stream)),
                "trtx_yolo_nms_after_scan_enqueue")
        return out[:batch], (self.idx[:batch] if self.idx is not None else None)


# --------------------------------------------------------------------------------------------------
# Decode_TRT (RetinaFace)
# --------------------------------------------------------------------------------------------------
class DecodePlugin:
    PLUGIN_TYPE = "Decode_TRT"
    PLUGIN_VERSION = "1"

    def __init__(self, input_h: int = 480, input_w: int = 640, anticov: bool = False):
        """anticov=True: the Decode_TRT of retinafaceAntiCov/decode.cu (38-channel inputs, 16-float rows, 640x640 there)."""
        self._lib = L.load()
        p = L.RetinaParams()
        p.in_h, p.in_w = int(input_h), int(input_w)
        p.gate = float_le_threshold(0.02)  # `conf2 <= 0.02` with a double literal (decode.cu:131)
        p.variant = L.RETINA_ANTICOV if anticov else L.RETINA_FACE
        self.params = p
        self.det_floats = 16 if anticov else 15
        self.total_priors = int(self._lib.trtx_retina_total_priors(C.byref(p)))

    def getNbOutputs(self) -> int:
        return 1

    def output_elems(self) -> int:
        return 1 + self.total_priors * self.det_floats

    def getOutputDimensions(self, index=0, inputs=None, nbInputDims=0):
        return (self.output_elems(), 1, 1)  # decode.cu:33-41

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return int(self._lib.trtx_retina_workspace_size(C.byref(self.params), int(maxBatchSize)))

    def enqueue(self, batchSize: int, inputs, outputs, workspace, stream=None) -> int:
        """The heads may be torch.float32 (the reference's mode) or torch.float16, all three alike; the rows are fp32."""
        p = L.RetinaParams.from_buffer_copy(self.params)  # per-call copy: enqueue never mutates the plugin
        p.in_dtype = _elem_dtype(inputs, "Decode_TRT inputs")
        _elem_dtype(outputs[:1], "Decode_TRT output", only=L.F32)
        ptrs = L.ptr_array([_ptr(t) for t in inputs])
        return int(self._lib.trtx_retina_decode_enqueue(C.byref(p), int(batchSize), ptrs, _ptr(outputs[0]),
                                                        _ptr(workspace), _nbytes(workspace), _stream(stream)))

    def getPluginType(self) -> str:
        return self.PLUGIN_TYPE

    def getPluginVersion(self) -> str:
        return self.PLUGIN_VERSION

    def clone(self) -> "DecodePlugin":
        return DecodePlugin(self.params.in_h, self.params.in_w, self.params.variant == L.RETINA_ANTICOV)

    def serialize(self) -> bytes:  # the reference serializes nothing (decode.cu:23-31); the runtime size is new state
        return struct.pack("<ii", self.params.in_h, self.params.in_w)

    @classmethod
    def deserialize(cls, data: bytes) -> "DecodePlugin":
        if len(data) == 0:
            return cls()
        h, w = struct.unpack("<ii", data)
        return cls(h, w)


# --------------------------------------------------------------------------------------------------
# Faster R-CNN plugins (rcnn/*Plugin.h): "null workspace returns the size" idiom kept
# --------------------------------------------------------------------------------------------------
def _rc64(rc: int, what: str) -> int:
    if rc < 0:
        L.check(-rc, what)
    return rc


def _status(rc: int) -> int:
    """enqueue()'s return value from a call that returns -error or a non-negative count: the error code, or 0."""
    return int(-rc if rc < 0 else 0)


class RpnDecodePlugin:
    def __init__(self, top_n: int, anchors: Sequence[float], stride: float, image_height: int, image_width: int,
                 height: int = 0, width: int = 0):
        self._lib = L.load()
        self._top_n, self._anchors, self._stride = int(top_n), [float(a) for a in anchors], float(stride)
        self._image_height, self._image_width = int(image_height), int(image_width)
        self._height, self._width = int(height), int(width)
        self._anc = (C.c_float * len(self._anchors))(*self._anchors)

    def configurePlugin(self, inputDims):  # RpnDecodePlugin.h:148-157: height/width from the scores tensor dims
        self._height, self._width = int(inputDims[0][1]), int(inputDims[0][2])

    def getNbOutputs(self) -> int:
        return 2

    def getOutputDimensions(self, index):
        return (self._top_n, 4 if index == 1 else 1)

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return _rc64(self._lib.trtx_rpn_decode(maxBatchSize, None, None, None, None, self._height, self._width,
                                               self._image_height, self._image_width, self._stride, self._anc,
                                               len(self._anchors) // 4, self._top_n, None, 0, None), "trtx_rpn_decode(size)")

    def enqueue(self, batchSize, inputs, outputs, workspace, stream=None) -> int:
        """Scores and deltas share one dtype, torch.float32 or torch.float16 (the result is then the fp32 result of the
        widened tensors, bit for bit); the output scores and boxes are torch.float32 in both modes."""
        dt = _elem_dtype(inputs[:2], "RpnDecode scores and deltas")
        _elem_dtype(outputs[:2], "RpnDecode outputs", only=L.F32)
        rc = self._lib.trtx_rpn_decode_typed(dt, batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(outputs[0]), _ptr(outputs[1]),
                                             self._height, self._width, self._image_height, self._image_width, self._stride,
                                             self._anc, len(self._anchors) // 4, self._top_n, _ptr(workspace), _nbytes(workspace),
                                             _stream(stream))
        return _status(rc)


class RpnNmsPlugin:
    def __init__(self, nms_thresh: float, post_nms_topk: int, pre_nms_topk: int = 1):
        self._lib = L.load()
        self._nms_thresh, self._post_nms_topk, self._pre_nms_topk = float(nms_thresh), int(post_nms_topk), int(pre_nms_topk)

    def configurePlugin(self, inputDims):
        self._pre_nms_topk = int(inputDims[0][0])

    def getNbOutputs(self) -> int:
        return 1

    def getOutputDimensions(self, index=0):
        return (self._post_nms_topk, 4)

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return _rc64(self._lib.trtx_rpn_nms(maxBatchSize, None, None, None, self._pre_nms_topk, self._post_nms_topk,
                                            self._nms_thresh, None, 0, None), "trtx_rpn_nms(size)")

    def enqueue(self, batchSize, inputs, outputs, workspace, stream=None) -> int:
        rc = self._lib.trtx_rpn_nms(batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(outputs[0]), self._pre_nms_topk,
                                    self._post_nms_topk, self._nms_thresh, _ptr(workspace), _nbytes(workspace), _stream(stream))
        return _status(rc)


class PredictorDecodePlugin:
    def __init__(self, num_boxes: int, image_height: int, image_width: int, bbox_reg_weights: Sequence[float],
                 num_classes: int = 0):
        self._lib = L.load()
        self._num_boxes, self._num_classes = int(num_boxes), int(num_classes)
        self._image_height, self._image_width = int(image_height), int(image_width)
        self._w = (C.c_float * 4)(*[float(x) for x in bbox_reg_weights])

    def configurePlugin(self, inputDims):
        self._num_classes = int(inputDims[0][1])

    def getNbOutputs(self) -> int:
        return 3

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return _rc64(self._lib.trtx_predictor_decode(maxBatchSize, None, None, None, None, None, None, self._num_boxes,
                                                     self._num_classes, self._image_height, self._image_width, self._w,
                                                     None, 0, None), "trtx_predictor_decode(size)")

    def enqueue(self, batchSize, inputs, outputs, workspace, stream=None) -> int:
        """Scores and deltas share one dtype, torch.float32 or torch.float16 (the result is then the fp32 result of the
        widened tensors, bit for bit); the proposals and the output scores, boxes and classes are torch.float32 in both modes."""
        dt = _elem_dtype(inputs[:2], "PredictorDecode scores and deltas")
        _elem_dtype(inputs[2:3], "PredictorDecode proposals", only=L.F32)
        _elem_dtype(outputs[:3], "PredictorDecode outputs", only=L.F32)
        rc = self._lib.trtx_predictor_decode_typed(dt, batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(inputs[2]),
                                                   _ptr(outputs[0]), _ptr(outputs[1]), _ptr(outputs[2]), self._num_boxes,
                                                   self._num_classes, self._image_height, self._image_width, self._w,
                                                   _ptr(workspace), _nbytes(workspace), _stream(stream))
        return _status(rc)


class BatchedNmsPlugin:
    def __init__(self, nms_method: int, nms_thresh: float, detections_per_im: int, count: int = 1):
        self._lib = L.load()
        self._nms_method, self._nms_thresh = int(nms_method), float(nms_thresh)
        self._detections_per_im, self._count = int(detections_per_im), int(count)

    def configurePlugin(self, inputDims):
        self._count = int(inputDims[0][0])

    def getNbOutputs(self) -> int:
        return 3

    def getOutputDimensions(self, index):
        return (self._detections_per_im, 4 if index == 1 else 1)

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return _rc64(self._lib.trtx_batched_nms(self._nms_method, maxBatchSize, None, None, None, None, None, None,
                                                self._count, self._detections_per_im, self._nms_thresh, None, 0, None),
                     "trtx_batched_nms(size)")

    def enqueue(self, batchSize, inputs, outputs, workspace, stream=None) -> int:
        rc = self._lib.trtx_batched_nms(self._nms_method, batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(inputs[2]),
                                        _ptr(outputs[0]), _ptr(outputs[1]), _ptr(outputs[2]), self._count,
                                        self._detections_per_im, self._nms_thresh, _ptr(workspace), _nbytes(workspace),
                                        _stream(stream))
        return _status(rc)


# --------------------------------------------------------------------------------------------------
# Pre-process (preprocess.h)
# --------------------------------------------------------------------------------------------------
class Int8CalibratorBatcher:
    """The host pre-process of Int8EntropyCalibrator2::getBatch (yolov8/src/calibrator.cpp:33-52): every image goes through
    preprocess_img (letterbox, cv::resize INTER_LINEAR) and cv::dnn::blobFromImages(1 / 255.0, swapRB); `get_batch(images)` returns
    the [B, 3, input_h, input_w] fp32 batch the calibrator copies to the device.  HOST code (trtx_calib_letterbox_host), as in the
    reference; bit-identical to OpenCV 4.13 (tests/test_calibrator_cpu.py)."""

    def __init__(self, batchsize: int, input_w: int, input_h: int):
        self._lib = L.load()
        self.batchsize, self.input_w, self.input_h = int(batchsize), int(input_w), int(input_h)
        self.input_count = 3 * self.input_w * self.input_h * self.batchsize     # calibrator.cpp:20

    def getBatchSize(self) -> int:
        return self.batchsize

    def get_batch(self, images) -> "np.ndarray":
        import numpy as np

        if len(images) != self.batchsize:
            raise L.TrtxError(f"Int8CalibratorBatcher: {len(images)} images for a batch of {self.batchsize}")
        out = np.empty((self.batchsize, 3, self.input_h, self.input_w), np.float32)
        for i, img in enumerate(images):
            img = np.ascontiguousarray(img, np.uint8)
            h, w = img.shape[:2]
            L.check(self._lib.trtx_calib_letterbox_host(img.ctypes.data_as(C.c_void_p), w, h, img.strides[0], self.input_w, self.input_h,
                                                        out[i].ctypes.data_as(C.c_void_p)), "trtx_calib_letterbox_host")
        return out


class RoiAlignPlugin:
    """rcnn/RoiAlignPlugin.h:27-170 (plugin "RoiAlign"): inputs proposals [B,N,4], features [B,C,H,W] ->
    [B, N, C, P, P].  No workspace, no device synchronisation (the reference syncs after every image)."""

    def __init__(self, pooler_resolution: int, spatial_scale: float, sampling_ratio: int, num_proposals: int,
                 out_channels: int, feature_h: int = 0, feature_w: int = 0):
        self._lib = L.load()
        self._pooler_resolution, self._spatial_scale = int(pooler_resolution), float(spatial_scale)
        self._sampling_ratio, self._num_proposals, self._out_channels = int(sampling_ratio), int(num_proposals), int(out_channels)
        self._feature_h, self._feature_w = int(feature_h), int(feature_w)

    def configurePlugin(self, inputDims):  # RoiAlignPlugin.h:140-153
        self._feature_h, self._feature_w = int(inputDims[1][1]), int(inputDims[1][2])

    def getNbOutputs(self) -> int:
        return 1

    def getOutputDimensions(self, index=0):
        return (self._num_proposals, self._out_channels, self._pooler_resolution, self._pooler_resolution)

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return 0

    def enqueue(self, batchSize, inputs, outputs, workspace=None, stream=None) -> int:
        """Features and output share one dtype, torch.float32 or torch.float16 (the bins are then the fp32 bins of the widened
        features, rounded once); the proposals are torch.float32 in both modes."""
        _elem_dtype(inputs[:1], "RoiAlign proposals", only=L.F32)
        dt = _elem_dtype([inputs[1], outputs[0]], "RoiAlign features and output")
        return int(self._lib.trtx_roi_align_typed(dt, batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(outputs[0]),
                                                  self._pooler_resolution, self._spatial_scale, self._sampling_ratio,
                                                  self._num_proposals, self._out_channels, self._feature_h, self._feature_w,
                                                  _stream(stream)))


class MaskRcnnInferencePlugin:
    """rcnn/MaskRcnnInferencePlugin.h:27-140 (plugin "MaskRcnnInference"): indices [B,D] (float class ids),
    masks [B,D,num_classes,S,S] -> [B,D,1,S,S] = sigmoid of the predicted class' mask."""

    def __init__(self, detections_per_im: int, output_size: int, num_classes: int = 1):
        self._lib = L.load()
        self._detections_per_im, self._output_size, self._num_classes = int(detections_per_im), int(output_size), int(num_classes)

    def configurePlugin(self, inputDims):  # MaskRcnnInferencePlugin.h:109-120
        self._num_classes = int(inputDims[1][1])

    def getNbOutputs(self) -> int:
        return 1

    def getOutputDimensions(self, index=0):
        return (self._detections_per_im, 1, self._output_size, self._output_size)

    def getWorkspaceSize(self, maxBatchSize: int) -> int:
        return 0

    def enqueue(self, batchSize, inputs, outputs, workspace=None, stream=None) -> int:
        """The masks may be torch.float32 or torch.float16; indices and output are torch.float32 in both modes."""
        _elem_dtype([inputs[0], outputs[0]], "MaskRcnnInference indices and output", only=L.F32)
        dt = _elem_dtype(inputs[1:2], "MaskRcnnInference masks")
        return int(self._lib.trtx_mask_rcnn_inference_typed(dt, batchSize, _ptr(inputs[0]), _ptr(inputs[1]), _ptr(outputs[0]),
                                                            self._detections_per_im, self._output_size, self._num_classes,
                                                            _stream(stream)))


def _image_descs(images: Sequence[torch.Tensor]):
    """trtx_image_desc array of u8 HWC BGR device frames [h, w, 3]: rows may be pitched, pixels may not."""
    descs = (L.ImageDesc * len(images))()
    for i, im in enumerate(images):
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or im.stride(2) != 1 or im.stride(1) != 3:
            raise L.TrtxError("images must be u8 HWC BGR with packed pixels")
        descs[i].data_dev = im.data_ptr()
        descs[i].height, descs[i].width = int(im.shape[0]), int(im.shape[1])
        descs[i].pitch = int(im.stride(0))
    return descs


def _letterbox_dst(dst: torch.Tensor, n: int, dst_width: int, dst_height: int) -> int:
    """TRTX_F32 / TRTX_F16 of the letterbox output dst, which must be a float32 or float16 tensor [n, 3, dst_h, dst_w]:
    TrtxError for another dtype, ValueError for another shape, both before the library is called."""
    dt = _elem_dtype([dst], "letterbox dst")
    _out_tensor(dst, (n, 3, int(dst_height), int(dst_width)), dst.dtype, dst.device,
                f"dst must be float32 or float16 [{n}, 3, {dst_height}, {dst_width}]", contiguous=False)
    return dt


def cuda_batch_preprocess(img_batch: Sequence[torch.Tensor], dst: torch.Tensor, dst_width: int, dst_height: int,
                          stream=None) -> None:
    """Drop-in for cuda_batch_preprocess (yolov8/src/preprocess.cu:119-127) with DEVICE images:
    img_batch[i] is a u8 HWC BGR cuda tensor [h, w, 3] (row-contiguous); dst is [B, 3, dst_h, dst_w] fp32/fp16.
    One launch for the whole batch, no synchronisation."""
    lib = L.load()
    descs = _image_descs(img_batch)
    dt = _letterbox_dst(dst, len(img_batch), dst_width, dst_height)
    L.check(lib.trtx_preprocess_batch_enqueue(descs, len(img_batch), _ptr(dst), dst_width, dst_height, dt, _stream(stream)),
            "trtx_preprocess_batch_enqueue")


class PreprocessPlan:
    """cuda_batch_preprocess with the descriptors prepared once for persistent device frame buffers
    (the reference rebuilds nothing either: its staging buffers are allocated in cuda_preprocess_init,
    preprocess.cu:129-134).  enqueue() is a single C call -> a single kernel launch."""

    def __init__(self, img_batch: Sequence[torch.Tensor], dst: torch.Tensor, dst_width: int, dst_height: int):
        self._lib = L.load()
        self.n = len(img_batch)
        self.descs = _image_descs(img_batch)
        self._keep = list(img_batch)
        self.dst, self.dw, self.dh = dst, int(dst_width), int(dst_height)
        self.dt = _letterbox_dst(dst, self.n, self.dw, self.dh)

    def enqueue(self, stream=None) -> None:
        L.check(self._lib.trtx_preprocess_batch_enqueue(self.descs, self.n, _ptr(self.dst), self.dw, self.dh, self.dt,
                                                        _stream(stream)), "trtx_preprocess_batch_enqueue")


def get_rect(img_w: int, img_h: int, bbox, net_w: int = 640, net_h: int = 640, variant: int = L.YOLO_V8):
    """get_rect(img, bbox) of yolov8/src/postprocess.cpp:6-36 (variant YOLO_V5: yolov5/src/postprocess.cpp:4-29; YOLO_V3:
    the truncating get_rect of yolov3, yolov4, scaled-yolov4 and yolov3-tiny; RECT_YOLOV3_SPP: yolov3-spp's, with
    net_w = net_h = MAX_INPUT_SIZE) -> (x, y, width, height) in the original image, (0, 0, 0, 0) where the reference's
    conversions are undefined."""
    lib = L.load()
    b = (C.c_float * 4)(*[float(v) for v in bbox])
    r = (C.c_int * 4)()
    L.check(lib.trtx_get_rect(variant, net_w, net_h, img_w, img_h, b, r), "trtx_get_rect")
    return tuple(r)


def get_rect_adapt_landmark(img_w: int, img_h: int, bbox, lmk, net_w: int = 640, net_h: int = 640):
    """get_rect_adapt_landmark(img, bbox, lmk) of yolov8/src/postprocess.cpp:38-69 -> ((x, y, w, h), mapped keypoints)."""
    lib = L.load()
    b = (C.c_float * 4)(*[float(v) for v in bbox])
    k = (C.c_float * len(lmk))(*[float(v) for v in lmk])
    r = (C.c_int * 4)()
    L.check(lib.trtx_get_rect_adapt_landmark(net_w, net_h, img_w, img_h, b, k, len(lmk) // 3, r), "trtx_get_rect_adapt_landmark")
    return tuple(r), list(k)


def get_corner(img_w: int, img_h: int, cxcywh, angle: float, net_w: int = 640, net_h: int = 640):
    """get_corner(img, box) of yolov8/src/postprocess.cpp:395-472 (net_w = net_h = 1024: yolo11's get_rect_obb) ->
    ((x0, y0), (x1, y1), (x2, y2), (x3, y3)) in the original image."""
    b = (C.c_float * 4)(*[float(v) for v in cxcywh])
    c = (C.c_int * 8)()
    L.check(L.load().trtx_get_corner(net_w, net_h, img_w, img_h, b, float(angle), c), "trtx_get_corner")
    return tuple((c[2 * k], c[2 * k + 1]) for k in range(4))


def scale_mask(masks: torch.Tensor, img_w: int, img_h: int, out=None, stream=None) -> torch.Tensor:
    """scale_mask(mask, img) of yolov8/src/postprocess.cpp:207-226 for a stack of device masks [n, net_h, net_w] fp32 ->
    [n, img_h, img_w]: the letterboxed region, bilinearly resized (cv::resize) to the original image."""
    lib = L.load()
    n, nh, nw = masks.shape
    if out is None:
        out = torch.empty((n, img_h, img_w), dtype=torch.float32, device=masks.device)
    L.check(lib.trtx_scale_mask_enqueue(_ptr(masks), n, nw, nh, img_w, img_h, _ptr(out), _stream(stream)), "trtx_scale_mask_enqueue")
    return out


def rcnn_letterbox_pads(img_w: int, img_h: int, net_w: int, net_h: int):
    """The pads preprocessImg (rcnn/common.hpp:79-102) puts around an img_w x img_h image in the net_w x net_h model input:
    (left, right, top, bottom)."""
    p = (C.c_int * 4)()
    L.check(L.load().trtx_rcnn_letterbox_pads(img_w, img_h, net_w, net_h, p), "trtx_rcnn_letterbox_pads")
    return tuple(p)


def rcnn_preprocess(images: Sequence[torch.Tensor], net_w: int, net_h: int, out: torch.Tensor | None = None,
                    stream=None) -> torch.Tensor:
    """GPU drop-in for the pre-process of rcnn/rcnn.cpp:497-506 (preprocessImg, rcnn/common.hpp:79-110, then the widening
    of every byte to float) for a batch of device frames: images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed
    pixels (rows may be pitched, sizes may differ) -> [B, net_h, net_w, 3] float32 BGR, 0..255, 128 around the resized
    image: the engine input.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, net_h, net_w, 3), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, {net_h}, {net_w}, 3]", contiguous=False)
    L.check(lib.trtx_rcnn_preprocess_enqueue(descs, n, net_w, net_h, _ptr(out), _stream(stream)), "trtx_rcnn_preprocess_enqueue")
    return out


def cls_preprocess(images: Sequence[torch.Tensor], variant: int, net_w: int, net_h: int, out: torch.Tensor | None = None,
                   stream=None) -> torch.Tensor:
    """GPU drop-in for batch_preprocess of the YOLO cls drivers for a batch of device frames: images[i] is a u8 HWC BGR cuda
    tensor [h, w, 3] with packed pixels (rows may be pitched, sizes may differ) -> [B, 3, net_h, net_w] float32 planar RGB, the
    engine input.  variant _lib.YOLO_V8 (yolov8, yolo11, yolo26): centre square crop, resize, / 255; _lib.YOLO_V5 (yolov5): the
    letterbox on a 128-grey canvas, ImageNet mean / std.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_cls_preprocess_enqueue(variant, descs, n, net_w, net_h, _ptr(out), _stream(stream)),
            "trtx_cls_preprocess_enqueue")
    return out


YOLOP_NET = (640, 384)  # Yolo::INPUT_W, INPUT_H (yolop/yololayer.h)
YOLOP_MAP = (640, 360)  # Yolo::IMG_W, IMG_H: the drivable-area and lane maps


def yolop_preprocess(images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net_w: int = YOLOP_NET[0],
                     net_h: int = YOLOP_NET[1], stream=None) -> torch.Tensor:
    """GPU drop-in for YOLOP's preprocess_img (yolop/utils.h:11-36) and the driver's plane copy (yolop/yolop.cpp:110-127)
    for a batch of device frames: images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched,
    sizes may differ) -> [B, 3, net_h, net_w] float32 planes in B, G, R order, the engine input: the letterbox on a 114-grey
    canvas, / 255, minus the ImageNet mean, over its std.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_yolop_preprocess_enqueue(descs, n, net_w, net_h, _ptr(out), _stream(stream)), "trtx_yolop_preprocess_enqueue")
    return out


def yolop_get_rect(img_w: int, img_h: int, bbox, net_w: int = YOLOP_NET[0], net_h: int = YOLOP_NET[1]):
    """get_rect(img, bbox) of yolop/common.hpp:13-37: bbox cx, cy, w, h in network pixels -> (x, y, w, h) in the frame."""
    b = (C.c_float * 4)(*[float(v) for v in bbox])
    r = (C.c_int * 4)()
    L.check(L.load().trtx_yolop_get_rect(net_w, net_h, img_w, img_h, b, r), "trtx_yolop_get_rect")
    return tuple(r)


def yolop_postprocess(dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *, max_rows: int,
                      seg: torch.Tensor | None = None, lane: torch.Tensor | None = None, labels: bool = True,
                      row_floats: int = 7, net_w: int = YOLOP_NET[0], net_h: int = YOLOP_NET[1],
                      rows_out: torch.Tensor | None = None, canvases_out: Sequence[torch.Tensor] | None = None, stream=None):
    """GPU drop-in for YOLOP's host stages after NMS: get_rect per box (yolop/common.hpp:13-37) and the per-pixel label loop
    over the drivable-area and lane maps (yolop/yolop.cpp:148-169), for a batch of frames of any sizes.
    dets [B, 1 + max_rows*row_floats]: count, then (cx, cy, w, h, conf, class, keep) rows -- batch_nms(..., box_format=
    BOX_CXCYWH, det_floats=6); seg, lane [B, map_h, map_w] int32: the engine's TopK index maps; image_sizes[b] = (img_w,
    img_h) of frame b -> (rows [B, 1 + max_rows*6] fp32: the count, then (x, y, w, h, conf, class), rows past the count zero;
    per-frame u8 canvases [img_h, img_w]: 2 on a lane, else 1 on the drivable area, else 0 -- or None with labels=False).
    `canvases_out[b]` may be any u8 cuda tensor [img_h, img_w] with contiguous rows (e.g. a view [:, :img_w] of a pitched
    buffer); bytes past img_w are not written.  Frame b reads maps b.  Two launches per 64 frames."""
    lib = L.load()
    B = len(image_sizes)
    if dets.dim() != 2 or tuple(dets.shape) != (B, 1 + max_rows * row_floats):
        raise ValueError(f"dets must be [{B}, {1 + max_rows * row_floats}]")
    _f32_rows(dets)
    rows_out = _out_tensor(rows_out, (B, 1 + max_rows * 6), torch.float32, dets.device,
                           f"rows_out must be contiguous float32 [{B}, {1 + max_rows * 6}]")
    map_w, map_h = YOLOP_MAP
    if labels:
        if seg is None or lane is None or seg.shape != lane.shape or seg.dim() != 3 or seg.shape[0] != B:
            raise ValueError(f"seg and lane must be int32 [{B}, map_h, map_w]")
        for t in (seg, lane):
            if t.dtype != torch.int32 or not t.is_contiguous():
                raise ValueError("seg and lane must be contiguous int32")
        map_h, map_w = int(seg.shape[1]), int(seg.shape[2])
        if canvases_out is None:
            canvases_out = [torch.zeros((h, w), dtype=torch.uint8, device=dets.device) for w, h in image_sizes]
        descs, canvases = _frames(image_sizes, [c.unsqueeze(0) for c in canvases_out], 1, dets.device, True)
        canvases_out = [c.squeeze(0) for c in canvases]
    else:
        descs, canvases_out = _frames(image_sizes, None, 1, dets.device, False)
    q = L.YolopPostParams(net_w, net_h, map_w, map_h, row_floats)
    L.check(lib.trtx_yolop_postprocess_enqueue(C.byref(q), descs, B, _ptr(dets), max_rows,
                                               _ptr(seg) if labels else None, _ptr(lane) if labels else None,
                                               _ptr(rows_out), _stream(stream)), "trtx_yolop_postprocess_enqueue")
    return rows_out, canvases_out


DETR_NET = (1066, 800)  # INPUT_W, INPUT_H (detr/detr.cpp:13-14)


def detr_preprocess(images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net_w: int = DETR_NET[0],
                    net_h: int = DETR_NET[1], stream=None) -> torch.Tensor:
    """GPU drop-in for DETR's preprocessImg (detr/common.hpp:81-89) and the driver's plane copy (detr/detr.cpp:754-767) for a
    batch of device frames: images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched, sizes
    may differ) -> [B, 3, net_h, net_w] float32 planes in R, G, B order, the engine input: the whole frame resized to the
    whole net, / 255, minus the ImageNet mean, over its std.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_detr_preprocess_enqueue(descs, n, net_w, net_h, _ptr(out), _stream(stream)), "trtx_detr_preprocess_enqueue")
    return out


def detr_get_rect(img_w: int, img_h: int, box):
    """The cv::Rect of detr/detr.cpp:795-803: box cx, cy, w, h (normalised) -> (x, y, w, h) in the img_w x img_h frame."""
    b = (C.c_float * 4)(*[float(v) for v in box])
    r = (C.c_int * 4)()
    L.check(L.load().trtx_detr_get_rect(img_w, img_h, b, r), "trtx_detr_get_rect")
    return tuple(r)


def detr_postprocess(scores: torch.Tensor, boxes: torch.Tensor, image_sizes: Sequence[tuple[int, int]], *,
                     score_thresh: float = 0.5, out: torch.Tensor | None = None, stream=None) -> torch.Tensor:
    """GPU drop-in for DETR's host loop after inference (detr/detr.cpp:777-806) for a batch of frames of any sizes.
    scores [B, Q, C] float32: the engine's softmax scores, class C - 1 the no-object class; boxes [B, Q, 4] float32: its
    (cx, cy, w, h), normalised; image_sizes[b] = (img_w, img_h) of frame b -> rows [B, 1 + Q*6] float32: the kept count, then
    per kept query in query order (x, y, w, h, score, class) -- the first maximum over the classes, kept when score >
    score_thresh (float) and the class is not C - 1, the rectangle as detr_get_rect -- rows past the count zero.  Frame b
    reads queries b.  One launch per 64 frames, no workspace."""
    lib = L.load()
    B = len(image_sizes)
    if scores.dim() != 3 or scores.shape[0] != B or tuple(boxes.shape) != (B, scores.shape[1], 4):
        raise ValueError(f"scores must be [{B}, Q, C] and boxes [{B}, Q, 4]")
    for t in (scores, boxes):
        if t.dtype != torch.float32:
            raise ValueError("scores and boxes must be float32")
    Q, Cn = int(scores.shape[1]), int(scores.shape[2])
    out = _out_tensor(out, (B, 1 + Q * 6), torch.float32, scores.device, f"out must be contiguous float32 [{B}, {1 + Q * 6}]")
    q = L.DetrPostParams(Q, Cn, score_thresh)
    L.check(lib.trtx_detr_postprocess_enqueue(C.byref(q), _frame_wh(image_sizes), B, _ptr(scores), _ptr(boxes), _ptr(out),
                                              _stream(stream)), "trtx_detr_postprocess_enqueue")
    return out


CENTERNET_NET, CENTERNET_DOWN = 512, 4  # centernet/sample/test.py: cv.resize(img, (512, 512)), `4*s`


def centernet_preprocess(images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net: int = CENTERNET_NET,
                         stream=None) -> torch.Tensor:
    """GPU drop-in for CenterNet's pre_process (centernet/sample/test.py:34-41) for a batch of device frames: images[i] is a
    u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched, sizes may differ) -> [B, 3, net, net] float32
    planes in B, G, R order, the engine input: the frame at the top-left of an L x L zero canvas (L = max(h, w, 3)), resized
    on float64 as cv.resize does, then ((v / 255.) - 0.5) / 0.5.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net, net), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net}, {net}]", contiguous=False)
    L.check(lib.trtx_centernet_preprocess_enqueue(descs, n, net, _ptr(out), _stream(stream)),
            "trtx_centernet_preprocess_enqueue")
    return out


def centernet_decode(heat: torch.Tensor, wh: torch.Tensor, reg: torch.Tensor, k: int = 100, *,
                     image_sizes: Sequence[tuple[int, int]] | None = None, score_thresh: float = 0.5,
                     net: int = CENTERNET_NET, down: int = CENTERNET_DOWN, workspace: torch.Tensor | None = None,
                     out: torch.Tensor | None = None, rows_out: torch.Tensor | None = None, stream=None):
    """GPU drop-in for ctdet_decode(hm, wh, reg, K=k) (centernet/sample/test.py:44-102) on the engine outputs heat
    [B, C, H, W], wh and reg [B, 2, H, W] float32 -> dets [B, k, 6] float32 (x1, y1, x2, y2, score, class) in map units:
    sigmoid, the 3 x 3 peak test, the k best cells of each image ordered NaN first, then by descending score, ties to the
    smaller flat index.  With image_sizes[b] = (img_w, img_h), also the driver loop (:126-132): rows [B, 1 + k*6] with the
    count of score > score_thresh, then those rows with the box times (float)(down * (L / net)), L = max(img_h, img_w, 3),
    zeros past the count -> (dets, rows).  Two launches, no synchronisation."""
    lib = L.load()
    if heat.dim() != 4:
        raise ValueError("heat must be [B, C, H, W]")
    B, Cn, H, W = (int(v) for v in heat.shape)
    for t, what in ((wh, "wh"), (reg, "reg")):
        if tuple(t.shape) != (B, 2, H, W):
            raise ValueError(f"{what} must be [{B}, 2, {H}, {W}]")
    for t in (heat, wh, reg):
        if t.dtype != torch.float32:
            raise ValueError("heat, wh and reg must be float32")
    q = L.CenternetParams(Cn, H, W, k, net, down, score_thresh)
    ws_bytes = int(lib.trtx_centernet_workspace_size(C.byref(q), B))
    if ws_bytes == 0:
        L.check(L.ERR_INVALID if B <= 0 or k <= 0 or k > H * W else L.ERR_UNSUPPORTED, "trtx_centernet_workspace_size")
    if workspace is None:
        workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=heat.device)
    out = _out_tensor(out, (B, k, 6), torch.float32, heat.device, f"out must be contiguous float32 [{B}, {k}, 6]")
    wh_arr = None
    if image_sizes is not None:
        if len(image_sizes) != B:
            raise ValueError(f"expected {B} image sizes")
        wh_arr = _frame_wh(image_sizes)
        rows_out = _out_tensor(rows_out, (B, 1 + k * 6), torch.float32, heat.device,
                               f"rows_out must be contiguous float32 [{B}, {1 + k * 6}]")
    L.check(lib.trtx_centernet_decode_enqueue(C.byref(q), B, _ptr(heat), _ptr(wh), _ptr(reg), _ptr(workspace),
                                              _nbytes(workspace), _ptr(out), wh_arr,
                                              _ptr(rows_out) if wh_arr is not None else None, _stream(stream)),
            "trtx_centernet_decode_enqueue")
    return (out, rows_out) if wh_arr is not None else out


UFLD_NET = (800, 288)  # INPUT_W, INPUT_H (ufld/lane_det.cpp:13-14)
UFLD_SHAPE = (101, 56, 4)  # OUTPUT_C, OUTPUT_H, OUTPUT_W
UFLD_COL_SAMPLE_W = 8
UFLD_TUSIMPLE_ROW_ANCHOR = tuple(range(64, 288, 4))  # tusimple_row_anchor (ufld/lane_det.cpp:358-363)
UFLD_VIS = (1280, 720)  # vis_w, vis_h: the driver's drawing frame


def ufld_preprocess(images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net_w: int = UFLD_NET[0],
                    net_h: int = UFLD_NET[1], stream=None) -> torch.Tensor:
    """GPU drop-in for UFLD's prepareImage (ufld/lane_det.cpp:194-221) for a batch of device frames: images[i] is a u8 HWC BGR
    cuda tensor [h, w, 3] with packed pixels (rows may be pitched, sizes may differ) -> [B, 3, net_h, net_w] float32 planes in
    R, G, B order, the engine input: the whole frame resized to the whole net, then fmaf(u * (1 / 255.), 1 / std, -mean / std)
    as OpenCV folds the driver's `(c - mean) / std`.  The frames are not written.  One launch per 64 images, no
    synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_ufld_preprocess_enqueue(descs, n, net_w, net_h, _ptr(out), _stream(stream)), "trtx_ufld_preprocess_enqueue")
    return out


def ufld_postprocess(prob: torch.Tensor, image_sizes: Sequence[tuple[int, int]] | None = None, *,
                     row_anchor: Sequence[int] = UFLD_TUSIMPLE_ROW_ANCHOR, col_sample_w: int = UFLD_COL_SAMPLE_W,
                     net_w: int = UFLD_NET[0], net_h: int = UFLD_NET[1], out: torch.Tensor | None = None,
                     stream=None) -> torch.Tensor:
    """GPU drop-in for UFLD's host stages after inference (ufld/lane_det.cpp:358-410) for a batch: prob [B, C, H, W] float32,
    the engine output (C = 101 cells, the last one "no lane"; H = 56 row anchors; W = 4 lanes); image_sizes[b] = (w, h) of the
    picture frame b's points are for (default: the driver's 1280 x 720 `vis` for every frame); row_anchor: H ints ->
    rows [B, 1 + H*W*3] float32: the point count, then (x, y, lane) per point in the driver's draw order (engine rows H - 1
    .. 0, lanes ascending), zeros past the count.  One launch per 64 frames, no workspace."""
    lib = L.load()
    if prob.dim() != 4 or prob.dtype != torch.float32:
        raise ValueError("prob must be float32 [B, C, H, W]")
    B, Cn, H, W = (int(v) for v in prob.shape)
    if image_sizes is None:
        image_sizes = [UFLD_VIS] * B
    if len(image_sizes) != B or len(row_anchor) != H:
        raise ValueError(f"expected {B} image sizes and {H} row anchors")
    out = _out_tensor(out, (B, 1 + H * W * 3), torch.float32, prob.device,
                      f"out must be contiguous float32 [{B}, {1 + H * W * 3}]")
    q = L.UfldPostParams(Cn, H, W, net_w, net_h, col_sample_w)
    anchors = (C.c_int32 * H)(*[int(v) for v in row_anchor])
    L.check(lib.trtx_ufld_postprocess_enqueue(C.byref(q), anchors, _frame_wh(image_sizes), B, _ptr(prob), _ptr(out),
                                              _stream(stream)), "trtx_ufld_postprocess_enqueue")
    return out


REFINEDET_NET = 320        # INPUT_W = INPUT_H (refinedet/configure.h)
REFINEDET_NUM_CLASSES = 25  # num_class, the background included
REFINEDET_TOP_K = 1000     # nms()'s top_k (refinedet/refinedet.cpp:766)


def refinedet_num_priors(net: int = REFINEDET_NET) -> int:
    """P = 3 * ((S/8)^2 + (S/16)^2 + (S/32)^2 + (S/64)^2): 6375 at S = 320."""
    return 3 * sum((net >> s) ** 2 for s in (3, 4, 5, 6))


def refinedet_preprocess(images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net: int = REFINEDET_NET,
                         stream=None) -> torch.Tensor:
    """GPU drop-in for RefineDet's base_transform (refinedet/refinedet.cpp:822-839) for a batch of device frames: images[i]
    is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched, sizes may differ) -> [B, 3, net, net]
    float32 planes R - 123, G - 117, B - 104 of the whole frame resized to net x net, the engine input.  One launch per 64
    images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net, net), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net}, {net}]", contiguous=False)
    L.check(lib.trtx_refinedet_preprocess_enqueue(descs, n, net, _ptr(out), _stream(stream)),
            "trtx_refinedet_preprocess_enqueue")
    return out


def refinedet_postprocess(arm_loc: torch.Tensor, arm_conf: torch.Tensor, odm_loc: torch.Tensor, odm_conf: torch.Tensor,
                          image_sizes: Sequence[tuple[int, int]] | None = None, *, net: int = REFINEDET_NET,
                          obj_thresh: float = 0.01, conf_thresh: float = 0.01, nms_thresh: float = 0.45,
                          top_k: int = REFINEDET_TOP_K, max_det: int | None = None, score_thresh: float = 0.2,
                          workspace: torch.Tensor | None = None, out: torch.Tensor | None = None,
                          rows_out: torch.Tensor | None = None, stream=None):
    """GPU drop-in for RefineDet's libtorch post-process (refinedet/refinedet.cpp:730-815) on the engine outputs arm_loc
    [B, P, 4], arm_conf [B, P, 2], odm_loc [B, P, 4] and odm_conf [B, P, C], float32 -> dets [B, 1 + max_det*6] float32: the
    count, then (x1, y1, x2, y2, score, label) in the reference's order (classes ascending, each in NMS keep order), zeros
    past the count.  max_det defaults to (C - 1) * top_k, every row the reference can keep.  With image_sizes[b] = (cols,
    rows), also the driver's rectangles after `score < TH` and RoiCorrect (:957-993): rows [B, 1 + max_det*6] of (x, y, w, h,
    score, label) -> (dets, rows).  Two launches, no synchronisation."""
    lib = L.load()
    if odm_conf.dim() != 3:
        raise ValueError("odm_conf must be [B, P, C]")
    B, Pn, Cn = (int(v) for v in odm_conf.shape)
    if Pn != refinedet_num_priors(net):
        raise ValueError(f"the heads hold {Pn} priors; a {net} x {net} net has {refinedet_num_priors(net)}")
    for t, k, what in ((arm_loc, 4, "arm_loc"), (arm_conf, 2, "arm_conf"), (odm_loc, 4, "odm_loc")):
        if tuple(t.shape) != (B, Pn, k):
            raise ValueError(f"{what} must be [{B}, {Pn}, {k}]")
    for t in (arm_loc, arm_conf, odm_loc, odm_conf):
        if t.dtype != torch.float32:
            raise ValueError("arm_loc, arm_conf, odm_loc and odm_conf must be float32")
    if max_det is None:
        max_det = (Cn - 1) * top_k
    q = L.RefinedetParams(net, Cn, obj_thresh, conf_thresh, nms_thresh, top_k, max_det, score_thresh)
    ws_bytes = int(lib.trtx_refinedet_workspace_size(C.byref(q), B))
    if ws_bytes == 0:
        bad = B <= 0 or net <= 0 or Cn < 2 or top_k <= 0 or max_det <= 0 or any(
            v != v for v in (obj_thresh, conf_thresh, nms_thresh, score_thresh))
        L.check(L.ERR_INVALID if bad else L.ERR_UNSUPPORTED, "trtx_refinedet_workspace_size")
    if workspace is None:
        workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=odm_conf.device)
    row = 1 + max_det * 6
    out = _out_tensor(out, (B, row), torch.float32, odm_conf.device, f"out must be contiguous float32 [{B}, {row}]")
    wh_arr = None
    if image_sizes is not None:
        if len(image_sizes) != B:
            raise ValueError(f"expected {B} image sizes")
        wh_arr = _frame_wh(image_sizes)
        rows_out = _out_tensor(rows_out, (B, row), torch.float32, odm_conf.device,
                               f"rows_out must be contiguous float32 [{B}, {row}]")
    L.check(lib.trtx_refinedet_postprocess_enqueue(C.byref(q), B, _ptr(arm_loc), _ptr(arm_conf), _ptr(odm_loc),
                                                   _ptr(odm_conf), _ptr(workspace), _nbytes(workspace), _ptr(out), wh_arr,
                                                   _ptr(rows_out) if wh_arr is not None else None, _stream(stream)),
            "trtx_refinedet_postprocess_enqueue")
    return (out, rows_out) if wh_arr is not None else out


def cubic_preprocess(images: Sequence[torch.Tensor], variant: int, out: torch.Tensor | None = None, net_w: int = 608,
                     net_h: int = 608, stream=None) -> torch.Tensor:
    """GPU drop-in for preprocess_img with cv::resize(INTER_CUBIC) and the driver's plane loop of yolov3-tiny
    (yolov3-tiny/yolov3-tiny.cpp:40-60, :441-445; variant _lib.CUBIC_YOLOV3_TINY, u / 255.0) and retinafaceAntiCov
    (retinafaceAntiCov/retinafaceAntiCov.cpp:41-61, :528-532; variant _lib.CUBIC_ANTICOV, (u - 127.5) * 0.0078125, net
    640 x 640) for a batch of device frames: images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be
    pitched, sizes may differ) -> [B, 3, net_h, net_w] float32 planes in R, G, B order, the engine input: the letterbox on a
    128-grey canvas, resized as OpenCV's own 8-bit INTER_CUBIC (without IPP) does, bit for bit.  One launch per 64 images,
    no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_cubic_preprocess_enqueue(variant, descs, n, net_w, net_h, _ptr(out), _stream(stream)),
            "trtx_cubic_preprocess_enqueue")
    return out


def yolov3spp_letterbox(w: int, h: int, max_size: int = 608) -> tuple[tuple[int, int], tuple[int, int, int, int]]:
    """yolov3-spp's letterbox (yolov3-spp/yolov3-spp.cpp:43-56) of a w x h frame -> ((canvas_w, canvas_h), (x, y, w, h) of
    the resized frame on it).  The canvas is the engine input shape of the frame; the driver skips frames whose canvas is
    below 128 on either side."""
    g = (C.c_int * 6)()
    L.check(L.load().trtx_yolov3spp_letterbox(int(w), int(h), int(max_size), g), "trtx_yolov3spp_letterbox")
    return (g[0], g[1]), (g[2], g[3], g[4], g[5])


def linear_preprocess(images: Sequence[torch.Tensor], variant: int, out: torch.Tensor | None = None, net_w: int = 608,
                      net_h: int = 608, max_size: int = 608, stream=None) -> torch.Tensor:
    """GPU drop-in for preprocess_img with cv::resize(INTER_LINEAR) and the driver's plane loop of yolov3 / yolov4 /
    scaled-yolov4 (variant _lib.LINEAR_YOLOV3: u / 255.0, planes R, G, B; net 608 x 608, scaled-yolov4 512 x 512) and
    retina_r50 / retina_mnet (_lib.LINEAR_RETINA: u - 104, u - 117, u - 123, planes B, G, R; net 640 x 480), and for
    yolov3-spp's letterbox + cv::dnn::blobFromImage (_lib.LINEAR_YOLOV3_SPP: (float)u * (float)(1 / 255.0), planes R, G, B;
    every frame's canvas, yolov3spp_letterbox(w, h, max_size)[0], must be (net_w, net_h)), for a batch of device frames:
    images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched, sizes may differ) ->
    [B, 3, net_h, net_w] float32 planes, the engine input: the frame resized as OpenCV's 8-bit INTER_LINEAR does, bit for
    bit, on a 128-grey canvas.  One launch per 64 images, no synchronisation."""
    lib = L.load()
    n = len(images)
    descs = _image_descs(images)
    out = _out_tensor(out, (n, 3, net_h, net_w), torch.float32, images[0].device if n else "cuda",
                      f"out must be float32 [{n}, 3, {net_h}, {net_w}]", contiguous=False)
    L.check(lib.trtx_linear_preprocess_enqueue(variant, descs, n, net_w, net_h, max_size, _ptr(out), _stream(stream)),
            "trtx_linear_preprocess_enqueue")
    return out


def cls_postprocess(logits: torch.Tensor, k: int, softmax: bool, probs: bool = False, stream=None):
    """GPU drop-in for the cls drivers' softmax (softmax=True: yolov8, yolo11, yolov5) or raw output (softmax=False: yolo26)
    and topk(res, k): logits [B, C] float32 cuda -> (index [B, k] int32, value [B, k] float32[, probs [B, C] float32]).  The
    first min(k, C) entries of each row are written, in descending probability with ties in ascending index; with k > C the
    rest keep their initial zeros.  One launch, no synchronisation."""
    if logits.dtype != torch.float32 or logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous float32 [B, C] tensor")
    b, c = logits.shape
    index = torch.zeros((b, k), dtype=torch.int32, device=logits.device)
    value = torch.zeros((b, k), dtype=torch.float32, device=logits.device)
    p = torch.empty((b, c), dtype=torch.float32, device=logits.device) if probs else None
    L.check(L.load().trtx_cls_postprocess_enqueue(int(softmax), b, c, _ptr(logits), k, _ptr(index), _ptr(value),
                                                  _ptr(p) if p is not None else None, _stream(stream)),
            "trtx_cls_postprocess_enqueue")
    return (index, value, p) if probs else (index, value)


def rcnn_postprocess(scores: torch.Tensor, boxes: torch.Tensor, classes: torch.Tensor, masks: torch.Tensor | None = None, *,
                     img_w: int, img_h: int, net_w: int, net_h: int, score_thresh: float = 0.6, max_masks: int | None = None,
                     out=None, stream=None):
    """GPU drop-in for the post-process loop of rcnn/rcnn.cpp:516-550 for a batch of images of one original size.
    scores [B, D], boxes [B, D, 4], classes [B, D] (BatchedNms outputs), masks [B, D, S, S] (MaskRcnnInference output) or
    None -> (rows [B, 1 + D*7] fp32: count, then (x1, y1, x2, y2, score, class, slot) per kept detection in original-image
    pixels; canvases [B, max_masks, img_h, img_w] uint8 with 255 inside each kept detection's pasted mask, or None).
    `out` = (rows, canvases) to reuse buffers; canvases at or past an image's count are not written (new ones start zeroed)."""
    lib = L.load()
    B, D = scores.shape
    S = 1 if masks is None else masks.shape[-1]
    if tuple(boxes.shape) != (B, D, 4) or tuple(classes.shape) != (B, D) or (masks is not None and tuple(masks.shape) != (B, D, S, S)):
        raise ValueError("expected scores [B, D], boxes [B, D, 4], classes [B, D], masks [B, D, S, S]")
    max_masks = D if max_masks is None else int(max_masks)
    q = L.RcnnPostParams(net_w, net_h, img_w, img_h, D, S, max_masks, score_thresh)
    rows, canvases = out if out is not None else (None, None)
    if rows is None:
        rows = torch.empty((B, 1 + D * 7), dtype=torch.float32, device=scores.device)
    if masks is not None and canvases is None:
        canvases = torch.zeros((B, max_masks, img_h, img_w), dtype=torch.uint8, device=scores.device)
    if masks is None:
        canvases = None
    L.check(lib.trtx_rcnn_postprocess_enqueue(C.byref(q), B, _ptr(scores), _ptr(boxes), _ptr(classes),
                                              None if masks is None else _ptr(masks), _ptr(rows),
                                              None if canvases is None else _ptr(canvases), _stream(stream)),
            "trtx_rcnn_postprocess_enqueue")
    return rows, canvases


def rcnn_postprocess_frames(scores: torch.Tensor, boxes: torch.Tensor, classes: torch.Tensor, masks: torch.Tensor | None = None,
                            *, frames: Sequence[tuple[int, int]], net_w: int, net_h: int, score_thresh: float = 0.6,
                            max_masks: int | None = None, rows: torch.Tensor | None = None,
                            canvases: Sequence[torch.Tensor] | None = None, stream=None):
    """rcnn_postprocess for a batch of frames of mixed original sizes: frames[b] = (img_w, img_h) of frame b, which is
    rescaled and pasted with its own size and pads (the same as a batch-1 rcnn_postprocess of frame b).
    -> (rows [B, 1 + D*7] fp32, per-frame u8 canvases [max_masks, img_h, img_w], or None when masks is None).
    `canvases[b]` may be any u8 cuda tensor [max_masks, img_h, img_w] with contiguous rows and slots (e.g. a view
    [..., :img_w] of a pitched buffer); canvases at or past a frame's count are not written (new ones start zeroed).
    Two launches per 64 frames."""
    lib = L.load()
    B = len(frames)
    if B == 0 or scores.dim() != 2 or scores.shape[0] != B:
        raise ValueError(f"scores must be [{B}, D] for {B} frames")
    D = scores.shape[1]
    S = 1 if masks is None else masks.shape[-1]
    if tuple(boxes.shape) != (B, D, 4) or tuple(classes.shape) != (B, D) or (masks is not None and tuple(masks.shape) != (B, D, S, S)):
        raise ValueError("expected scores [B, D], boxes [B, D, 4], classes [B, D], masks [B, D, S, S]")
    for t in (scores, boxes, classes) + (() if masks is None else (masks,)):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("scores, boxes, classes and masks must be contiguous float32")
    max_masks = D if max_masks is None else int(max_masks)
    q = L.RcnnPostParams(net_w, net_h, 0, 0, D, S, max_masks, score_thresh)  # img_w / img_h: per frame below
    rows = _out_tensor(rows, (B, 1 + D * 7), torch.float32, scores.device, f"rows must be contiguous float32 [{B}, {1 + D * 7}]")
    descs, canvases = _frames(frames, canvases, max_masks, scores.device, masks is not None)
    L.check(lib.trtx_rcnn_postprocess_frames_enqueue(C.byref(q), descs, B, _ptr(scores), _ptr(boxes), _ptr(classes),
                                                     None if masks is None else _ptr(masks), _ptr(rows), _stream(stream)),
            "trtx_rcnn_postprocess_frames_enqueue")
    return rows, canvases


def rcnn_contours(rows: torch.Tensor, canvases: Sequence[torch.Tensor], *, frames: Sequence[tuple[int, int]],
                  detections_per_im: int, max_masks: int, max_contours: int, max_points: int, out=None, stream=None):
    """cv2.findContours(canvas, RETR_EXTERNAL, CHAIN_APPROX_NONE) of every kept canvas of an rcnn_postprocess(_frames) call
    (rcnn/rcnn.cpp:551-552), read inside each row's paste rectangle.  rows [B, 1 + D*7] and canvases[b] [max_masks, img_h,
    img_w] u8 as that call returned them (or views with contiguous rows and slots); frames[b] = (img_w, img_h).
    -> (counts [B, max_masks, 2] int32: (n_contours, n_points), true totals; lengths [B, max_masks, max_contours] int32;
    points [B, max_masks, max_points, 2] int32 (x, y)), contours in cv2's order.  Entries past the counts are not written
    (new tensors start zeroed); `out` = (counts, lengths, points) reuses tensors.  Allocates the workspace."""
    lib = L.load()
    B = len(frames)
    D = int(detections_per_im)
    if B == 0 or tuple(rows.shape) != (B, 1 + D * 7) or rows.dtype != torch.float32 or not rows.is_contiguous():
        raise ValueError(f"rows must be contiguous float32 [{B}, {1 + D * 7}]")
    q = L.RcnnPostParams(0, 0, 0, 0, D, 1, int(max_masks), 0.0)  # only detections_per_im and max_masks are read
    descs, _ = _frames(frames, canvases, int(max_masks), rows.device, True)
    shapes = ((B, max_masks, 2), (B, max_masks, max_contours), (B, max_masks, max_points, 2))
    out = tuple(_out_tensor(t, s, torch.int32, rows.device, f"out tensors must be contiguous int32 {shapes}", torch.zeros)
                for t, s in zip((None,) * 3 if out is None else out, shapes))
    n = lib.trtx_rcnn_contours_workspace_size(C.byref(q), descs, B)
    if n == 0:
        raise ValueError("trtx_rcnn_contours_workspace_size rejected the arguments")
    work = torch.empty(n, dtype=torch.uint8, device=rows.device)
    L.check(lib.trtx_rcnn_contours_enqueue(C.byref(q), descs, B, _ptr(rows), int(max_contours), int(max_points),
                                           _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(work), n, _stream(stream)),
            "trtx_rcnn_contours_enqueue")
    return tuple(out)

def letterbox_matrix(src_w: int, src_h: int, dst_w: int, dst_h: int):
    m = (C.c_float * 6)()
    L.load().trtx_letterbox_matrix(src_w, src_h, dst_w, dst_h, m)
    return list(m)


# The Python runners (the *_trt.py scripts).  Row format of each detection runner's post_process: (box format its xywh2xyxy
# reads, floats per plugin row, the float non_max_suppression compares as the label -- boxes[:, -1] after the runner's
# reshape or slice --, the column yolov3 multiplies into the confidence or -1).  The label is the row's last float, not its
# class: float 89 of a 90-float row is the OBB angle a detection plugin never writes, so those runners' NMS is class-blind
# wherever that float is equal; yolov9 compares float 37, a mask coefficient.
PYRUNNER_PRESETS = {
    "yolov8_det_trt": (L.BOX_LTRB, 90, 89, -1),
    "yolov8_5u_det_trt": (L.BOX_LTRB, 90, 89, -1),
    "yolo11_det_trt": (L.BOX_LTRB, 90, 89, -1),
    "yolov12_det_trt": (L.BOX_LTRB, 90, 89, -1),  # yolov12-tubro
    "yolov9_trt": (L.BOX_LTRB, 38, 37, -1),
    "yolov10_det_trt": (L.BOX_LTRB, 6, 5, -1),
    "yolov13_det_trt": (L.BOX_LTRB, 6, 5, -1),
    "yolov7_trt": (L.BOX_CXCYWH, 6, 5, -1),
    "yolov5_det_trt": (L.BOX_CXCYWH, 38, 5, -1),  # `pred[:, :6]`
    "yolov5_det_cuda_python": (L.BOX_CXCYWH, 6, 5, -1),
    "yolov3_trt": (L.BOX_CXCYWH, 7, 5, 6),  # `pred[:, 4] *= pred[:, 6]`, then `pred[:, :-1]`
}


def pyrunner_letterbox_rect(w: int, h: int, net_w: int = 640, net_h: int = 640) -> tuple[int, int, int, int]:
    """preprocess_image's rectangle (x, y, w, h) of a w x h frame in a net_w x net_h input (ratios in double)."""
    r = (C.c_int * 4)()
    L.check(L.load().trtx_pyrunner_letterbox_rect(int(w), int(h), int(net_w), int(net_h), r), "trtx_pyrunner_letterbox_rect")
    return tuple(r)


class PyRunnerPreprocessPlan:
    """GPU drop-in for the Python runners' preprocess_image (yolov8/yolov8_det_trt.py:207-253; the same body in every
    yolov5, yolov7, yolov8, yolo11, yolov9, yolov10, yolov12-tubro and yolov13 runner, seg / pose / obb included) for a batch
    of persistent device frames: images[i] is a u8 HWC BGR cuda tensor [h, w, 3] with packed pixels (rows may be pitched,
    sizes may differ) -> out [B, 3, net_h, net_w] float32 planes R, G, B, the frame resized by cv2.resize(INTER_LINEAR) into
    pyrunner_letterbox_rect's rectangle on a 128 canvas, / 255.0, bit for bit.  The descriptors are built once; enqueue() is
    one C call, one launch per 64 frames, no synchronisation."""

    def __init__(self, images: Sequence[torch.Tensor], out: torch.Tensor | None = None, net_w: int = 640, net_h: int = 640):
        self._lib = L.load()
        self.n = len(images)
        self.descs = _image_descs(images)
        self._keep = list(images)
        self.net_w, self.net_h = int(net_w), int(net_h)
        self.out = _out_tensor(out, (self.n, 3, self.net_h, self.net_w), torch.float32,
                               images[0].device if self.n else "cuda",
                               f"out must be float32 [{self.n}, 3, {self.net_h}, {self.net_w}]", contiguous=False)

    def enqueue(self, stream=None) -> torch.Tensor:
        L.check(self._lib.trtx_linear_preprocess_enqueue(L.LINEAR_PY, self.descs, self.n, self.net_w, self.net_h, 0,
                                                         _ptr(self.out), _stream(stream)), "trtx_linear_preprocess_enqueue")
        return self.out


class PyRunnerPostprocess:
    """GPU drop-in for a detection runner's post_process (non_max_suppression, bbox_iou, xywh2xyxy; yolov8_det_trt.py:255-381)
    for a batch of frames of any sizes.  runner: a key of PYRUNNER_PRESETS; max_rows: the plugin's max output rows (1000).
    __call__(dets, image_sizes): dets [B, 1 + max_rows*row_floats] float32, the plugin output; image_sizes[b] = (img_w,
    img_h) -> rows [B, 1 + max_rows*6] float32: the kept count, then (x1, y1, x2, y2, conf, class) per kept row at the frame's
    size, in the runner's order, zero past the count.  Bit for bit with the runner's numpy where its argsort has no ties;
    equal confidences keep ascending row order, and a front row that does not suppress itself (a NaN label or box, an
    inverted box: the runner never returns there) is kept once.  One launch per 64 frames, no workspace."""

    def __init__(self, runner: str, *, max_rows: int = 1000, net_w: int = 640, net_h: int = 640, conf_thresh: float = 0.5,
                 nms_thresh: float = 0.4):
        if runner not in PYRUNNER_PRESETS:
            raise ValueError(f"runner must be one of {sorted(PYRUNNER_PRESETS)}")
        box, self.row_floats, label_col, conf_col = PYRUNNER_PRESETS[runner]
        self.max_rows = int(max_rows)
        self.params = L.PyrunnerParams(box, int(net_w), int(net_h), self.row_floats, label_col, conf_col, conf_thresh,
                                       nms_thresh)

    def __call__(self, dets: torch.Tensor, image_sizes: Sequence[tuple[int, int]], rows_out: torch.Tensor | None = None,
                 stream=None) -> torch.Tensor:
        lib = L.load()
        B = len(image_sizes)
        if dets.dim() != 2 or dets.shape[0] != B or dets.shape[1] < 1 + self.max_rows * self.row_floats:
            raise ValueError(f"dets must be [{B}, >= {1 + self.max_rows * self.row_floats}]")
        _f32_rows(dets)
        rows_out = _out_tensor(rows_out, (B, 1 + self.max_rows * 6), torch.float32, dets.device,
                               f"rows_out must be contiguous float32 [{B}, {1 + self.max_rows * 6}]")
        L.check(lib.trtx_pyrunner_postprocess_enqueue(C.byref(self.params), _frame_wh(image_sizes), B, _ptr(dets),
                                                      self.max_rows, _ptr(rows_out), _stream(stream)),
                "trtx_pyrunner_postprocess_enqueue")
        return rows_out
