"""Detection hot path as one object: pinned frames -> H2D -> batched letterbox pre-process ->
[backbone: TensorRT in the reference, injected here] -> fused YoloLayer decode + NMS -> D2H of the
compact detections.  This is the call a user of the reference's `yolov8_det -d` loop makes per batch
(yolov8/yolov8_det.cpp:223-244), minus disk IO and drawing.

Everything is asynchronous on one CUDA stream; the only host synchronisation is the caller's.
Multi-GPU: one pipeline per process/GPU (batch-sharded, images are independent -- SURVEY 8e);
`gather()` is the single NCCL collective (fixed-size all-gather of the compact detections).
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch

from . import _lib as L
from .plugins import FusedYoloDecodeNms, PreprocessPlan, YoloLayerPlugin


class DetectionPipeline:
    def __init__(self, batch: int, src_h: int = 640, src_w: int = 640, net_h: int = 640, net_w: int = 640,
                 num_classes: int = 80, strides: Sequence[int] = (8, 16, 32), max_out: int = 1000,
                 conf_thresh: float = 0.5, nms_thresh: float = 0.45, device: str | torch.device = "cuda",
                 input_dtype: torch.dtype = torch.float32, head_dtype: int = L.F32,
                 backbone: Callable[[torch.Tensor], Sequence[torch.Tensor]] | None = None, plugin=None):
        """plugin: any YoloLayer plugin mirror (YoloLayerPluginV5 / V7 / ...); default = the yolov8 one."""
        self.batch, self.src_h, self.src_w, self.net_h, self.net_w = batch, src_h, src_w, net_h, net_w
        self.device = torch.device(device)
        self.backbone = backbone
        self.plugin = plugin if plugin is not None else YoloLayerPlugin(num_classes, 17, 0.0, net_w, net_h, max_out, False, False,
                                                                        False, strides, in_dtype=head_dtype)
        self.fused = FusedYoloDecodeNms(self.plugin, batch, conf_thresh, nms_thresh, max_det=max_out,
                                        device=self.device, return_index=False)
        self.frames_dev = torch.empty((batch, src_h, src_w, 3), dtype=torch.uint8, device=self.device)
        self.net_input = torch.empty((batch, 3, net_h, net_w), dtype=input_dtype, device=self.device)
        self.out_host = torch.empty((batch, 1 + max_out * 7), dtype=torch.float32).pin_memory()
        self.h2d_bytes = self.frames_dev.numel()
        self.d2h_bytes = self.out_host.numel() * 4
        # descriptors of the (persistent) device frame buffers are built once, not per step
        self.pre = PreprocessPlan(list(self.frames_dev.unbind(0)), self.net_input, net_w, net_h)
        # decode + NMS of the heads run on a high-priority side stream next to the letterbox (see run_device)
        self._side = torch.cuda.Stream(self.device, priority=-1) if self.device.type == "cuda" else None

    def run(self, frames_host: torch.Tensor, heads: Sequence[torch.Tensor] | None = None, stream=None) -> torch.Tensor:
        """frames_host: pinned uint8 [B, H, W, 3] BGR.  heads: the backbone's per-stride outputs when no
        backbone callable was given.  Returns the pinned host buffer [B, 1+K*7] (valid after a stream sync)."""
        self.frames_dev.copy_(frames_host, non_blocking=True)
        self.pre.enqueue(stream)
        if self.backbone is not None:
            heads = self.backbone(self.net_input)
        out, _ = self.fused.enqueue(self.batch, heads, stream)
        self.out_host.copy_(out, non_blocking=True)
        return self.out_host

    def run_device(self, heads: Sequence[torch.Tensor], stream=None, overlap: bool = True,
                   peer_gather: "PeerGather | None" = None, slot: int = 0) -> torch.Tensor:
        """Device-resident step: pre-process the frames already in HBM + decode + NMS (no host copies).

        The letterbox of this batch does not depend on the decode/NMS of the head tensors (with a real backbone the heads
        of batch i are decoded while the frames of batch i+1 are pre-processed), so the two halves are issued as
        parallel branches: scan -> NMS on a high-priority side stream forked from the current stream, the letterbox on
        the current stream, joined at the end.  Captured into a CUDA graph this becomes two concurrent branches; the
        latency-bound NMS (one CTA per image, 32 of 132 SMs) then runs underneath the HBM-bound letterbox instead of
        after it."""
        if not overlap or self._side is None or stream is not None:
            self.pre.enqueue(stream)
            out = self.decode_nms_gather(heads, peer_gather, stream, slot)
            return out
        cur = torch.cuda.current_stream(self.device)
        self._side.wait_stream(cur)                  # fork
        with torch.cuda.stream(self._side):
            out = self.decode_nms_gather(heads, peer_gather, None, slot)
        self.pre.enqueue()
        cur.wait_stream(self._side)                  # join
        return out

    def decode_nms_gather(self, heads, peer_gather: "PeerGather | None" = None, stream=None, slot: int = 0, fused_gather: bool = False,
                          wait: bool = True) -> torch.Tensor:
        """scan -> NMS (-> the multi-GPU gather into `slot`: push kernel after the NMS by default, from inside nms_kernel with
        fused_gather=True; then the wait kernel unless wait=False)."""
        if peer_gather is None:
            return self.fused.enqueue(self.batch, heads, stream)[0]
        if fused_gather:
            out, _ = self.fused.enqueue(self.batch, heads, stream, gather=peer_gather.desc(slot))
        else:
            out, _ = self.fused.enqueue(self.batch, heads, stream)
            peer_gather.push(out, slot, self.fused.max_det, 0, stream)
        if wait:
            peer_gather.wait(slot, stream)
        return out

    # ---- overlapped host pipeline: H2D of batch i+1 runs on a copy stream while batch i is decoded ----
    def _make_slots(self, n: int) -> None:
        self._slots = []
        for _ in range(n):
            fd = torch.empty_like(self.frames_dev)
            self._slots.append({
                "frames": fd,
                "pre": PreprocessPlan(list(fd.unbind(0)), self.net_input, self.net_w, self.net_h),
                "out_host": torch.empty_like(self.out_host).pin_memory(),
                "h2d": torch.cuda.Event(), "done": torch.cuda.Event(),
            })
            self._slots[-1]["done"].record(torch.cuda.current_stream(self.device))
        self._copy_stream = torch.cuda.Stream(self.device)
        self._next = 0

    def submit(self, frames_host: torch.Tensor, heads: Sequence[torch.Tensor] | None = None, slots: int = 2,
               peer_gather: "PeerGather | None" = None, gather_slot: int = 0):
        """Asynchronous step with double buffering: returns (pinned host result, event); the result is valid
        once the event has completed.  The H2D copy is issued on a dedicated copy stream so that it overlaps
        the kernels of the previous submit() (the reference serialises memcpy -> H2D -> kernel -> sync per
        image, yolov8/src/preprocess.cu:89-127)."""
        if not hasattr(self, "_slots"):
            self._make_slots(slots)
        sl = self._slots[self._next]
        self._next = (self._next + 1) % len(self._slots)
        compute = torch.cuda.current_stream(self.device)
        self._copy_stream.wait_event(sl["done"])           # slot buffers are free again
        with torch.cuda.stream(self._copy_stream):
            sl["frames"].copy_(frames_host, non_blocking=True)
            sl["h2d"].record(self._copy_stream)
        compute.wait_event(sl["h2d"])
        sl["pre"].enqueue()
        if self.backbone is not None:
            heads = self.backbone(self.net_input)
        out = self.decode_nms_gather(heads, peer_gather, None, gather_slot)
        sl["out_host"].copy_(out, non_blocking=True)
        sl["done"].record(compute)
        return sl["out_host"], sl["done"]

    # ---- CUDA graphs: the step is launch-bound (4 kernels of 10-30 us), so replaying a captured graph
    # removes the per-launch host cost (guide: "capture launch-bound inner loops in CUDA graphs") ----
    def capture(self, fn: Callable[[], object], capture_error_mode: str = "global") -> "torch.cuda.CUDAGraph":
        """Capture `fn` (which must only enqueue work on the current stream, or on streams forked from and joined
        back into it) into a CUDA graph.  Use capture_error_mode="thread_local" when other threads of the process
        (e.g. the NCCL watchdog) may touch CUDA during the capture."""
        fn()  # warm-up outside capture (lazy module loads, cudaFuncSetAttribute)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode=capture_error_mode):
            fn()
        return g


class RetinaPipeline:
    """retina_r50.cpp's per-batch loop on the device: letterbox of the frames, Decode_TRT over the three head tensors,
    nms() with landmarks (retinaface/retina_r50.cpp:320-360, common.hpp:110-130).  Same structure as DetectionPipeline:
    decode + NMS on a high-priority side stream next to the letterbox."""

    def __init__(self, batch: int, in_h: int = 640, in_w: int = 640, max_det: int = 2048, device="cuda"):
        from .plugins import DecodePlugin, float_le_threshold, nms_params

        self.batch, self.device = batch, torch.device(device)
        self.plugin = DecodePlugin(in_h, in_w)
        self._lib = L.load()
        self.frames_dev = torch.empty((batch, in_h, in_w, 3), dtype=torch.uint8, device=self.device)
        self.net_input = torch.empty((batch, 3, in_h, in_w), dtype=torch.float32, device=self.device)
        self.pre = PreprocessPlan(list(self.frames_dev.unbind(0)), self.net_input, in_w, in_h)
        self.rows = torch.empty((batch, self.plugin.output_elems()), dtype=torch.float32, device=self.device)
        self.ws = torch.empty(max(self.plugin.getWorkspaceSize(batch), 256), dtype=torch.uint8, device=self.device)
        self.q = nms_params(L.BOX_RETINA, L.NMS_GREEDY, float_le_threshold(0.1), 0.4, max_det, False, extra_floats=10, extra_offset=5)
        self.max_rows = self.plugin.total_priors
        self.out = torch.empty((batch, 1 + max_det * 17), dtype=torch.float32, device=self.device)
        import ctypes as C
        self.nms_ws_bytes = int(self._lib.trtx_nms_workspace_size(C.byref(self.q), batch, self.max_rows))
        self.nms_ws = torch.empty(max(self.nms_ws_bytes, 256), dtype=torch.uint8, device=self.device)
        self.out_host = torch.empty_like(self.out, device="cpu").pin_memory()
        self._side = torch.cuda.Stream(self.device, priority=-1)
        self.h2d_bytes, self.d2h_bytes = self.frames_dev.numel(), self.out.numel() * 4

    def decode_nms(self, heads) -> torch.Tensor:
        import ctypes as C

        from .plugins import _ptr, _stream
        rc = self.plugin.enqueue(self.batch, heads, [self.rows], self.ws)
        if rc:
            L.check(rc, "trtx_retina_decode_enqueue")
        L.check(self._lib.trtx_nms_enqueue(C.byref(self.q), self.batch, _ptr(self.rows), self.max_rows, 15, _ptr(self.out), None,
                                           _ptr(self.nms_ws), self.nms_ws_bytes, _stream(None)), "trtx_nms_enqueue")
        return self.out

    def run_device(self, heads, overlap: bool = True) -> torch.Tensor:
        cur = torch.cuda.current_stream(self.device)
        if not overlap:
            self.pre.enqueue()
            return self.decode_nms(heads)
        self._side.wait_stream(cur)
        with torch.cuda.stream(self._side):
            self.decode_nms(heads)
        self.pre.enqueue()
        cur.wait_stream(self._side)
        return self.out

    def run(self, frames_host: torch.Tensor, heads) -> torch.Tensor:
        self.frames_dev.copy_(frames_host, non_blocking=True)
        self.run_device(heads)
        self.out_host.copy_(self.out, non_blocking=True)
        return self.out_host

    capture = DetectionPipeline.capture


class RcnnHeadChain:
    """The four Faster R-CNN plugins chained on one stream exactly as rcnn.cpp wires them (rcnn/rcnn.cpp:134-195):
    RpnDecode -> RpnNms -> [RoIAlign + box head: TensorRT, not on this path; its outputs are inputs here] ->
    PredictorDecode -> BatchedNms.  All images of the batch per launch."""

    def __init__(self, batch: int, anchors, device="cuda", H: int = 50, W: int = 67, image_h: int = 800, image_w: int = 1067,
                 pre: int = 6000, post: int = 1000, classes: int = 80, dets: int = 100, nms_method: int = 1):
        from .plugins import BatchedNmsPlugin, PredictorDecodePlugin, RpnDecodePlugin, RpnNmsPlugin

        dev = torch.device(device)
        self.batch, self.device = batch, dev
        self.p_dec = RpnDecodePlugin(pre, anchors, 16.0, image_h, image_w, H, W)
        self.p_nms = RpnNmsPlugin(0.7, post, pre)
        self.p_pred = PredictorDecodePlugin(post, image_h, image_w, (10.0, 10.0, 5.0, 5.0), classes)
        self.p_bnms = BatchedNmsPlugin(nms_method, 0.5, dets, post)
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)  # noqa: E731
        self.s6, self.b6, self.props = z(batch, pre), z(batch, pre, 4), z(batch, post, 4)
        self.ps, self.pb, self.pc = z(batch, post), z(batch, post, 4), z(batch, post)
        self.fs, self.fb, self.fc = z(batch, dets), z(batch, dets, 4), z(batch, dets)
        self.ws = torch.empty(max(self.p_dec.getWorkspaceSize(batch), 4096), dtype=torch.uint8, device=dev)
        self.out_host = torch.empty((batch, dets, 6), dtype=torch.float32).pin_memory()
        self.d2h_bytes = self.out_host.numel() * 4

    def run_device(self, rpn_scores, rpn_deltas, cls_scores, box_deltas):
        for rc in (self.p_dec.enqueue(self.batch, [rpn_scores, rpn_deltas], [self.s6, self.b6], self.ws),
                   self.p_nms.enqueue(self.batch, [self.s6, self.b6], [self.props], self.ws),
                   self.p_pred.enqueue(self.batch, [cls_scores, box_deltas, self.props], [self.ps, self.pb, self.pc], self.ws),
                   self.p_bnms.enqueue(self.batch, [self.ps, self.pb, self.pc], [self.fs, self.fb, self.fc], self.ws)):
            if rc:
                raise L.TrtxError(f"rcnn plugin enqueue failed: {rc}")
        return self.fs, self.fb, self.fc

    capture = DetectionPipeline.capture


class _RawCuda:
    """A raw device pointer as something torch.as_tensor can wrap (no copy)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"data": (int(ptr), False), "shape": tuple(shape), "typestr": typestr, "version": 2}


class PeerGather:
    """The gather of the compact detections over NVLink peer memory (trtx_gather, include/trtx_hot.h): `push(out, slot)`
    enqueues the small kernel that copies this rank's kept rows into `slot` of the gathered buffer of EVERY rank and
    publishes the slot (it waits for nobody); `wait(slot)` enqueues the one-warp kernel that returns once every rank's rows
    of the round are in the local buffer.  No NCCL kernel competes with the step for SMs (the NCCL all-gather of round 1
    stretched the step by 8-20 %, DESIGN.md section 5).  `desc(slot)` is the descriptor for the variant fused into
    nms_kernel (FusedYoloDecodeNms.enqueue(gather=...)).

    Buffers are cudaMalloc'ed by the library and exchanged between the processes of the node as CUDA IPC handles through
    torch.distributed (object all-gather); torch is plumbing only.  `result(slot)` views this rank's gathered buffer
    [world*batch, 1 + max_det*7]; rows past each image's count are stale.  Slot reuse: see trtx_hot.h (use 2*G slots in
    halves, a round's pushes then its waits)."""

    def __init__(self, world: int, rank: int, batch: int, cols: int, device, slots: int = 8):
        import ctypes as C

        import torch.distributed as dist

        self._lib = L.load()
        self.world, self.rank, self.batch, self.cols, self.slots = world, rank, batch, cols, slots
        self.device = torch.device(device)
        out_bytes = slots * world * batch * cols * 4
        flag_bytes = world * slots * 4
        self._own, handles = [], []
        for nbytes in (out_bytes, flag_bytes, 16):
            ptr, h = C.c_void_p(), (C.c_ubyte * 64)()
            L.check(self._lib.trtx_peer_alloc(nbytes, C.byref(ptr), h), "trtx_peer_alloc")
            self._own.append(ptr.value)
            handles.append(bytes(h))
        every = [None] * world
        if world > 1:
            dist.all_gather_object(every, (rank, handles[0], handles[1]))
        else:
            every = [(rank, handles[0], handles[1])]
        self._out_ptrs, self._flag_ptrs = [0] * world, [0] * world
        self._opened = []
        for r, h_out, h_flags in every:
            if r == rank:
                self._out_ptrs[r], self._flag_ptrs[r] = self._own[0], self._own[1]
                continue
            for k, h in ((0, h_out), (1, h_flags)):
                ptr = C.c_void_p()
                buf = (C.c_ubyte * 64).from_buffer_copy(h)
                L.check(self._lib.trtx_peer_open(buf, C.byref(ptr)), "trtx_peer_open")
                self._opened.append(ptr.value)
                (self._out_ptrs if k == 0 else self._flag_ptrs)[r] = ptr.value
        self._descs = [self._make_desc(s) for s in range(slots)]
        self._out = torch.as_tensor(_RawCuda(self._own[0], (slots, world * batch, cols), "<f4"), device=self.device)
        self._ctrl = torch.as_tensor(_RawCuda(self._own[2], (4,), "<u4"), device=self.device)
        self._flags = torch.as_tensor(_RawCuda(self._own[1], (world, slots), "<u4"), device=self.device)
        if world > 1:
            dist.barrier()  # every rank has mapped every buffer before anyone stores into them

    def _make_desc(self, slot: int):
        g = L.Gather()
        g.world, g.rank, g.slots, g.slot = self.world, self.rank, self.slots, slot
        for r in range(self.world):
            g.out_dev[r], g.flags_dev[r] = self._out_ptrs[r], self._flag_ptrs[r]
        g.ctrl_dev = self._own[2]
        return g

    def desc(self, slot: int):
        return self._descs[slot]

    def result(self, slot: int) -> torch.Tensor:
        return self._out[slot]

    def published(self) -> torch.Tensor:
        """[world, slots] publish counters as seen by this rank."""
        return self._flags

    def error(self) -> int:
        return int(self._ctrl[2].item())

    def push(self, local_out: torch.Tensor, slot: int, max_det: int, extra_floats: int = 0, stream=None) -> None:
        import ctypes as C

        from .plugins import _ptr, _stream
        L.check(self._lib.trtx_gather_push_enqueue(C.byref(self._descs[slot]), _ptr(local_out), int(local_out.shape[0]), int(max_det),
                                                   int(extra_floats), _stream(stream)), "trtx_gather_push_enqueue")

    def wait(self, slot: int, stream=None, n: int = 1) -> None:
        """Wait for slots slot .. slot+n-1 (one launch)."""
        import ctypes as C

        from .plugins import _stream
        L.check(self._lib.trtx_gather_wait_many_enqueue(C.byref(self._descs[slot]), int(n), _stream(stream)), "trtx_gather_wait_many_enqueue")

    def push_many(self, local_outs, slot: int, max_det: int, extra_floats: int = 0, stream=None) -> None:
        """Publish len(local_outs) local outputs into slots slot .. in ONE launch (one system-scope release for the round)."""
        import ctypes as C

        from .plugins import _ptr, _stream
        ptrs = L.ptr_array([_ptr(t) for t in local_outs])
        L.check(self._lib.trtx_gather_push_many_enqueue(C.byref(self._descs[slot]), ptrs, len(local_outs), int(local_outs[0].shape[0]),
                                                        int(max_det), int(extra_floats), _stream(stream)), "trtx_gather_push_many_enqueue")

    def close(self) -> None:
        for p in self._opened:
            self._lib.trtx_peer_close(p)
        self._opened = []
        for p in self._own:
            self._lib.trtx_peer_free(p)
        self._own = []


def gather(local: torch.Tensor, world_size: int) -> torch.Tensor:
    """The one collective of the path: fixed-size all-gather of [B_local, 1+K*7] (SURVEY 8e)."""
    import torch.distributed as dist

    if world_size == 1:
        return local
    out = torch.empty((world_size * local.shape[0], local.shape[1]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous())
    return out


class GatherRing:
    """The same all-gather, pipelined: step i's compact detections travel on a side stream while step i+1 computes.

    `slots` preallocated destination buffers ([world*B_local, 1+K*7]); `launch(local, slot)` orders the collective
    after everything queued so far on the current stream and returns immediately; `reuse(slot)` makes the current stream
    wait until that slot's previous collective has read its source (call it before overwriting the source buffer);
    `join()` makes the current stream wait for all collectives (call before the closing timing event / before reading).
    On a CPU process group (gloo, tests) there are no streams and every call is synchronous."""

    def __init__(self, world_size: int, rows: int, cols: int, device, slots: int = 4, dtype=torch.float32):
        self.world = world_size
        self.cuda = torch.device(device).type == "cuda"
        self.bufs = [torch.empty((world_size * rows, cols), dtype=dtype, device=device) for _ in range(slots)]
        if self.cuda:
            self.comm = torch.cuda.Stream(device=device)
            self.done = [torch.cuda.Event() for _ in range(slots)]
            self.ready = [torch.cuda.Event() for _ in range(slots)]
            self.used = [False] * slots

    def launch(self, local: torch.Tensor, slot: int) -> torch.Tensor:
        import torch.distributed as dist

        out = self.bufs[slot]
        if self.world == 1:
            return local
        if not self.cuda:
            dist.all_gather_into_tensor(out, local.contiguous())
            return out
        cur = torch.cuda.current_stream(local.device)
        self.ready[slot].record(cur)
        self.comm.wait_event(self.ready[slot])
        with torch.cuda.stream(self.comm):
            dist.all_gather_into_tensor(out, local)
            self.done[slot].record(self.comm)
        self.used[slot] = True
        return out

    def reuse(self, slot: int) -> None:
        if self.cuda and self.world > 1 and self.used[slot]:
            torch.cuda.current_stream(self.bufs[slot].device).wait_event(self.done[slot])

    def join(self) -> None:
        if self.cuda and self.world > 1:
            torch.cuda.current_stream(self.bufs[0].device).wait_stream(self.comm)
