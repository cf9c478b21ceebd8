"""The half-precision mode of RpnDecode and PredictorDecode, as far as it goes without a device: the ctypes signatures of
trtx_rpn_decode_typed / trtx_predictor_decode_typed, the argument checks that come before the launch, the dtype selection of
the Python wrappers, and the TensorRT adapters' host surface (tests/trt_adapter_rcnn_half_check.cpp against tests/mock_trt)."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

from tensorrtx_b200 import _lib as L
from tensorrtx_b200 import plugins as P

ROOT = Path(__file__).resolve().parents[1]
INV, UNS = -L.ERR_INVALID, -L.ERR_UNSUPPORTED
ANCHORS = (C.c_float * 60)(*([1.0] * 60))
W4 = (C.c_float * 4)(10.0, 10.0, 5.0, 5.0)
NOMINAL = 256


def _fake(n):
    """a non-null address that is never dereferenced: every call below returns before the launch"""
    return 0x10000 * n


def test_ctypes_signatures():
    lib = L.load()
    rpn, pred = lib.trtx_rpn_decode_typed, lib.trtx_predictor_decode_typed
    assert rpn.restype is C.c_int64 and pred.restype is C.c_int64
    # the typed calls are the untyped ones with the element type in front
    assert rpn.argtypes[0] is C.c_int and rpn.argtypes[1:] == lib.trtx_rpn_decode.argtypes
    assert pred.argtypes[0] is C.c_int and pred.argtypes[1:] == lib.trtx_predictor_decode.argtypes
    assert len(rpn.argtypes) == 17 and len(pred.argtypes) == 16


def _rpn(dtype=L.F16, scores=_fake(1), deltas=_fake(2), os_=_fake(3), ob=_fake(4), batch=1, h=50, w=67, anchors=15, top_n=6000,
         ws=_fake(5), typed=True):
    lib = L.load()
    args = (batch, scores, deltas, os_, ob, h, w, 800, 1067, 16.0, ANCHORS, anchors, top_n, ws, 0 if ws is None else 4096, None)
    return lib.trtx_rpn_decode_typed(dtype, *args) if typed else lib.trtx_rpn_decode(*args)


def _pred(dtype=L.F16, scores=_fake(1), deltas=_fake(2), props=_fake(3), outs=(_fake(4), _fake(5), _fake(6)), batch=1, n=1000,
          nc=80, ws=_fake(7), typed=True):
    lib = L.load()
    args = (batch, scores, deltas, props, *outs, n, nc, 800, 1067, W4, ws, 0 if ws is None else 4096, None)
    return lib.trtx_predictor_decode_typed(dtype, *args) if typed else lib.trtx_predictor_decode(*args)


def test_workspace_query_does_not_depend_on_the_type():
    for f in (_rpn, _pred):
        assert f(dtype=L.F32, ws=None) == f(dtype=L.F16, ws=None) == f(ws=None, typed=False) == NOMINAL
        assert f(dtype=2, ws=None) == f(dtype=-1, ws=None) == INV          # an unknown type is never a size


def test_rpn_decode_argument_checks_before_the_launch():
    assert _rpn(dtype=2) == _rpn(dtype=-1) == _rpn(dtype=0x101) == INV
    assert _rpn(scores=_fake(1) + 1) == _rpn(deltas=_fake(2) + 1) == INV                  # half pointers on odd addresses
    assert _rpn(scores=None) == _rpn(deltas=None) == _rpn(os_=None) == _rpn(ob=None) == INV
    assert _rpn(batch=0) == _rpn(h=0) == _rpn(w=0) == _rpn(top_n=0) == _rpn(anchors=-1) == INV
    assert _rpn(anchors=65) == _rpn(top_n=8193) == _rpn(anchors=0) == UNS                  # limits as in the fp32 call
    assert _rpn(scores=_fake(1) + 1, top_n=8193) == INV                                    # alignment is an argument error
    # the fp32 mode checks what the untyped call checks, no more: a 2-byte-aligned float pointer gets past the checks in
    # both; the unsupported top_n stops either call before the launch
    for typed in (True, False):
        assert _rpn(dtype=L.F32, scores=_fake(1) + 2, deltas=_fake(2) + 1, top_n=8193, typed=typed) == UNS
        assert _rpn(dtype=L.F32, scores=None, typed=typed) == INV


def test_predictor_decode_argument_checks_before_the_launch():
    assert _pred(dtype=3) == _pred(dtype=-2) == INV
    assert _pred(scores=_fake(1) + 1) == _pred(deltas=_fake(2) + 1) == INV
    assert _pred(deltas=_fake(2) + 2) == _pred(deltas=_fake(2) + 4) == INV                  # 4 half deltas are one 8-byte load
    assert _pred(deltas=_fake(2) + 8, n=8193) == UNS                                        # 8-byte alignment is enough
    assert _pred(scores=_fake(1) + 2, n=8193) == UNS                                        # a half score needs 2 bytes
    assert _pred(scores=None) == _pred(props=None) == _pred(outs=(_fake(4), 0, _fake(6))) == _pred(n=0) == _pred(nc=0) == INV
    for typed in (True, False):
        assert _pred(dtype=L.F32, deltas=_fake(2) + 4, scores=_fake(1) + 2, n=8193, typed=typed) == UNS
        assert _pred(dtype=L.F32, batch=0, typed=typed) == INV


def test_python_wrappers_take_the_dtype_from_the_tensors():
    f32, f16 = torch.zeros(4), torch.zeros(4, dtype=torch.float16)
    rpn = P.RpnDecodePlugin(10, [1.0] * 4, 16.0, 80, 80, 5, 5)
    ws = torch.zeros(256, dtype=torch.uint8)
    # mixes and other dtypes are refused before any pointer is taken: these are host tensors, which _ptr would refuse with
    # another message
    with pytest.raises(L.TrtxError, match="RpnDecode scores and deltas: tensors of mixed dtypes"):
        rpn.enqueue(1, [f32, f16], [f32, f32], ws)
    with pytest.raises(L.TrtxError, match="RpnDecode scores and deltas: torch.bfloat16"):
        rpn.enqueue(1, [f32.bfloat16(), f32.bfloat16()], [f32, f32], ws)
    with pytest.raises(L.TrtxError, match="RpnDecode outputs: must be torch.float32"):
        rpn.enqueue(1, [f16, f16], [f16, f16], ws)
    with pytest.raises(L.TrtxError, match="RpnDecode outputs: tensors of mixed dtypes"):
        rpn.enqueue(1, [f32, f32], [f32, f16], ws)
    with pytest.raises(L.TrtxError, match="expected a CUDA tensor"):                          # both types get to the pointers
        rpn.enqueue(1, [f16, f16], [f32, f32], ws)
    pred = P.PredictorDecodePlugin(10, 80, 80, (10.0, 10.0, 5.0, 5.0), 4)
    with pytest.raises(L.TrtxError, match="PredictorDecode scores and deltas: tensors of mixed dtypes"):
        pred.enqueue(1, [f16, f32, f32], [f32, f32, f32], ws)
    with pytest.raises(L.TrtxError, match="PredictorDecode scores and deltas: torch.float64"):
        pred.enqueue(1, [f32.double(), f32.double(), f32], [f32, f32, f32], ws)
    with pytest.raises(L.TrtxError, match="PredictorDecode proposals: must be torch.float32"):
        pred.enqueue(1, [f16, f16, f16], [f32, f32, f32], ws)
    with pytest.raises(L.TrtxError, match="PredictorDecode outputs: tensors of mixed dtypes"):
        pred.enqueue(1, [f16, f16, f32], [f32, f32, f16], ws)
    with pytest.raises(L.TrtxError, match="PredictorDecode outputs: must be torch.float32"):
        pred.enqueue(1, [f32, f32, f32], [f16, f16, f16], ws)
    with pytest.raises(L.TrtxError, match="expected a CUDA tensor"):
        pred.enqueue(1, [f16, f16, f32], [f32, f32, f32], ws)


def _build_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda = Path(nvcc).resolve().parents[1]
    exe = tmp_path / "trt_adapter_rcnn_half_check"
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-I", str(ROOT / "include"), "-I", str(ROOT / "tests" / "mock_trt"),
           "-I", str(cuda / "include"), str(ROOT / "tests" / "trt_adapter_rcnn_half_check.cpp"), "-o", str(exe),
           str(L.LIB_PATH), f"-Wl,-rpath,{L.LIB_PATH.parent}", "-L", str(cuda / "lib64"), "-lcudart", f"-Wl,-rpath,{cuda / 'lib64'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_rcnn_half_adapters_host_surface(tmp_path):
    """Format combinations at every position, output data types, configurePlugin -> serialize -> deserialize -> clone with
    the trailing element type, the reference-length blob deserializing through the registry as fp32, wrong lengths refused."""
    r = subprocess.run([str(_build_check(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "trt adapter rcnn half check ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_rcnn_half_adapters_enqueue_on_gpu(tmp_path, dev):
    """enqueue through each adapter equals the direct typed C call, halves and floats."""
    r = subprocess.run([str(_build_check(tmp_path)), "--gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "gpu rcnn half enqueue ok" in r.stdout, r.stdout + r.stderr
