"""Host-side logic that needs no GPU: the C-ABI library loads and exports every declared symbol,
plugin (de)serialization keeps the reference's byte layout, parameter validation, the letterbox
matrix of the library equals the oracle's (and therefore cv2's), and the N>1 gather path under gloo."""
import ctypes as C
import os
import re
import struct
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    from tensorrtx_b200 import _lib as L

    lib = L.load()
    hdr = (ROOT / "include" / "trtx_hot.h").read_text()
    declared = set(re.findall(r"TRTX_API\s+[\w\s\*]+?\b(trtx_\w+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(L.SYMBOLS), declared ^ set(L.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.trtx_version()
    out = subprocess.run(["nm", "-D", "--defined-only", str(L.LIB_PATH)], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    # exactly the declared C ABI is exported: no C++ symbols, no undeclared tuning / profiling hooks
    assert declared == exported, declared ^ exported


def test_no_mutable_globals_and_struct_sizes_match_the_binding():
    """SURVEY 8b "Threading": enqueue must not depend on process-global mutable state.  The launch tuning lives in
    trtx_yolo_params (per call); the only writable data of the library is the thread-local last-error slot and lazily
    resolved driver entry points.  Also: the ctypes mirrors have the size the library was compiled with."""
    import ctypes as C

    from tensorrtx_b200 import _lib as L

    lib = L.load()
    for which, st in enumerate((L.YoloParams, L.NmsParams, L.RetinaParams, L.ImageDesc, L.MaskParams)):
        assert lib.trtx_abi_sizeof(which) == C.sizeof(st), st.__name__
    assert lib.trtx_abi_sizeof(99) == 0
    out = subprocess.run(["nm", "-C", "--defined-only", str(L.LIB_PATH)], capture_output=True, text=True).stdout
    writable = [l.split(maxsplit=2)[2] for l in out.splitlines()
                if len(l.split(maxsplit=2)) == 3 and l.split()[1] in ("b", "B", "d", "D") and "trtx::" in l]
    # thread-local error slot; function-local static holding the driver entry point of cuTensorMapEncodeTiled
    allowed = ("g_last_cuda_error", "tma_encoder", "guard variable")
    assert all(any(a in w for a in allowed) for w in writable), writable


def test_no_torch_types_in_abi():
    hdr = (ROOT / "include" / "trtx_hot.h").read_text()
    assert "torch" not in hdr.lower() and "at::" not in hdr and "#include <cuda" not in hdr


def test_yolo_plugin_serialization_layout_v8():
    from tensorrtx_b200 import plugins as P

    p = P.YoloLayerPlugin(80, 17, 0.0, 640, 640, 1000, False, True, False, (8, 16, 32))
    blob = p.serialize()
    # yololayer.cu:75-95: classCount, nKpt, kptThr(float), threadCount, W, H, maxOut, nStrides, strides..., 3 bools
    assert len(blob) == p.getSerializationSize() == 4 * 8 + 12 + 3
    assert struct.unpack_from("<ii", blob, 0) == (80, 17)
    assert struct.unpack_from("<i", blob, 12)[0] == 256
    assert struct.unpack_from("<iii", blob, 32) == (8, 16, 32)
    assert blob[-3:] == b"\x00\x01\x00"
    q = P.YoloLayerPlugin.deserialize(blob)
    assert q.serialize() == blob and q.is_pose_ and q.mStrides == [8, 16, 32]
    with pytest.raises(Exception):
        P.YoloLayerPlugin.deserialize(blob + b"\0")
    c = p.clone()
    assert c.serialize() == blob and c is not p
    assert p.getOutputDimensions() == (1000 * 90 + 1, 1, 1)
    assert p.getPluginType() == "YoloLayer_TRT" and p.getPluginVersion() == "1"
    assert p.getWorkspaceSize(32) > 0


def test_yolo_creator_fields():
    from tensorrtx_b200 import plugins as P

    cr = P.YoloPluginCreator()
    cr.setPluginNamespace("ns")
    # combinedInfo of yolov8/src/block.cpp:264-296
    ci = [80, 17, 0, 640, 640, 1000, 0, 0, 0, 8, 16, 32]
    p = cr.createPlugin("yololayer", {"combinedInfo": ci})
    assert p.mClassCount == 80 and p.mStrides == [8, 16, 32] and p.getPluginNamespace() == "ns"
    assert cr.deserializePlugin("yololayer", p.serialize()).serialize() == p.serialize()
    with pytest.raises(Exception):
        cr.createPlugin("yololayer", {"netinfo": ci})


def test_yolo_v5_serialization_layout():
    from tensorrtx_b200 import plugins as P
    from tensorrtx_b200 import synth

    ks = [P.YoloKernel(640 // s, 640 // s, a) for s, a in zip((8, 16, 32), synth.V5_ANCHORS)]
    p = P.YoloLayerPluginV5(80, 640, 640, 1000, False, ks)
    blob = p.serialize()
    assert len(blob) == p.getSerializationSize() == 25 + 3 * 32   # yolov5 yololayer.cu:48-83
    q = P.YoloLayerPluginV5.deserialize(blob)
    assert q.serialize() == blob
    assert [k.anchors for k in q.mYoloKernel] == [list(map(float, a)) for a in synth.V5_ANCHORS]


def test_param_validation_returns_error_codes_without_gpu():
    from tensorrtx_b200 import _lib as L

    lib = L.load()
    p = L.YoloParams()
    assert lib.trtx_yolo_workspace_size(C.byref(p), 1) == 0          # zeroed params are invalid
    strides = (C.c_int * 3)(8, 16, 32)
    assert lib.trtx_yolo_params_init_v8(C.byref(p), 80, 640, 640, 1000, strides, 3) == L.OK
    assert list(p.grid_w[:3]) == [80, 40, 20] and p.det_floats == 90
    assert lib.trtx_yolo_params_init_v8(C.byref(p), 80, 640, 640, 1000, strides, 9) == L.ERR_INVALID
    assert lib.trtx_yolo_workspace_size(C.byref(p), 32) >= 32 * 8400 * 32
    # null device pointers are rejected before any CUDA call
    assert lib.trtx_yolo_decode_enqueue(C.byref(p), 1, None, None, None, 0, None) == L.ERR_INVALID
    q = L.NmsParams()
    q.max_det = 0
    assert lib.trtx_nms_workspace_size(C.byref(q), 1, 1000) == 0
    r = L.RetinaParams()
    r.in_h, r.in_w = 640, 640
    assert lib.trtx_retina_total_priors(C.byref(r)) == 16800


def test_library_letterbox_matrix_equals_oracle(oracle):
    from tensorrtx_b200 import plugins as P

    rng = np.random.default_rng(1)
    for _ in range(300):
        sw, sh = (int(v) for v in rng.integers(40, 4000, 2))
        assert np.array_equal(np.asarray(P.letterbox_matrix(sw, sh, 640, 640), np.float32),
                              oracle.letterbox_matrix(sw, sh, 640, 640))


def test_threshold_rounding_for_double_literals():
    from tensorrtx_b200.plugins import float_le_threshold

    for lit in (0.1, 0.02, 0.5, 0.45):
        t = np.float32(float_le_threshold(lit))
        assert float(t) <= lit < float(np.nextafter(t, np.float32(np.inf)))


def test_missing_library_raises(monkeypatch, tmp_path):
    from tensorrtx_b200 import _lib as L

    monkeypatch.setattr(L, "_lib", None)
    monkeypatch.setattr(L, "LIB_PATH", tmp_path / "nope.so")
    with pytest.raises(L.TrtxError):
        L.load()


_GLOO_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TRTX_ROOT"])
from tensorrtx_b200.pipeline import gather
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
B, K = 4, 10
local = torch.full((B, 1 + K * 7), float(rank)) + torch.arange(B)[:, None]
out = gather(local, world)
assert out.shape == (world * B, 1 + K * 7)
for r in range(world):
    assert torch.equal(out[r * B:(r + 1) * B], torch.full((B, 1 + K * 7), float(r)) + torch.arange(B)[:, None])
# batch sharding: rank r owns images [B*r, B*(r+1)) of the global batch
# the pipelined form used by bench.py (side stream on CUDA, synchronous on a CPU group): several steps, rotating slots
from tensorrtx_b200.pipeline import GatherRing
ring = GatherRing(world, B, 1 + K * 7, "cpu", slots=2)
for step in range(5):
    ring.reuse(step % 2)
    src = local + 100.0 * step
    got = ring.launch(src, step % 2)
    ring.join()
    for r in range(world):
        assert torch.equal(got[r * B:(r + 1) * B], torch.full((B, 1 + K * 7), float(r)) + torch.arange(B)[:, None] + 100.0 * step)
dist.barrier(); dist.destroy_process_group(); print("ok", rank)
"""


def test_gather_world_size_2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER)
    env = dict(os.environ, TRTX_ROOT=str(ROOT), MASTER_ADDR="127.0.0.1", MASTER_PORT="29631", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert all("ok" in o for o in outs)


def test_bench_reference_arm_prints_contract_json():
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    import json

    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "frames/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"].split()[0] in ("port", "reference") and line["e2e"]["h2d_bytes_per_step"] == 0
    # both arms print the same config dict (the driver's same_config check)
    sys.path.insert(0, str(ROOT))
    import bench
    assert line["config"] == bench.config_dict("v8n_b32", 1)
    assert line["config"]["stages"] == "pre-process + decode + NMS"


@pytest.mark.parametrize("config", ["v5s_b1", "retina_b16", "rcnn_b8"])
def test_bench_reference_arm_other_configs(config):
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--config", config, "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    import json

    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["value"] > 0 and line["config"]["config"] == config


def test_division_free_overlap_test_is_exact(tmp_path):
    """nms.cu decides `iou > thresh` from the sign of fma(-thresh, denom, inter) unless the quotient is within 1e-5 of the
    threshold: tools/verify_overlap_test.c replays that rule on random and adversarial (few-ulp) operands against the
    IEEE division; zero disagreements (3.2e9 cases in the full run, a bounded sample here)."""
    exe = tmp_path / "verify_overlap"
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-o", str(exe), str(ROOT / "tools" / "verify_overlap_test.c"),
                        "-lm"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "2000000"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches=0" in r.stdout, r.stdout


def test_logit_domain_class_loop_equals_reference_loop(tmp_path):
    """The scan kernels keep the reference's class loop in the logit domain (running max logit, first argmax, max before
    it, slice merge, group-max gate, one sigmoid, collision replay): tools/verify_logit_domain.c runs that algorithm in C
    next to the reference loop on noise + planted near-ulp pairs, ties, saturating, non-finite and underflowing logits
    for every gate / slice / group-size combination; zero mismatches (2e8 cases in the full run, a bounded sample here)."""
    exe = tmp_path / "verify_logit"
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-o", str(exe), str(ROOT / "tools" / "verify_logit_domain.c"),
                        "-lm"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "150000"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches=0" in r.stdout, r.stdout
    assert "collision_replays=0 " not in r.stdout   # the replay path is exercised


def test_nms_bitmap_phase_equals_greedy(tmp_path):
    """nms_kernel phase E (closed-form work-unit layout, one bitmap byte per unit, chunked ballot resolve) replayed in C for
    random class segments of every length 1..96 against plain greedy NMS: tools/verify_nms_bitmap.c."""
    exe = tmp_path / "verify_nms"
    r = subprocess.run(["gcc", "-O2", "-fopenmp", "-o", str(exe), str(ROOT / "tools" / "verify_nms_bitmap.c")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "20000"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches=0" in r.stdout, r.stdout


def test_abi_header_is_plain_c(tmp_path):
    """include/trtx_hot.h is the FFI boundary (cgo / JNI / ctypes bind it): it must compile as C99 without extensions."""
    src = tmp_path / "hdr.c"
    src.write_text('#include "trtx_hot.h"\nint main(void) { trtx_nms_params q; trtx_mask_params m; (void)q; (void)m; return 0; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", str(ROOT / "include"), "-fsyntax-only",
                        str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr



def test_committed_scan_traffic_summary_matches_what_bench_reads():
    """profiles/scan_traffic.json feeds `roofline.traffic`: either it describes the CURRENT scan-kernel sources with the keys
    bench.py prints, or bench.scan_traffic() returns None (never a KeyError in the middle of the JSON line)."""
    import importlib.util
    import json

    spec = importlib.util.spec_from_file_location("bench_mod", ROOT / "bench.py")
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    t = bench.scan_traffic()
    f = ROOT / "profiles" / "scan_traffic.json"
    if f.exists():
        j = json.loads(f.read_text())
        for k in ("dram_bytes_per_launch", "capture", "src_sha256"):
            assert k in j, k
    if t is not None:
        assert 0.9 * 90316800 < t["dram_bytes_per_launch"] < 1.3 * 90316800      # every head byte read once (SURVEY 8d)
        assert isinstance(t["capture"], str)


def test_roi_align_window_kernel_arithmetic_shortcuts_are_exact(tmp_path):
    """Two shortcuts of roi_align_window_kernel (tensorrtx_b200/csrc/roi_align.cu) that must not change a bit:
    (1) `output_val * (1 / count)` instead of `output_val / count` (rcnn/RoiAlign.cu:147) when the sample count is a power of
        two -- tools/verify_pow2_div.c over every float bit pattern (full run: 3.9e10 pairs, 0 mismatches; a strided one here);
    (2) window row of a cell by multiplication: (cell * ceil(2^16 / ww)) >> 16 == cell / ww whenever cells * ww <= 2^16
        (the kernel divides otherwise), with the product inside 32 bits for the <= 4096 cells a window can hold."""
    exe = tmp_path / "verify_pow2_div"
    r = subprocess.run(["gcc", "-O2", "-o", str(exe), str(ROOT / "tools" / "verify_pow2_div.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "1021"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and " 0 mismatches" in r.stdout, r.stdout
    for ww in range(1, 4097):
        m = (65536 + ww - 1) // ww
        cmax = min(65536 // ww, 4096)
        cell = np.arange(cmax, dtype=np.int64)
        assert cmax * m < 2 ** 32
        assert np.array_equal((cell * m) >> 16, cell // ww), ww
    src = (ROOT / "tensorrtx_b200" / "csrc" / "roi_align.cu").read_text()
    assert "cells * ww <= 65536 ? (cell * m_ww) >> 16 : cell / ww" in src and "kRoiWindowFloats / 4" in src


def test_gather_ring_schedule_never_overwrites_an_unread_slot_group():
    """bench.py's multi-GPU step (DESIGN.md section 5): replay k of a rank PUBLISHES group k-1 into slot group k mod 2D of every
    rank and WAITS for every rank's publish of group k-D (D = --gather-depth; D = 1: the group just published); consumers of a
    group run in the replay that waited for it.  Claim: with a ring of 2D slot groups no rank ever overwrites a slot group a
    peer has not finished reading, whatever the ranks' relative speeds.  Event-driven replay of the schedule with random
    per-replay durations (a wait blocks until the peers' publishes exist); the publish of replay k lands at the replay's start,
    the read of the awaited group lasts until the replay's end."""
    rng = np.random.default_rng(7)
    for D in (1, 2, 3):
        NG = 2 * D
        for world in (2, 3, 8):
            for trial in range(20):
                n_replays = 60
                dur = rng.uniform(0.2, 3.0, (world, n_replays)) * rng.uniform(0.5, 2.0, (world, 1))  # some ranks are slower overall
                start = np.zeros((world, n_replays)); end = np.zeros((world, n_replays))
                pub = np.full((world, n_replays), np.inf)   # time at which rank r published group g (g = replay index - 1)
                # iterate to the fixed point of the dependency graph (replay k of r starts after replay k-1 of r ended; it ends
                # after its own work AND after every peer has published group k-D, i.e. started replay k-D+1)
                for k in range(n_replays):
                    for r in range(world):
                        start[r, k] = end[r, k - 1] if k else 0.0
                        if k >= 1:
                            pub[r, k - 1] = start[r, k]                     # group k-1 published at the start of replay k
                    for r in range(world):
                        need = k - D
                        t_wait = max(pub[p, need] for p in range(world)) if need >= 0 else 0.0
                        assert np.isfinite(t_wait), "a wait for a group that nobody can have published yet: deadlock"
                        end[r, k] = max(start[r, k] + dur[r, k], t_wait)
                # safety: group g occupies slot group (g+1) mod NG on every rank from pub[., g] on; it is overwritten by group
                # g + NG, published by rank p at pub[p, g + NG]; rank q reads group g during the replay that waited for it
                # (replay g + D), i.e. until end[q, g + D]
                for g in range(n_replays - NG - 1):
                    for p in range(world):
                        for q in range(world):
                            assert pub[p, g + NG] >= end[q, g + D] - 1e-12, (D, world, trial, g, p, q)


def test_no_undefined_global_names_in_bench_and_package():
    """bench.py's GPU legs cannot run here; at least every global name its functions (and the package's) load must exist --
    a cheap guard against a typo that would only surface at the end of a GPU run."""
    import builtins
    import dis
    import importlib.util
    import types

    for rel in ("bench.py", "__graft_entry__.py", "tensorrtx_b200/pipeline.py", "tensorrtx_b200/plugins.py", "tensorrtx_b200/_lib.py",
                "tensorrtx_b200/synth.py", "tensorrtx_b200/build.py"):
        path = ROOT / rel
        name = "chk_" + rel.replace("/", "_").replace(".py", "")
        if rel.startswith("tensorrtx_b200/"):
            name = "tensorrtx_b200." + name      # relative imports of the package modules resolve
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        try:
            spec.loader.exec_module(mod)
            missing, stored = set(), set()

            def walk(co):
                for ins in dis.get_instructions(co):
                    if ins.opname in ("STORE_NAME", "STORE_GLOBAL"):
                        stored.add(ins.argval)        # e.g. an import under `if __name__ == "__main__":`
                    if ins.opname in ("LOAD_GLOBAL", "LOAD_NAME") and isinstance(ins.argval, str):
                        if not hasattr(mod, ins.argval) and not hasattr(builtins, ins.argval):
                            missing.add((co.co_name, ins.argval))
                for c in co.co_consts:
                    if isinstance(c, types.CodeType):
                        walk(c)
            walk(compile(path.read_text(), str(path), "exec"))
            missing = {m for m in missing if m[1] not in stored}
            assert not missing, (rel, sorted(missing))
        finally:
            sys.modules.pop(name, None)


def test_all_gpu_sampler_summary_is_robust():
    """bench.py's AllGpuSampler (N > 1: every GPU's clocks / temperatures during the timed blocks) must never raise: malformed
    lines, [N/A] fields, samples outside the windows, no nvidia-smi at all."""
    import importlib.util
    import time

    spec = importlib.util.spec_from_file_location("bench_mod2", ROOT / "bench.py")
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.AllGpuSampler()
    now = time.time()
    s.lines = [(now, "0, 1965, 3996, 55, 62, 810.5, 0x0"), (now, "1, 1965, 3996, 61, 70, 820.1, 0x4"), (now, "1, [N/A], 3996, 63, 71, 825.1, 0x4"),
               (now - 100, "2, 1, 1, 1, 1, 1, x"), (now, "garbage"), (now, "")]
    out = s.summary([(now - 1, now + 1)])
    assert [g["gpu"] for g in out] == [0, 1] and out[1]["samples"] == 2 and out[1]["hbm_temp_c"] == 71.0 and out[1]["sm_mhz"] == 1965.0
    assert s.summary([]) is None and bench.AllGpuSampler().summary([(0, 1)]) is None
    s2 = bench.AllGpuSampler()
    s2.start()          # no nvidia-smi on the build container: must not raise
    s2.stop()
