"""Outputs of the reference's own compiled code, stored for the tests that compare against it.

Where oracle/_ref/<lib> was built (oracle/Makefile compiles it from the reference sources) a test calls the reference and
compares in full.  Elsewhere it compares against tests/golden/<name>.npz, which keeps per output what the comparison needs:
a SHA-256 of the canonical bytes for a bit-exact comparison (the same verdict as comparing the arrays), the values -- or a
fixed, seeded sample of them -- for a comparison within a tolerance.  The inputs are not stored: the tests rebuild them from
seeds.  With TRTX_GOLDEN_RECORD=<dir> in the environment, a pytest run against oracle/_ref writes <dir>/<name>.npz
(ref_gpu.npz on a GPU: `pytest -m gpu tests/test_vs_reference_gpu.py tests/test_variants_gpu.py`)."""
from __future__ import annotations

import atexit
import ctypes as C
import hashlib
import os
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
REF = ROOT / "oracle" / "_ref"
GOLDEN = ROOT / "tests" / "golden"


def digest(a) -> np.ndarray:
    """SHA-256 of shape + values; NaNs by position, -0.0 == 0.0 (as np.array_equal sees them)."""
    f = np.asarray(a).astype(np.float64)
    nan = np.isnan(f)
    f = np.where(nan, 0.0, f) + 0.0
    h = hashlib.sha256(repr(f.shape).encode())
    h.update(nan.tobytes())
    h.update(np.ascontiguousarray(f).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


_RECORDS: dict = {}   # name -> outputs recorded in this process (test modules that share a file share one record)


class RefOutputs:
    def __init__(self, name: str):
        self.name = name
        p = GOLDEN / f"{name}.npz"
        self.stored = dict(np.load(p)) if p.exists() else {}
        rec = os.environ.get("TRTX_GOLDEN_RECORD")
        self.record = None
        if rec:
            if name not in _RECORDS:
                _RECORDS[name] = {}
                atexit.register(self._save, Path(rec))
            self.record = _RECORDS[name]

    def _save(self, d: Path) -> None:
        if self.record:
            d.mkdir(parents=True, exist_ok=True)
            np.savez_compressed(d / f"{self.name}.npz", **{**self.stored, **self.record})

    @staticmethod
    def lib(name: str):
        """The reference library oracle/_ref/<name>, or None where it was not built."""
        p = REF / name
        return C.CDLL(str(p)) if p.exists() else None

    def _get(self, key: str) -> np.ndarray:
        assert key in self.stored, f"{key}: no stored reference output in tests/golden/{self.name}.npz"
        return self.stored[key]

    def array(self, key: str, ref=None) -> np.ndarray:
        """A reference output stored whole, for a test that feeds it to the next stage: `ref` (live) or the stored one."""
        if ref is not None:
            ref = np.asarray(ref)
            if self.record is not None:
                self.record[key] = ref.copy()
            return ref
        return self._get(key)

    def equal(self, key: str, got, ref=None, nan_ok: bool = False, msg="") -> None:
        """got == the reference output `ref` (computed live) or the stored one, bit for bit.  A live `ref` must also match
        the stored digest, if there is one, so that a stale file fails where it can be recorded again."""
        got = np.asarray(got)
        if ref is not None:
            ref = np.asarray(ref)
            assert np.array_equal(got, ref, equal_nan=nan_ok), (key, msg)
            if self.record is not None:
                self.record[key] = digest(ref)
            elif key in self.stored:
                assert np.array_equal(digest(ref), self.stored[key]), \
                    f"{key}: the reference's output differs from tests/golden/{self.name}.npz {msg}"
            return
        assert nan_ok or not np.isnan(got.astype(np.float64)).any(), (key, msg)
        assert np.array_equal(digest(got), self._get(key)), f"{key}: differs from the reference's output {msg}"

    def close(self, key: str, got, ref=None, rtol: float = 1e-7, atol: float = 0.0, sample: int = 512, msg="") -> None:
        """got within (rtol, atol) of the reference output; the stored form keeps `sample` seeded elements of a larger one."""
        got = np.asarray(got)
        if ref is not None:
            ref = np.asarray(ref)
            np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol, err_msg=f"{key} {msg}")
            if self.record is not None:
                idx = np.arange(ref.size)
                if ref.size > sample:
                    idx = np.sort(np.random.default_rng(0).choice(ref.size, sample, replace=False))
                self.record[key] = ref.reshape(-1)[idx].copy()
                self.record[key + "#idx"] = idx.astype(np.int32)
                self.record[key + "#shape"] = np.asarray(ref.shape, np.int64)
            return
        assert tuple(got.shape) == tuple(self._get(key + "#shape")), (key, got.shape)
        idx = self._get(key + "#idx")
        np.testing.assert_allclose(got.reshape(-1)[idx], self._get(key), rtol=rtol, atol=atol, err_msg=f"{key} {msg}")
