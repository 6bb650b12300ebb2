"""What the unmodified reference computed, stored so that the comparisons against it run without it.

The tests that pin the oracle (and the live host adapter) to the reference reduce the reference's outputs to what the
comparison needs: a SHA-256 digest for an output that must match bit for bit, a fixed sample for one compared within a
tolerance.  `reference(key, compute)` returns that reduced record from tests/golden/reference_outputs.npz.  With
WF_RECORD_REFERENCE=1 and the reference built (WF_REFERENCE_DIR=<checkout> python __graft_entry__.py), it calls
`compute()` against the live reference instead and rewrites the store when the session ends:

    WF_RECORD_REFERENCE=1 python -m pytest tests -m "not gpu" -k reference      # then the GPU tests that use it
"""
from __future__ import annotations

import atexit
import hashlib
import json
import os
from pathlib import Path

import numpy as np

STORE = Path(__file__).resolve().parent / "golden" / "reference_outputs.npz"
RECORDING = os.environ.get("WF_RECORD_REFERENCE") == "1"

_loaded: dict | None = None
_recorded: dict = {}


def digest(a) -> np.ndarray:
    """SHA-256 of an array's dtype, shape and bytes (an absent output digests to an empty array)."""
    if a is None:
        return np.zeros(0, dtype=np.uint8)
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


def sample_index(shape, n: int, seed: int) -> np.ndarray:
    """n sorted positions along the last axis of `shape` (first and last included), the same on every run."""
    size = shape[-1]
    if size <= n:
        return np.arange(size)
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([[0, size - 1], rng.choice(size, n - 2, replace=False)]))


def frame_peak(db, db_min):
    """Linear peak of every frame of a dB spectrum, floor bins excluded (the frame_peak of helpers.parity_report)."""
    db = np.asarray(db, dtype=np.float64)
    lin = np.where(db <= db_min + 1.0, 0.0, np.power(10.0, db / 20.0))
    return np.maximum(lin.max(axis=-1, keepdims=True), 1e-300)


def reference(key: str, compute) -> dict:
    """The stored record `key`; compute() -> dict of arrays runs against the live reference when recording."""
    global _loaded
    if RECORDING:
        rec = {k: np.asarray(v) for k, v in compute().items()}
        if not _recorded:
            atexit.register(_save)
        _recorded[key] = rec
        return rec
    if _loaded is None:
        _loaded = _load()
    assert key in _loaded, f"{key}: not in {STORE.name}; record it with WF_RECORD_REFERENCE=1 against the reference"
    return _loaded[key]


def _load() -> dict:
    """The store is one JSON index (key -> field -> dtype, shape, offset) and one byte blob, compressed."""
    with np.load(STORE, allow_pickle=False) as z:
        index, blob = json.loads(z["index"].tobytes()), z["data"]
    out = {}
    for key, fields in index.items():
        out[key] = {f: blob[o: o + int(np.prod(shape, dtype=np.int64)) * np.dtype(dt).itemsize].view(dt).reshape(tuple(shape))
                    for f, (dt, shape, o) in fields.items()}
    return out


def _save():
    recs = _load() if STORE.exists() else {}
    recs.update(_recorded)
    index, parts, off = {}, [], 0
    for key in sorted(recs):
        index[key] = {}
        for f, v in sorted(recs[key].items()):
            v = np.asarray(v)
            index[key][f] = (v.dtype.str, list(v.shape), off)
            parts.append(v.tobytes())
            off += v.nbytes
    np.savez_compressed(STORE, index=np.frombuffer(json.dumps(index).encode(), dtype=np.uint8),
                        data=np.frombuffer(b"".join(parts), dtype=np.uint8))
