"""Shared GPU test scaffolding: the library's environment knobs and their reset, the catalogue of spectrum kernel
routes, and bit-equality and CUDA graph helpers."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import pytest

# Every environment knob the library reads (waveform_b200/csrc; test_knobs_cpu.py holds this list to the sources).  Each
# is an A/B switch read when an engine is created, so one left in the caller's shell would change what a test exercises.
KNOBS = ("WF_FORCE_GENERIC", "WF_V3", "WF_WIDE_R", "WF_TEAM_W", "WF_PAR16384", "WF_WARP2", "WF_WARP2_DISPLAY",
         "WF_SPLIT", "WF_ZERO_COPY", "WF_METER_FUSED", "WF_WAVE_CHUNK")


def set_knobs(monkeypatch, env):
    """Clears every knob, then sets env ({name: value}) for the engines created after this call."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.fixture
def clean_knobs(monkeypatch):
    """The test's engines see no knob unless the test sets it through set_knobs."""
    set_knobs(monkeypatch, {})


# ---- the spectrum kernel routes --------------------------------------------------------------------------------------

FAMILIES = ["stft2048_fast_kernel", "stft2048_team_kernel", "stft_warp2_kernel", "stft_warp2_kernel/display",
            "stft_v3_kernel", "stft16384_parity_kernel", "stft_wide_kernel", "stft_fused_kernel",
            "stft_anyn_kernel/smem", "stft_anyn_kernel/L2"]


class Route(NamedTuple):
    """A call that reaches one kernel family: the family (the kernel's name, with a '/' note on the variant), fft_size,
    capture channels, stereo channel mode, the knobs it needs and whether it asks for display outputs."""
    family: str
    N: int
    cc: int
    stereo: bool
    env: dict
    display: bool


FAST, TEAM, WARP2, V3 = "stft2048_fast_kernel", "stft2048_team_kernel", "stft_warp2_kernel", "stft_v3_kernel"
PARITY, WIDE, FUSED = "stft16384_parity_kernel", "stft_wide_kernel", "stft_fused_kernel"
SMEM, L2 = "stft_anyn_kernel/smem", "stft_anyn_kernel/L2"

# name -> route.  Names ending in "-display" ask for display outputs.
CATALOGUE = {
    "fast-2048": Route(FAST, 2048, 1, False, {"WF_TEAM_W": "1"}, False),
    "fast-2048-split": Route(FAST + "/split", 2048, 1, False, {"WF_TEAM_W": "1"}, False),  # more streams than SMs
    "team-2048": Route(TEAM, 2048, 1, False, {"WF_TEAM_W": "4"}, False),
    **{f"warp2-{n}": Route(WARP2, n, 1, False, {}, False) for n in (800, 1456, 1664, 1408, 1792)},
    **{f"warp2-{n}-display": Route(WARP2 + "/display", n, 1, False, {}, True) for n in (800, 1456, 1024, 2048)},
    "v3-1024": Route(V3, 1024, 1, False, {}, False),
    "v3-1024-stereo-display": Route(V3, 1024, 2, True, {}, True),
    "v3-2048-generic": Route(V3, 2048, 1, False, {"WF_FORCE_GENERIC": "1"}, False),
    "v3-4096-stereo": Route(V3, 4096, 2, True, {}, False),
    "v3-4096-stereo-display": Route(V3, 4096, 2, True, {}, True),
    "v3-4096-mix": Route(V3, 4096, 2, False, {}, False),
    "v3-4096-mix-display": Route(V3, 4096, 2, False, {}, True),
    "v3-8192": Route(V3, 8192, 1, False, {}, False),
    "v3-16384": Route(V3, 16384, 1, False, {"WF_PAR16384": "0"}, False),
    "parity-16384": Route(PARITY, 16384, 1, False, {}, False),
    "wide-4096": Route(WIDE, 4096, 1, False, {"WF_V3": "0", "WF_WIDE_R": "2"}, False),
    "wide-4096-display": Route(WIDE, 4096, 1, False, {"WF_V3": "0", "WF_WIDE_R": "2"}, True),
    "wide-4096-stereo-display": Route(WIDE, 4096, 2, True, {"WF_V3": "0"}, True),
    "wide-8192-display": Route(WIDE, 8192, 1, False, {"WF_V3": "0"}, True),
    "wide-32768": Route(WIDE, 32768, 1, False, {"WF_WIDE_R": "2"}, False),
    **{f"fused-{n}": Route(FUSED, n, 1, False, {}, False) for n in (128, 256, 512)},
    "fused-256-display": Route(FUSED, 256, 1, False, {}, True),
    "fused-512-display": Route(FUSED, 512, 1, False, {"WF_V3": "0", "WF_WIDE_R": "1", "WF_WARP2_DISPLAY": "0"}, True),
    "fused-2048": Route(FUSED, 2048, 1, False, {"WF_FORCE_GENERIC": "1", "WF_V3": "0", "WF_WIDE_R": "1"}, False),
    "fused-2048-mix": Route(FUSED, 2048, 2, False, {"WF_FORCE_GENERIC": "1", "WF_V3": "0", "WF_WIDE_R": "1"}, False),
    "fused-2048-stereo-display": Route(FUSED, 2048, 2, True, {"WF_V3": "0", "WF_WIDE_R": "1"}, True),
    "fused-32768": Route(FUSED, 32768, 1, False, {"WF_WIDE_R": "1"}, False),
    **{f"smem-{n}": Route(SMEM, n, 1, False, {"WF_WARP2": "0"}, False) for n in (800, 1456, 1664)},
    "smem-800-display": Route(SMEM, 800, 1, False, {"WF_WARP2": "0"}, True),
    "smem-800-stereo-display": Route(SMEM, 800, 2, True, {}, True),
    "smem-1456-display": Route(SMEM, 1456, 1, False, {"WF_WARP2": "0"}, True),
    "smem-8128": Route(SMEM, 8128, 1, False, {}, False),
    **{f"l2-{n}": Route(L2, n, 1, False, {}, False) for n in (40000, 65344, 65488, 65536)},
    "l2-65536-stereo-display": Route(L2, 65536, 2, True, {}, True),
}


def route_id(r):
    """The test id of a route, or of a tuple that starts with one's family, N, channels and stereo flag."""
    fam, N, cc, stereo = r[:4]
    return f"{fam.replace('/', '-')}-{N}{'-stereo' if stereo else ('-mix' if cc == 2 else '')}"


# ---- bit equality and graphs -----------------------------------------------------------------------------------------

def _numpy(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def to_host(out):
    """A dict of outputs (tensors on any device, or numpy) as numpy arrays; entries that are None are left out."""
    return {k: _numpy(v) for k, v in out.items() if v is not None}


def bits(a):
    """The bytes of an array or tensor, as a flat uint8 array."""
    return np.ascontiguousarray(_numpy(a)).view(np.uint8).reshape(-1)


def assert_bits_equal(got, want, what):
    """got and want are the same bit for bit: numpy arrays or tensors with the same shape, dtype and bytes, or dicts of
    them with the same keys (None entries left out)."""
    if isinstance(want, dict):
        got, want = to_host(got), to_host(want)
        assert got.keys() == want.keys(), (what, sorted(got), sorted(want))
        for k in want:
            assert_bits_equal(got[k], want[k], (what, k))
        return
    g, w = _numpy(got), _numpy(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, g.dtype, w.shape, w.dtype)
    bad = np.flatnonzero((bits(g) != bits(w)).reshape(-1, g.itemsize).any(axis=1))
    assert bad.size == 0, (what, bad.size, bad[:8])


def capture(fn):
    """fn() captured into a CUDA graph under torch's default (global) capture mode; returns the graph and what fn
    returned."""
    import torch

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def replay(g, inputs, values):
    """Writes fresh values (numpy) into the captured input buffers, replays the graph and waits for it."""
    import torch

    for buf, v in zip(inputs, values):
        buf.copy_(torch.from_numpy(v).cuda())
    g.replay()
    torch.cuda.synchronize()
