"""Which spectrum kernel every kind of call runs, against a recorded table (tests/golden/routes_h100.json).

Each case below flips one routing condition of wf_engine.cu: size, channels, stereo, display outputs, the options that
select a kernel's EXTRA variant, pcm / out_db / hop alignment, stream and tick counts, host or device buffers, and the
environment knobs.  For every call the test compares the exact last_kernel_name() (template arguments and grid
included) and the number of launches the call made (materialize_hold_kernel and the out_peak fill count too) with the
table.  Only the routing is under test, so the data are zeros and small.

Grids are min(streams, SM count) and stream counts scale with the SM count, so the table holds for the GPU model it was
recorded on; on a device with another SM count the test skips.  To record the table, on the GPU it is meant for:

    WF_RECORD_ROUTES=1 python -m pytest tests/test_gpu_routes.py -m gpu -q
"""
from __future__ import annotations

import atexit
import ctypes as C
import json
import os
from pathlib import Path

import numpy as np
import pytest

from gpu_common import clean_knobs, set_knobs  # noqa: F401 (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

STORE = Path(__file__).resolve().parent / "golden" / "routes_h100.json"
RECORDING = os.environ.get("WF_RECORD_ROUTES") == "1"

OPT = {"fast_peaks": True}                      # an option that selects a kernel's EXTRA variant and needs no input
LANCZOS = {"interp_mode": "lanczos"}


def call(**kw):
    """One process call: hop (default N), pcm_off / db_off (floats), outputs (db, silent, points, pixels, peak) and the
    kind of buffers ("device", "host": numpy, "mapped": wf_host_alloc); {"get_state": True} is a get_state() call."""
    return kw


# id -> (N, settings, channels, environment, streams, ticks, calls); streams (k, a) means k x SM count + a
CASES = {
    # the N=2048 warp-per-stream kernel and its template variants <MAXW, TSM, GATE, EXTRA>
    "fast-many-streams": (2048, {}, 1, {}, (9, 1), 2, [call()]),
    **{f"fast-tsm{t}-gate{g}-x{x}": (2048, {"temporal_smoothing": "exp_moving_avg" if t else "none", "silence_gate": g,
                                            **(OPT if x else {})}, 1, {}, 1, 1, [call()])
       for t in (0, 1) for g in (0, 1) for x in (0, 1)},
    "fast-peak-output": (2048, {}, 1, {}, 1, 1, [call(peak=True)]),
    "fast-split0": (2048, {}, 1, {"WF_SPLIT": "0"}, (9, 1), 2, [call()]),
    "fast-team-w1": (2048, {}, 1, {"WF_TEAM_W": "1"}, (1, 0), 16, [call()]),
    # what keeps a call off the N=2048 kernels
    "fast-no-pcm-offset": (2048, {}, 1, {}, 2, 2, [call(pcm_off=1)]),
    "fast-no-hop": (2048, {}, 1, {}, 2, 2, [call(hop=2046)]),
    "fast-no-db-offset": (2048, {}, 1, {}, 2, 2, [call(db_off=1)]),
    "fast-no-mix": (2048, {}, 2, {}, 2, 2, [call()]),
    "fast-no-stereo": (2048, {"channel_mode": "stereo"}, 2, {}, 2, 2, [call()]),
    "fast-no-display": (2048, {}, 1, {}, 2, 2, [call(points=True)]),
    "fast-no-db": (2048, {}, 1, {}, 2, 2, [call(db=False)]),
    "fast-no-generic": (2048, {}, 1, {"WF_FORCE_GENERIC": "1"}, 2, 2, [call()]),
    # teams of W warps per stream
    "team-1-per-sm": (2048, {}, 1, {}, (1, 0), 16, [call()]),
    "team-2-per-sm": (2048, {}, 1, {}, (2, 0), 16, [call()]),
    "team-5-per-sm": (2048, {}, 1, {}, (5, 0), 16, [call()]),
    "team-opt": (2048, OPT, 1, {}, (1, 0), 16, [call()]),
    "team-t4": (2048, {}, 1, {}, (1, 0), 4, [call()]),
    "team-t2": (2048, {}, 1, {}, (1, 0), 2, [call()]),
    "team-w8": (2048, {}, 1, {"WF_TEAM_W": "8"}, (9, 1), 8, [call()]),
    # N=16384 parity clusters
    "parity": (16384, {}, 1, {}, 2, 2, [call()]),
    "parity-opt": (16384, OPT, 1, {}, 2, 2, [call()]),
    "parity-off": (16384, {}, 1, {"WF_PAR16384": "0"}, 2, 2, [call()]),
    "parity-v3-off": (16384, {}, 1, {"WF_V3": "0"}, 2, 2, [call()]),
    "parity-display": (16384, {}, 1, {}, 2, 2, [call(points=True)]),
    # warp-per-stream plans N = 2*L*P, plain and with display outputs
    "warp2-800": (800, {}, 1, {}, 2, 2, [call()]),
    "warp2-800-opt": (800, OPT, 1, {}, 2, 2, [call()]),
    "warp2-800-many-streams": (800, {}, 1, {}, (9, 1), 2, [call()]),
    **{f"warp2-display-{n}": (n, {}, 1, {}, 2, 2, [call(points=True)]) for n in (800, 1024, 2048)},
    "warp2-display-pixels": (800, OPT, 1, {}, 2, 2, [call(points=True, pixels=True)]),
    "warp2-display-bars": (1024, {"display_mode": "bars"}, 1, {}, 2, 2, [call(points=True)]),
    "warp2-off": (800, {}, 1, {"WF_WARP2": "0"}, 2, 2, [call()]),
    "warp2-display-off": (1024, {}, 1, {"WF_WARP2_DISPLAY": "0"}, 2, 2, [call(points=True)]),
    "warp2-display-generic": (1024, {}, 1, {"WF_FORCE_GENERIC": "1"}, 2, 2, [call(points=True)]),
    "warp2-mix": (800, {}, 2, {}, 2, 2, [call()]),
    "warp2-pcm-offset": (800, {}, 1, {}, 2, 2, [call(pcm_off=1)]),
    "warp2-no-db": (800, {}, 1, {}, 2, 2, [call(db=False)]),
    # display areas too large for all 16 warps, or for one warp (then the call falls through to the next family)
    **{f"warp2-curve-{w}": (2048, {"width": w, **LANCZOS}, 1, {}, 2, 2, [call(points=True, pixels=True)])
       for w in (1500, 3000, 6000, 12000)},
    # CTA-per-tick clusters: sizes, channels, R from the stream count, EXTRA 0 / 1 (out_peak only) / 3
    **{f"v3-{n}-{m}": (n, {"channel_mode": "stereo"} if m == "stereo" else {}, 1 if m == "mono" else 2, {}, 2, 8,
                       [call()])
       for n in (1024, 4096, 8192, 16384) for m in ("mono", "mix", "stereo")},
    **{f"v3-4096-s{s}": (4096, {}, 1, {}, s, 16, [call()]) for s in (1, 2, 3, 100, 150)},
    "v3-4096-many-streams": (4096, {}, 1, {}, (3, 0), 16, [call()]),
    "v3-peak": (4096, {}, 1, {}, 2, 8, [call(peak=True)]),
    "v3-opt": (4096, OPT, 1, {}, 2, 8, [call()]),
    "v3-display": (4096, {}, 1, {}, 2, 8, [call(points=True)]),
    **{f"v3-wide-r{r}": (4096, {}, 1, {"WF_WIDE_R": str(r)}, 2, 16, [call()]) for r in (1, 2, 4, 8)},
    "v3-16384-r8": (16384, {}, 1, {"WF_PAR16384": "0", "WF_WIDE_R": "8"}, 2, 16, [call()]),
    # wide clusters
    "wide-32768": (32768, {}, 1, {}, 1, 4, [call()]),
    "wide-32768-mix": (32768, {}, 2, {}, 1, 4, [call()]),
    "wide-4096": (4096, {}, 1, {"WF_V3": "0", "WF_WIDE_R": "2"}, 2, 8, [call()]),
    # one group of threads per stream
    **{f"fused-{n}": (n, {}, 1, {}, 2, 2, [call()]) for n in (128, 256, 512)},
    **{f"fused-{n}-display": (n, {}, 1, {}, 2, 2, [call(points=True)]) for n in (128, 256, 512)},
    "fused-32768-r1": (32768, {}, 1, {"WF_WIDE_R": "1"}, 1, 4, [call()]),
    "fused-32768-many-streams": (32768, {}, 1, {}, (2, 0), 1, [call()]),
    "fused-2048-mix-v3-off": (2048, {}, 2, {"WF_V3": "0"}, 2, 2, [call()]),
    # run-time mixed-radix plans, from shared memory and from the L2 scratch
    "anyn-2000": (2000, {}, 1, {}, 2, 2, [call()]),
    "anyn-2000-display": (2000, {}, 1, {}, 2, 2, [call(points=True)]),
    "anyn-8128": (8128, {}, 1, {}, 2, 2, [call()]),
    "anyn-40000": (40000, {}, 1, {}, 2, 2, [call()]),
    "anyn-65536": (65536, {}, 2, {}, 2, 2, [call()]),
    # sequences on one engine
    "seq-fast-then-display": (2048, {}, 1, {}, 2, 2, [call(), call(points=True), call()]),
    "seq-fast-then-mix-call": (2048, {}, 1, {}, 2, 2, [call(), call(pcm_off=1), call(), call(get_state=True)]),
    "seq-fast-get-state": (2048, {}, 1, {}, 2, 2, [call(), call(get_state=True), call(get_state=True)]),
    "seq-host-chunks": (2048, {}, 1, {}, 8200, 1, [call(buffers="host"), call(buffers="host", peak=True)]),
    "seq-host-small": (800, {}, 1, {}, 2, 2, [call(buffers="host"), call(buffers="host", points=True)]),
    "seq-mapped": (2048, {}, 1, {}, 1, 1, [call(buffers="mapped"), call(buffers="mapped")]),
    "seq-mapped-staged": (2048, {}, 1, {"WF_ZERO_COPY": "0"}, 1, 1, [call(buffers="mapped")]),
}


def _run(eng, S, T, c):
    """Runs one call of a case on `eng`; returns (last_kernel_name, launches the call made)."""
    import torch

    before = eng.launch_count
    if c.get("get_state"):
        eng.get_state()
        return eng.last_kernel_name(), eng.launch_count - before
    N, cc, dch, B, P = eng.fft_size, eng.capture_channels, eng.display_channels, eng.bins, eng.num_points
    hop = c.get("hop", N)
    ns = (T - 1) * hop + N
    sizes = {"db": S * T * dch * B, "silent": S * T, "points": S * T * dch * P, "pixels": S * T * dch * P,
             "min": S * T * 2, "peak": T}
    want = {"db": c.get("db", True), "silent": True, "points": c.get("points", False),
            "pixels": c.get("pixels", False), "min": c.get("pixels", False), "peak": c.get("peak", False)}
    buffers = c.get("buffers", "device")
    if buffers == "host":
        eng.process(np.zeros((S, cc, ns), np.float32), T, hop, want_db=want["db"], want_points=want["points"],
                    want_peak=want["peak"], want_pixels=want["pixels"])
        return eng.last_kernel_name(), eng.launch_count - before
    if buffers == "mapped":
        L = eng.L
        ptrs = {"pcm": L.wf_host_alloc(S * cc * ns * 4)}
        ptrs.update({k: L.wf_host_alloc(sizes[k] * 4) for k in sizes if want[k]})
        assert all(ptrs.values())
        C.memset(ptrs["pcm"], 0, S * cc * ns * 4)
        before = eng.launch_count
        eng.process_raw(ptrs["pcm"], S, T, hop, cc * ns, ns, out_db=ptrs.get("db"), out_silent=ptrs.get("silent"),
                        out_points=ptrs.get("points"), out_peak=ptrs.get("peak"))
        for p in ptrs.values():
            L.wf_host_free(p)
        return eng.last_kernel_name(), eng.launch_count - before
    # device buffers, offset by pcm_off / db_off floats from a 16-byte aligned allocation
    pcm = torch.zeros(S * cc * ns + 4, dtype=torch.float32, device="cuda")
    outs = {k: torch.empty(sizes[k] + 4, dtype=torch.uint8 if k == "silent" else torch.float32, device="cuda")
            for k in sizes if want[k]}

    def ptr(k, off=0):
        return outs[k].data_ptr() + 4 * off if k in outs else None

    eng.process_raw(pcm.data_ptr() + 4 * c.get("pcm_off", 0), S, T, hop, cc * ns, ns, out_db=ptr("db", c.get("db_off", 0)),
                    out_silent=ptr("silent"), out_points=ptr("points"), out_pixels=ptr("pixels"), out_min=ptr("min"),
                    out_peak=ptr("peak"), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return eng.last_kernel_name(), eng.launch_count - before


_recorded: dict = {}


def _save():
    import torch

    props = torch.cuda.get_device_properties(0)
    STORE.write_text(json.dumps({"device": props.name, "sm_count": props.multi_processor_count,
                                 "routes": dict(sorted(_recorded.items()))}, indent=1) + "\n")


@pytest.mark.parametrize("case", list(CASES))
def test_route(case, monkeypatch):
    import torch
    from waveform_b200 import Engine

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    if not RECORDING:
        table = json.loads(STORE.read_text())
        if table["sm_count"] != sm:
            pytest.skip(f"routes recorded on a {table['device']} with {table['sm_count']} SMs; this device has {sm}")
        assert case in table["routes"], f"{case}: not in {STORE.name}; record it with WF_RECORD_ROUTES=1"
    N, settings, cc, env, S, T, calls = CASES[case]
    set_knobs(monkeypatch, env)
    if isinstance(S, tuple):
        S = S[0] * sm + S[1]
    eng = Engine({"fft_size": N, **settings}, channels=cc, max_streams=S)
    got = [list(_run(eng, S, T, c)) for c in calls]
    eng.close()
    if RECORDING:
        if not _recorded:
            atexit.register(_save)
        _recorded[case] = got
    else:
        assert got == table["routes"][case]
