"""CUDA graphs of the waveform engine: engines created with device_clock=True keep their clock on the GPU, plan every call
in a kernel, and may be captured and replayed.

Every comparison is bit for bit (out, silent, points, pixels, min) against a host-clock twin engine fed the same samples
through eager calls.  Captures use torch's default (global) capture mode on a fresh engine, with no warm-up call.

Run on an H100:  python -m pytest tests/test_gpu_wave_graph.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

from gpu_common import assert_bits_equal, capture, clean_knobs, replay, set_knobs, to_host  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]
SR = 48000
GOLD = sorted((Path(__file__).parent / "golden").glob("wave_*.npz"))


def _samples(S, cc, n, seed, fmt):
    x = synth_pcm(S, cc, n, seed=seed)
    x[:, :, n // 3: n // 3 + n // 4] = 0.0  # digital silence: the all-zero silent rule
    x[-1, :, : n // 5] = 1.0                 # |x| == 1: exact 0 dBFS entries
    if fmt == "s16":
        return np.round(x * 32767.0).astype(np.int16)
    return x.astype(np.float32)


def _dev(x):
    import torch

    return torch.from_numpy(x).cuda()


def _twins(settings, ch, S):
    from waveform_b200 import WaveEngine

    return WaveEngine(settings, channels=ch, max_streams=S, device_clock=True), WaveEngine(settings, channels=ch, max_streams=S)


def _walk(settings, hops):
    """The timestamp walk of tick_waveform restated with Python integers, from a fresh engine over ticks of the given hops:
    per tick the points emitted and whether the clock caught up (waveform_ts < start_ts) after a tick that emitted."""
    width, ms = settings.get("width", 800), settings.get("meter_buf", 150)
    off = settings.get("audio_sync_offset", 0)
    D = SR * off // 1000 if off > 0 else 0
    ws = int(SR * (ms / 1000.0))
    step = ms * 1000000 // width
    ns = lambda f: f * 1000000000 // SR  # noqa: E731
    clock, wts, buffered, emitted = 10 ** 10, 0, width, False
    counts, catch_up = [], []
    for hop in hops:
        clock += ns(hop)
        total = min(buffered + hop, ws + D)
        buffered, count, caught = total, 0, False
        if total > D:
            start, stop = clock - ns(total), clock - ns(D)
            caught = emitted and wts < start
            wts = max(wts, start)
            if wts > stop and wts - stop > step:
                wts = start
            while count < width and wts + count * step < stop:
                count += 1
            wts += count * step
            buffered, emitted = D, True
        counts.append(count)
        catch_up.append(caught)
    return counts, catch_up


# ---- 1. eager calls: the device planner against the host walk --------------------------------------------------------

EAGER = [  # name, settings, capture channels, PCM format, display outputs
    ("mix-f32", {"width": 800, "meter_buf": 150}, 2, "f32", {}),
    ("stereo-s16-offset-display", {"width": 300, "meter_buf": 50, "channel_mode": "stereo", "audio_sync_offset": 40}, 2,
     "s16", {"want_pixels": True}),
    ("single-offset-points", {"width": 200, "meter_buf": 10, "channel_mode": "single", "audio_sync_offset": 25,
                              "filter_mode": "gauss"}, 1, "f32", {"want_points": True}),
    ("mono-as-stereo-s16-normalized", {"width": 640, "meter_buf": 20, "channel_mode": "stereo",
                                       "normalize_volume": True}, 1, "s16", {"want_points": True, "want_pixels": True}),
]


def _hops(settings):
    ms, off = settings.get("meter_buf", 150), settings.get("audio_sync_offset", 0)
    big = int(SR * ms / 1000) + (SR * off // 1000 if off > 0 else 0) + 300  # more than the buffer: the clock catches up
    return [800, 1, 7, big, 800, 7, 1]


@pytest.mark.parametrize("name,settings,ch,fmt,want", EAGER, ids=[e[0] for e in EAGER])
def test_eager_calls_equal_the_host_clock(name, settings, ch, fmt, want):
    S, T = 3, 3
    hops = _hops(settings)
    counts, caught = _walk(settings, [h for h in hops for _ in range(T)])
    assert any(caught) and 0 in counts and max(counts) > 0  # the catch-up branch and ticks without points are reached
    a, b = _twins(settings, ch, S)
    for i, hop in enumerate(hops):
        x = _dev(_samples(S, ch, T * hop, 10 + i, fmt))
        rms = _dev(np.random.default_rng(i).uniform(0.01, 0.3, (S, T)).astype(np.float32)) \
            if settings.get("normalize_volume") else None
        la, lb = a.launch_count, b.launch_count
        got = to_host(a.process(x, T, hop, input_rms=rms, pcm_format=fmt, **want))
        assert_bits_equal(got, to_host(b.process(x, T, hop, input_rms=rms, pcm_format=fmt, **want)), (name, i, hop))
        assert a.launch_count - la == b.launch_count - lb + 1  # the plan kernel
        assert a.last_kernel_ms() >= 0


@pytest.mark.parametrize("width,want", [(1, {}), (2, {"want_pixels": True}), (8192, {"want_points": True, "want_pixels": True})])
def test_eager_extreme_widths(width, want):
    S, T = 2, 4
    settings = {"width": width, "meter_buf": 150, "channel_mode": "stereo"}
    a, b = _twins(settings, 2, S)
    for i, hop in enumerate((800, 3, 9000, 441)):
        x = _dev(_samples(S, 2, T * hop, 40 + i, "f32"))
        assert_bits_equal(to_host(a.process(x, T, hop, **want)), to_host(b.process(x, T, hop, **want)), (width, i))


@pytest.mark.parametrize("seed", range(8))
def test_long_calls_through_runs_and_breaks(seed):
    """Long calls (up to thousands of ticks) with random settings and hops: the planner's steady-state runs span several
    windows, and the start-up, catch-ups (hops longer than the buffer) and changes of hop between calls break them."""
    rng = np.random.default_rng(900 + seed)
    ch = int(rng.choice([1, 2]))
    settings = {"width": int(rng.choice([1, 64, 301, 800, 2048])), "meter_buf": int(rng.choice([5, 20, 150, 500])),
                "audio_sync_offset": int(rng.choice([0, 0, 25, 170]))}
    a, b = _twins(settings, ch, 1)
    for i in range(5):
        hop = int(rng.choice([1, 7, 97, 441, 800, 2000, 9000, 30000]))
        T = max(1, min(int(rng.integers(1, 3000)), 3_000_000 // hop))
        x = _dev(_samples(1, ch, T * hop, 950 + 10 * seed + i, "f32"))
        la, lb = a.launch_count, b.launch_count
        assert_bits_equal(to_host(a.process(x, T, hop)), to_host(b.process(x, T, hop)), (settings, ch, i, hop, T))
        assert a.launch_count - la == b.launch_count - lb + 1


# ---- 2., 3. replays, alone and interleaved with eager calls ----------------------------------------------------------

def test_replays_from_a_fresh_engine_cross_the_startup():
    """With a 40 ms offset (1920 samples) the first ticks of 800 samples emit nothing; the replays go through that start-up
    and on, as the twin's eager calls do."""
    import torch

    S, T, hop = 2, 1, 800
    settings = {"width": 800, "meter_buf": 150, "audio_sync_offset": 40}
    counts, _ = _walk(settings, [hop] * 8)
    assert counts[0] == 0 and counts[-1] > 0
    a, b = _twins(settings, 2, S)
    xin = torch.zeros((S, 2, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, want_pixels=True))
    assert a.last_kernel_ms() < 0
    for i in range(8):
        x = _samples(S, 2, T * hop, 100 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(to_host(out), to_host(b.process(_dev(x), T, hop, want_pixels=True)), ("replay", i))


def test_replays_interleaved_with_eager_calls_and_two_graphs():
    import torch

    S = 2
    settings = {"width": 300, "meter_buf": 50, "channel_mode": "stereo", "audio_sync_offset": 10}
    a, b = _twins(settings, 2, S)
    shapes = [(1, 800), (4, 97)]
    xins = [torch.zeros((S, 2, T * hop), device="cuda") for T, hop in shapes]
    graphs = [capture(lambda T=T, hop=hop, xin=xin: a.process(xin, T, hop)) for (T, hop), xin in zip(shapes, xins)]
    for i in range(9):
        T, hop = shapes[i % 2] if i % 3 else (2, 2000)
        x = _samples(S, 2, T * hop, 200 + i, "f32")
        want = to_host(b.process(_dev(x), T, hop))
        if i % 3:
            g, out = graphs[i % 2]
            replay(g, [xins[i % 2]], [x])
            got = to_host(out)
        else:
            got = to_host(a.process(_dev(x), T, hop))
        assert_bits_equal(got, want, ("interleaved", i))


# ---- 4. live ticks ---------------------------------------------------------------------------------------------------

def test_live_tick_in_mapped_host_memory():
    """1 stream x 1 tick, stereo capture, out_pixels + out_min, every buffer in wf_host_alloc memory, with a sync offset."""
    import torch
    from waveform_b200.engine import WfWaveBatch

    hop, W = 800, 800
    settings = {"width": W, "meter_buf": 150, "channel_mode": "stereo", "audio_sync_offset": 40}
    a, b = _twins(settings, 2, 1)
    L = a.L
    pin, ppx, pmin, psil = L.wf_host_alloc(2 * hop * 4), L.wf_host_alloc(2 * W * 4), L.wf_host_alloc(8), L.wf_host_alloc(16)
    try:
        x_h = np.ctypeslib.as_array((C.c_float * (2 * hop)).from_address(pin)).reshape(1, 2, hop)
        px_h = np.ctypeslib.as_array((C.c_float * (2 * W)).from_address(ppx)).reshape(1, 1, 2, W)
        min_h = np.ctypeslib.as_array((C.c_float * 2).from_address(pmin)).reshape(1, 1, 2)
        sil_h = np.ctypeslib.as_array((C.c_uint8 * 1).from_address(psil)).reshape(1, 1)
        wb = WfWaveBatch(struct_size=C.sizeof(WfWaveBatch), n_streams=1, n_ticks=1, hop=hop, pcm=pin,
                         stream_stride=2 * hop, channel_stride=hop, out_silent=psil, out_pixels=ppx, out_min=pmin)

        def tick():
            assert L.wf_wave_process_async(a.h, C.byref(wb), torch.cuda.current_stream().cuda_stream) == 0

        g, _ = capture(tick)
        for i in range(6):
            x = _samples(1, 2, hop, 300 + i, "f32")
            x_h[...] = x
            g.replay()
            torch.cuda.synchronize()
            want = to_host(b.process(_dev(x), 1, hop, want_db=False, want_pixels=True))
            assert_bits_equal({"silent": sil_h.copy(), "pixels": px_h.copy(), "min": min_h.copy()}, want, ("mapped", i))
    finally:
        for p in (pin, ppx, pmin, psil):
            L.wf_host_free(p)


def test_rms_feed_and_waveform_chain_as_one_graph():
    """A waveform-mode tick: RMS feed -> waveform with normalize_volume, out_pixels and out_min, captured as one graph."""
    import torch
    from waveform_b200 import MeterEngine, WaveEngine
    from waveform_b200.engine import METER_INPUT_RMS

    S, T, hop, cc = 2, 2, 800, 2
    settings = {"width": 800, "meter_buf": 150, "channel_mode": "stereo", "normalize_volume": True, "audio_sync_offset": 20}
    chains = [(MeterEngine({"audio_sync_offset": 20}, channels=cc, max_streams=S, mode=METER_INPUT_RMS),
               WaveEngine(settings, channels=cc, max_streams=S, device_clock=clock)) for clock in (True, False)]

    def tick(m, w, x):
        rms = m.process(x, T, hop)["rms"]
        return {"rms": rms, **w.process(x, T, hop, input_rms=rms, want_db=False, want_pixels=True)}

    xin = torch.zeros((S, cc, T * hop), device="cuda")
    g, out = capture(lambda: tick(*chains[0], xin))
    for i in range(6):
        x = _samples(S, cc, T * hop, 400 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(to_host(out), to_host(tick(*chains[1], _dev(x))), ("chain", i))


# ---- 5. the per-tick kernel ------------------------------------------------------------------------------------------

def test_per_tick_kernel_replays(monkeypatch):
    import torch

    set_knobs(monkeypatch, {"WF_WAVE_CHUNK": "0"})
    S, T, hop = 2, 3, 441
    settings = {"width": 301, "meter_buf": 40, "channel_mode": "stereo", "audio_sync_offset": 15}
    a, b = _twins(settings, 1, S)
    xin = torch.zeros((S, 1, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, want_points=True))
    for i in range(6):
        x = _samples(S, 1, T * hop, 500 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(to_host(out), to_host(b.process(_dev(x), T, hop, want_points=True)), ("per-tick", i))


# ---- 6. buffer growth ------------------------------------------------------------------------------------------------

def test_larger_eager_call_after_a_capture_keeps_the_graph_working():
    import torch

    S, T, hop = 2, 2, 800
    settings = {"width": 800, "meter_buf": 150, "audio_sync_offset": 30}
    a, b = _twins(settings, 2, S)
    xin = torch.zeros((S, 2, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop))
    for i in range(4):
        x = _samples(S, 2, T * hop, 600 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(to_host(out), to_host(b.process(_dev(x), T, hop)), ("replay", i))
        big = _dev(_samples(S, 2, (40 + 8 * i) * hop, 650 + i, "f32"))  # more plan space and a larger window each time
        assert_bits_equal(to_host(a.process(big, 40 + 8 * i, hop)), to_host(b.process(big, 40 + 8 * i, hop)), ("growth", i))


# ---- 7. refusals -----------------------------------------------------------------------------------------------------

def test_pageable_pcm_is_refused_under_capture_and_the_clock_stays():
    import torch
    from waveform_b200.engine import WF_ERR_INVALID_ARG, WfError

    S, T, hop = 2, 2, 800
    settings = {"width": 800, "meter_buf": 150, "audio_sync_offset": 20}
    a, b = _twins(settings, 2, S)
    c, d = _twins(settings, 2, S)
    host = _samples(S, 2, T * hop, 700, "f32")
    xin = torch.zeros((S, 2, T * hop), device="cuda")
    errors = []

    def body():
        with pytest.raises(WfError) as ei:
            a.process(host, T, hop, stream=torch.cuda.current_stream().cuda_stream)
        errors.append(ei.value)
        return c.process(xin, T, hop)

    g, out = capture(body)
    assert len(errors) == 1 and errors[0].status == WF_ERR_INVALID_ARG and "graph" in str(errors[0])
    x = _samples(S, 2, T * hop, 701, "f32")
    replay(g, [xin], [x])
    assert_bits_equal(to_host(out), to_host(d.process(_dev(x), T, hop)), "capture after the refusal")
    y = _dev(_samples(S, 2, T * hop, 702, "f32"))
    assert_bits_equal(to_host(a.process(y, T, hop)), to_host(b.process(y, T, hop)), "first eager call after the refusal")


# ---- 8. the reference's rows through replays -------------------------------------------------------------------------

@pytest.mark.parametrize("path", GOLD, ids=[p.stem for p in GOLD])
def test_one_tick_graph_replays_reproduce_the_golden_rows(path):
    """A 1-tick graph replayed n_ticks times over the fixture's packets, under test_wave.py's rule for GPU calls: the DB_MIN
    pattern (which points exist) and the silent flags exact, dB values within 1e-4 dB."""
    import torch
    from waveform_b200 import WaveEngine

    z = np.load(path, allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    ch, hop, T = int(z["channels"]), int(z["hop"]), int(z["n_ticks"])
    rms = z["rms"] if z["rms"].size else None
    eng = WaveEngine(settings, channels=ch, max_streams=1, device_clock=True)
    xin = torch.zeros((1, ch, hop), device="cuda")
    rin = torch.zeros((1, 1), device="cuda")
    g, o = capture(lambda: eng.process(xin, 1, hop, input_rms=rin if rms is not None else None))
    rows, sil = [], []
    for t in range(T):
        replay(g, [xin, rin], [np.ascontiguousarray(z["pcm"][None, :, t * hop:(t + 1) * hop]),
                               np.full((1, 1), 0.0 if rms is None else rms[t], np.float32)])
        rows.append(o["out"].cpu().numpy()[0, 0])
        sil.append(int(o["silent"].cpu().numpy()[0, 0]))
    out, ref = np.stack(rows), z["out"]
    assert np.array_equal(np.array(sil, np.uint8), z["silent"])
    lo = ref < -700.0
    assert np.array_equal(out < -700.0, lo)
    raw = (~lo) & (np.abs(ref) <= 1.0) & (ref == out)
    assert np.max(np.abs(out[lo] - ref[lo]), initial=0.0) < 1e-3  # DB_MIN + volume compensation (log10f)
    assert np.max(np.abs(out[~lo & ~raw] - ref[~lo & ~raw]), initial=0.0) < 1e-4
