"""CUDA graphs: spectrum, render, peak-normalise, level-meter and RMS-feed calls captured once and replayed.

Every case captures a call (or a chain of calls) on a fresh engine under torch's default (global) capture mode, with no
warm-up call, and replays it with fresh samples written into the captured input buffers before each replay.  A twin engine
gets the same samples through eager calls; outputs, state and capture rings must agree bit for bit after every replay.

Run on an H100:  python -m pytest tests/test_gpu_graph.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from gpu_common import assert_bits_equal, capture, clean_knobs, replay, to_host  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]
K = 5  # replays per case: more than the start-up ticks of the sync offsets below last


def _samples(S, cc, n, seed, fmt):
    x = synth_pcm(S, cc, n, seed=seed)
    x[:, :, n // 3: n // 3 + n // 4] = 0.0  # digital silence: the gate and m_last_silent
    if fmt == "s16":
        return np.round(x * 32767.0).astype(np.int16)
    return x.astype(np.float32)


def _same_state(a, b):
    assert_bits_equal(a.get_state(), b.get_state(), "state")


# ---- spectrum ------------------------------------------------------------------------------------------------------

PLAIN = [("n2048", {"fft_size": 2048}, 1, 64, 4, 800, "f32", {}),
         ("n800", {"fft_size": 800}, 2, 8, 3, 400, "f32", {}),
         ("n4096-stereo-display", {"fft_size": 4096, "channel_mode": "stereo"}, 2, 4, 3, 1024, "f32",
          {"want_points": True, "want_pixels": True, "want_peak": True}),
         ("n2048-s16", {"fft_size": 2048}, 1, 16, 4, 800, "s16", {}),
         ("n1024-s16-display", {"fft_size": 1024, "display_mode": "bars"}, 2, 4, 2, 512, "s16", {"want_points": True})]


@pytest.mark.parametrize("name,settings,cc,S,T,hop,fmt,want", PLAIN, ids=[p[0] for p in PLAIN])
def test_spectrum_plain_replays_equal_eager(name, settings, cc, S, T, hop, fmt, want):
    import torch
    from waveform_b200 import Engine

    a, b = Engine(settings, channels=cc, max_streams=S), Engine(settings, channels=cc, max_streams=S)
    n = (T - 1) * hop + a.fft_size
    xs = [_samples(S, cc, n, 100 + i, fmt) for i in range(K)]
    xin = torch.zeros(xs[0].shape, dtype=torch.int16 if fmt == "s16" else torch.float32, device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, pcm_format=fmt, **want))
    assert a.last_kernel_ms() < 0  # captured: not timed
    for i in range(K):
        replay(g, [xin], [xs[i]])
        want_i = to_host(b.process(torch.from_numpy(xs[i]).cuda(), T, hop, pcm_format=fmt, **want))
        torch.cuda.synchronize()
        assert_bits_equal(to_host(out), want_i, (name, i))
        _same_state(a, b)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("ms", [0, 100])
def test_ring_replays_skip_startup_once(ms, fmt):
    """Ring calls from a fresh engine: the start-up ticks the sync offset owes (100 ms = 4800 samples: the first 5 ticks
    of 800 samples, over the first 3 calls) are skipped over the first replays and never again, as over the twin's eager
    calls."""
    import torch
    from waveform_b200 import Engine

    S, T, hop = 3, 2, 800
    st = {"fft_size": 2048, "audio_sync_offset": ms}
    a, b = Engine(st, channels=1, max_streams=S), Engine(st, channels=1, max_streams=S)
    xs = [_samples(S, 1, T * hop, 200 + i, fmt) for i in range(K)]
    xin = torch.zeros(xs[0].shape, dtype=torch.int16 if fmt == "s16" else torch.float32, device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, pcm_format=fmt, capture_ring=True, want_peak=True))
    for i in range(K):
        replay(g, [xin], [xs[i]])
        w = to_host(b.process(torch.from_numpy(xs[i]).cuda(), T, hop, pcm_format=fmt, capture_ring=True, want_peak=True))
        torch.cuda.synchronize()
        assert_bits_equal(to_host(out), w, ("ring", ms, fmt, i))
        _same_state(a, b)
        assert np.array_equal(a.get_ring(), b.get_ring())


def test_ring_mapped_live_tick():
    """One live tick (1 stream x 1 frame, N=800) in wf_host_alloc buffers: replays read and write them in place."""
    import torch
    from waveform_b200 import Engine

    N, hop = 800, 800
    st = {"fft_size": N, "audio_sync_offset": 40}
    a, b = Engine(st, channels=2, max_streams=1), Engine(st, channels=2, max_streams=1)
    L = a.L
    dch, B = a.display_channels, a.bins
    pin, pout, psil = L.wf_host_alloc(2 * hop * 4), L.wf_host_alloc(dch * B * 4), L.wf_host_alloc(16)
    try:
        x_h = np.ctypeslib.as_array((C.c_float * (2 * hop)).from_address(pin)).reshape(1, 2, hop)
        db_h = np.ctypeslib.as_array((C.c_float * (dch * B)).from_address(pout)).reshape(1, 1, dch, B)
        sil_h = np.ctypeslib.as_array((C.c_uint8 * 1).from_address(psil)).reshape(1, 1)

        def tick():
            a.process_raw(pin, 1, 1, hop, 2 * hop, hop, out_db=pout, out_silent=psil, capture_ring=True,
                          stream=torch.cuda.current_stream().cuda_stream, sync=False)

        g, _ = capture(tick)
        for i in range(K):
            x = _samples(1, 2, hop, 300 + i, "f32")
            x_h[...] = x
            g.replay()
            torch.cuda.synchronize()
            w = to_host(b.process(torch.from_numpy(x).cuda(), 1, hop, capture_ring=True))
            assert_bits_equal({"db": db_h.copy(), "silent": sil_h.copy()}, w, ("mapped", i))
        _same_state(a, b)
        assert np.array_equal(a.get_ring(), b.get_ring())
    finally:
        for p in (pin, pout, psil):
            L.wf_host_free(p)


def test_frame_seconds_replay_keeps_captured_gains():
    """TV-exponential smoothing with per-tick seconds: replays apply the gains they were captured with, while eager calls
    with other seconds run in between."""
    import torch
    from waveform_b200 import Engine

    S, T, hop = 4, 3, 800
    st = {"fft_size": 2048, "temporal_smoothing": "tv_exp_moving_avg"}
    a, b = Engine(st, channels=1, max_streams=S), Engine(st, channels=1, max_streams=S)
    fs_cap, fs_other = np.array([1 / 60, 1 / 30, 1 / 90], np.float32), np.array([0.1, 0.002, 0.05], np.float32)
    n = (T - 1) * hop + 2048
    xin = torch.zeros((S, 1, n), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, frame_seconds=fs_cap))
    for i in range(K):
        x = _samples(S, 1, n, 400 + i, "f32")
        replay(g, [xin], [x])
        got = to_host(out)
        w = to_host(b.process(torch.from_numpy(x).cuda(), T, hop, frame_seconds=fs_cap))
        torch.cuda.synchronize()
        assert_bits_equal(got, w, ("frame_seconds", i))
        y = torch.from_numpy(_samples(S, 1, n, 450 + i, "f32")).cuda()
        assert_bits_equal(to_host(a.process(y, T, hop, frame_seconds=fs_other)),
                          to_host(b.process(y, T, hop, frame_seconds=fs_other)), ("eager between", i))
        torch.cuda.synchronize()
        _same_state(a, b)


def test_replays_interleaved_with_eager_calls():
    """Replays and eager calls on one engine advance the same EMA state, capture rings and start-up counts."""
    import torch
    from waveform_b200 import Engine

    S, T, hop = 2, 2, 800
    st = {"fft_size": 2048, "audio_sync_offset": 60}
    a, b = Engine(st, channels=1, max_streams=S), Engine(st, channels=1, max_streams=S)
    xin = torch.zeros((S, 1, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, capture_ring=True))
    for i in range(2 * K):
        x = _samples(S, 1, T * hop, 500 + i, "f32")
        w = to_host(b.process(torch.from_numpy(x).cuda(), T, hop, capture_ring=True))
        if i % 2:
            got = to_host(a.process(torch.from_numpy(x).cuda(), T, hop, capture_ring=True))
        else:
            replay(g, [xin], [x])
            got = to_host(out)
        torch.cuda.synchronize()
        assert_bits_equal(got, w, ("interleaved", i))
        _same_state(a, b)
        assert np.array_equal(a.get_ring(), b.get_ring())


def test_larger_call_after_capture_keeps_graph_buffers():
    """An eager call with a larger shape grows the scratch buffers; the old graph still replays correctly.  The meters
    cover both paths: the general one (hop 700) and the one-pass one (hop 800), whose block partials move to a new layout
    when an eager call with hop 400 needs twice the blocks per stream."""
    import torch
    from waveform_b200 import Engine, MeterEngine

    S, T, hop = 2, 1, 800
    st = {"fft_size": 2048, "audio_sync_offset": 30}
    a, b = Engine(st, channels=2, max_streams=S), Engine(st, channels=2, max_streams=S)
    ma, mb = MeterEngine({}, channels=2, max_streams=S), MeterEngine({}, channels=2, max_streams=S)
    mc, md = MeterEngine({}, channels=2, max_streams=S), MeterEngine({}, channels=2, max_streams=S)
    xin = torch.zeros((S, 2, T * hop), device="cuda")
    g, out = capture(lambda: (a.process(xin, T, hop, capture_ring=True), ma.process(xin, T, 700),
                              mc.process(xin, T, 800)))
    for i in range(4):
        x = _samples(S, 2, T * hop, 600 + i, "f32")
        replay(g, [xin], [x])
        got = [to_host(o) for o in out]
        xd = torch.from_numpy(x).cuda()
        w = [to_host(b.process(xd, T, hop, capture_ring=True)), to_host(mb.process(xd, T, 700)), to_host(md.process(xd, T, 800))]
        for gg, ww in zip(got, w):
            assert_bits_equal(gg, ww, ("replay", i))
        if i % 2 == 0:  # every other round: larger eager calls between the replays
            big = torch.from_numpy(_samples(S, 2, 48 * hop, 650 + i, "f32")).cuda()
            for e in (a, b):
                e.process(big, 48, hop, capture_ring=True)
            for e in (ma, mb):
                e.process(big, 48, 700)
            assert_bits_equal(to_host(mc.process(big, 48, 400)), to_host(md.process(big, 48, 400)), ("one-pass growth", i))
        torch.cuda.synchronize()
    for i in range(2):  # eager one-pass calls on the new layout, partials reused from the first
        y = torch.from_numpy(_samples(S, 2, 4 * 400, 680 + i, "f32")).cuda()
        assert_bits_equal(to_host(mc.process(y, 4, 400)), to_host(md.process(y, 4, 400)), ("after", i))
    _same_state(a, b)
    assert np.array_equal(a.get_ring(), b.get_ring())


def test_meter_mixed_hops_on_subsets_keep_each_streams_partials():
    """One-pass calls with different hops on different streams: a whole-engine call with hop 400, stream 1 alone with hop
    800, then stream 0 alone with hop 400, which reuses the block partials its first call left.  Each stream must get what
    an engine of that stream alone gets, eagerly and with the stream-1 call replayed from a graph."""
    import torch
    from waveform_b200 import MeterEngine

    S, T, cc = 4, 3, 2
    st = {"rms_mode": False, "meter_buf": 100}  # PEAK, W = 4800: hops 400 and 800 both take the one-pass path
    h1, h2 = 400, 800
    x0 = _samples(S, cc, T * h1, 1100, "f32")
    x1 = _samples(1, cc, T * h2, 1101, "f32")
    x2 = _samples(1, cc, T * h1, 1102, "f32")
    dev = lambda v: torch.from_numpy(v).cuda()  # noqa: E731

    # per-stream references: an engine of one stream fed that stream's calls
    ref0 = MeterEngine(st, channels=cc, max_streams=1)
    ref0.process(dev(x0[0:1]), T, h1)
    want0 = to_host(ref0.process(dev(x2), T, h1))
    ref1 = MeterEngine(st, channels=cc, max_streams=1)
    ref1.process(dev(x0[1:2]), T, h1)
    want1 = to_host(ref1.process(dev(x1), T, h2))

    eager = MeterEngine(st, channels=cc, max_streams=S)
    eager.process(dev(x0), T, h1)
    assert_bits_equal(to_host(eager.process(dev(x1), T, h2, first_stream=1)), want1, "eager stream 1")
    assert_bits_equal(to_host(eager.process(dev(x2), T, h1, first_stream=0)), want0, "eager stream 0")

    graph = MeterEngine(st, channels=cc, max_streams=S)
    xin = torch.zeros((1, cc, T * h2), device="cuda")
    g, out = capture(lambda: graph.process(xin, T, h2, first_stream=1))
    graph.process(dev(x0), T, h1)
    replay(g, [xin], [x1])
    assert_bits_equal(to_host(out), want1, "replayed stream 1")
    assert_bits_equal(to_host(graph.process(dev(x2), T, h1, first_stream=0)), want0, "stream 0 after the replay")


def test_display_graph_after_lazy_n2048_calls():
    """N=2048 mono: a display call (which reads hold_db as it is) captured on a fresh engine, replayed after eager plain calls
    whose kernel leaves the m_decibels mirrors implicit.  Tick 0 is skipped, so its outputs come from those mirrors."""
    import torch
    from waveform_b200 import Engine

    S, T, hop, N = 4, 3, 800, 2048
    a, b = Engine({"fft_size": N}, channels=1, max_streams=S), Engine({"fft_size": N}, channels=1, max_streams=S)
    n = (T - 1) * hop + N
    mask = torch.zeros((S, T), dtype=torch.uint8, device="cuda")
    mask[:, 0] = 1
    xin = torch.zeros((S, 1, n), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, skip_mask=mask, want_points=True))
    for i in range(K):
        y = torch.from_numpy(_samples(S, 1, n, 1200 + i, "f32")).cuda()
        assert_bits_equal(to_host(a.process(y, T, hop)), to_host(b.process(y, T, hop)), ("plain", i))
        x = _samples(S, 1, n, 1250 + i, "f32")
        replay(g, [xin], [x])
        w = to_host(b.process(torch.from_numpy(x).cuda(), T, hop, skip_mask=mask, want_points=True))
        torch.cuda.synchronize()
        assert_bits_equal(to_host(out), w, ("display replay", i))
        _same_state(a, b)


# ---- render and peak normalisation -----------------------------------------------------------------------------------

def test_rms_feed_spectrum_render_chain():
    """One spectrum-mode tick as one graph: RMS feed -> ring spectrum with normalize_volume and out_peak -> wf_render with
    the peak, and wf_peak_normalize on a copy of the rows."""
    import torch
    from waveform_b200 import Engine, MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    S, T, hop, cc = 3, 2, 800, 2
    st = {"fft_size": 2048, "normalize_volume": True, "audio_sync_offset": 20}
    engines = [(Engine(st, channels=cc, max_streams=S),
                MeterEngine({"audio_sync_offset": 20}, channels=cc, max_streams=S, mode=METER_INPUT_RMS))
               for _ in range(2)]

    def tick(e, m, x):
        rms = m.process(x, T, hop)["rms"]
        o = e.process(x, T, hop, input_rms=rms, capture_ring=True, want_peak=True)
        r = e.render(o["db"], peak=o["peak"], want_points=True, want_pixels=True)
        rows = o["db"].clone()
        e.peak_normalize(rows, o["peak"], -3.0, 30.0)
        return {"rms": rms, **o, **r, "normalized": rows}

    xin = torch.zeros((S, cc, T * hop), device="cuda")
    g, out = capture(lambda: tick(*engines[0], xin))
    for i in range(K):
        x = _samples(S, cc, T * hop, 700 + i, "f32")
        replay(g, [xin], [x])
        got = to_host(out)
        w = to_host(tick(*engines[1], torch.from_numpy(x).cuda()))
        torch.cuda.synchronize()
        assert_bits_equal(got, w, ("chain", i))
    _same_state(engines[0][0], engines[1][0])
    assert engines[0][0].last_kernel_ms() < 0 and engines[0][1].last_kernel_ms() < 0


# ---- level meter and RMS feed ----------------------------------------------------------------------------------------

METER = [("peak", {"rms_mode": False, "meter_buf": 100}, None), ("rms", {"rms_mode": True, "meter_buf": 150}, None),
         ("feed", {}, "feed")]


@pytest.mark.parametrize("hop", [800, 700], ids=["one-pass", "general"])
@pytest.mark.parametrize("ms", [0, 30])
@pytest.mark.parametrize("name,settings,feed", METER, ids=[m[0] for m in METER])
def test_meter_replays_equal_eager(name, settings, feed, ms, hop):
    """Whole-engine calls, then a captured subset call (stream 1 of 3) replayed between them: the other streams' rings
    stay where they were, and a final whole-engine call agrees with the twin's."""
    import torch
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    S, T, cc = 3, 3, 2
    st = {**settings, "audio_sync_offset": ms}
    mode = METER_INPUT_RMS if feed else None
    a, b = (MeterEngine(st, channels=cc, max_streams=S, mode=mode) for _ in range(2))
    want_px = not feed

    def call(e, x, first=0):
        return to_host(e.process(x, T, hop, first_stream=first, want_pixels=want_px))

    # a fresh engine captured first (no warm-up), then whole-engine eager calls around the subset replays
    xin = torch.zeros((1, cc, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, first_stream=1, want_pixels=want_px))
    for i in range(K):
        if i % 2:
            x = torch.from_numpy(_samples(S, cc, T * hop, 800 + i, "f32")).cuda()
            assert_bits_equal(call(a, x), call(b, x), (name, "whole", i))
        x1 = _samples(1, cc, T * hop, 850 + i, "f32")
        replay(g, [xin], [x1])
        got = to_host(out)
        assert_bits_equal(got, call(b, torch.from_numpy(x1).cuda(), 1), (name, "subset", i))
    x = torch.from_numpy(_samples(S, cc, T * hop, 899, "f32")).cuda()
    assert_bits_equal(call(a, x), call(b, x), (name, "final"))
    assert a.last_kernel_ms() >= 0  # the last call was eager


@pytest.mark.parametrize("hop", [800, 700], ids=["one-pass", "general"])
def test_meter_s16_whole_replays(hop):
    import torch
    from waveform_b200 import MeterEngine

    S, T, cc = 4, 2, 2
    a, b = (MeterEngine({"audio_sync_offset": 25}, channels=cc, max_streams=S) for _ in range(2))
    xin = torch.zeros((S, cc, T * hop), dtype=torch.int16, device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, pcm_format="s16"))
    for i in range(K):
        x = _samples(S, cc, T * hop, 900 + i, "s16")
        replay(g, [xin], [x])
        got = to_host(out)
        assert_bits_equal(got, to_host(b.process(torch.from_numpy(x).cuda(), T, hop, pcm_format="s16")), ("s16", i))


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refusals_leave_capture_and_state_intact():
    """Pageable host buffers under capture, and any waveform call under capture: WF_ERR_INVALID_ARG with the reason, nothing
    enqueued or advanced, and the capture still ends and replays."""
    import torch
    from waveform_b200 import Engine, MeterEngine, WaveEngine
    from waveform_b200.engine import WF_ERR_INVALID_ARG, WfError

    S, T, hop = 2, 2, 800
    st = {"fft_size": 2048, "audio_sync_offset": 50}
    a, b = Engine(st, channels=1, max_streams=S), Engine(st, channels=1, max_streams=S)
    m = MeterEngine({}, channels=1, max_streams=S)
    wa, wb = WaveEngine({}, channels=2, max_streams=1), WaveEngine({}, channels=2, max_streams=1)
    host = _samples(S, 1, T * hop, 1000, "f32")
    host_out = np.zeros((S, T, 1, a.bins), np.float32)
    wave_x = torch.from_numpy(_samples(1, 2, T * 800, 1001, "f32")).cuda()
    xin = torch.zeros((S, 1, T * hop), device="cuda")
    errors = []

    def body():
        cs = torch.cuda.current_stream().cuda_stream
        for f in (lambda: a.process_raw(host.ctypes.data, S, T, hop, T * hop, T * hop, out_db=host_out.ctypes.data,
                                        capture_ring=True, stream=cs, sync=False),
                  lambda: m.process(host, T, hop, stream=cs),
                  lambda: a.render(torch.zeros((S, T, 1, a.bins), device="cuda"), peak=np.zeros(T, np.float32),
                                   want_points=True),
                  lambda: wa.process(wave_x, T, 800)):
            with pytest.raises(WfError) as ei:
                f()
            errors.append(ei.value)
        return a.process(xin, T, hop, capture_ring=True)

    g, out = capture(body)
    assert len(errors) == 4
    for e in errors:
        assert e.status == WF_ERR_INVALID_ARG and ("graph" in str(e)), str(e)
    # nothing changed: the state, the rings and the start-up counts are a fresh engine's
    _same_state(a, b)
    assert np.array_equal(a.get_ring(), b.get_ring())
    x = _samples(S, 1, T * hop, 1002, "f32")
    replay(g, [xin], [x])
    assert_bits_equal(to_host(out), to_host(b.process(torch.from_numpy(x).cuda(), T, hop, capture_ring=True)), "after refusal")
    assert_bits_equal(to_host(wa.process(wave_x, T, 800)), to_host(wb.process(wave_x, T, 800)), "wave after refusal")
    torch.cuda.synchronize()
