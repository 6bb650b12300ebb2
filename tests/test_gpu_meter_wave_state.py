"""Checkpoints of the level-meter and waveform engines on the GPU: wf_meter_get_state / wf_meter_set_state,
wf_wave_get_state / wf_wave_set_state and wf_wave_get_clock / wf_wave_set_clock.

The core criterion is the split run: engine A runs calls c1..c4; after c2 its state (and, for the waveform, its clock) goes
into a fresh engine B with the same config but another max_streams, at another first_stream; B then runs c3..c4 on the same
input.  Every output of B's c3..c4 and a final get_state must equal A's bit for bit.

Run on an H100:  python -m pytest tests/test_gpu_meter_wave_state.py -m gpu -q
"""
from __future__ import annotations

import numpy as np
import pytest

from gpu_common import assert_bits_equal, bits, capture, clean_knobs, replay, set_knobs  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]
SR = 48000


def _slots(out, lo, hi):
    return {k: v[lo:hi] for k, v in out.items()}


def _samples(S, cc, n, seed, fmt, silent_stream=None):
    x = synth_pcm(S, cc, n, seed=seed)
    x[:, :, n // 3: n // 3 + n // 4] = 0.0  # digital silence
    x[-1, :, : n // 5] = 1.0                 # |x| == 1: exact 0 dBFS entries
    if silent_stream is not None:
        x[silent_stream] = 0.0
    if fmt == "s16":
        return np.round(x * 32767.0).astype(np.int16)
    return x.astype(np.float32)


def _db_min():
    from waveform_b200 import Engine

    return np.float32(Engine({"fft_size": 1024}, channels=1).db_min)


# ---- level meter: split runs ------------------------------------------------------------------------------------------

METER = [  # name, settings, mode, capture channels, PCM format
    ("rms-stereo-f32", {"rms_mode": True}, None, 2, "f32"),
    ("rms-mono-s16-offset", {"rms_mode": True, "audio_sync_offset": 40}, None, 1, "s16"),
    ("peak-stereo-s16-offset", {"rms_mode": False, "fast_peaks": True, "audio_sync_offset": 40}, None, 2, "s16"),
    ("peak-mono-f32-nosmooth", {"rms_mode": False, "temporal_smoothing": "none"}, None, 1, "f32"),
    ("feed-stereo-f32-offset", {"audio_sync_offset": 40}, "feed", 2, "f32"),
    ("feed-mono-s16", {}, "feed", 1, "s16"),
]
# (n_ticks, hop) of c1..c4: the window of 150 ms (7200 samples) is 9 hops of 800 or 8 of 900, so those calls take the
# one-pass path and hops of 7 the three-kernel path.  "same-hop": the checkpoint falls between two one-pass calls with one
# hop (A reuses its partials, B reduces the restored ring); "switch": it falls between a three-kernel and a one-pass call.
METER_CALLS = {"same-hop": [(3, 800), (12, 800), (5, 800), (40, 7)], "switch": [(2, 800), (30, 7), (6, 900), (3, 900)]}


def _meter_pair(settings, mode, cc, S, S_b):
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    m = METER_INPUT_RMS if mode == "feed" else None
    return (MeterEngine(settings, channels=cc, max_streams=S, mode=m),
            MeterEngine(settings, channels=cc, max_streams=S_b, mode=m))


def _meter_call(e, x, T, hop, fmt, first=0):
    from waveform_b200.engine import METER_INPUT_RMS

    return e.process(x, T, hop, first_stream=first, pcm_format=fmt, want_pixels=e.cfg.mode != METER_INPUT_RMS)


@pytest.mark.parametrize("dest", ["fresh", "used"])
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "three-kernel"])
@pytest.mark.parametrize("calls", list(METER_CALLS), ids=list(METER_CALLS))
@pytest.mark.parametrize("name,settings,mode,cc,fmt", METER, ids=[m[0] for m in METER])
def test_meter_split_run(name, settings, mode, cc, fmt, calls, fused, dest, monkeypatch):
    """dest "used": before the restore B runs one call (an odd number) with the hop of c3 over other audio, so its slots'
    rings are in the second half and, on the one-pass path, their partials are valid for c3's hop.  The restore must write
    the half the parity selects and drop those partials, or B's c3 reads B's own earlier audio."""
    if not fused:
        set_knobs(monkeypatch, {"WF_METER_FUSED": "0"})
    S, first = 3, 2
    a, b = _meter_pair(settings, mode, cc, S, S + 4)
    schedule = METER_CALLS[calls]
    if dest == "used":
        hop = schedule[2][1]
        _meter_call(b, _samples(S + 4, cc, 10 * hop, 90, fmt), 10, hop, fmt)
    xs = [_samples(S, cc, T * hop, 100 + i, fmt, silent_stream=1 if i in (1, 2) else None)
          for i, (T, hop) in enumerate(schedule)]
    for i, (T, hop) in enumerate(schedule):
        want = _meter_call(a, xs[i], T, hop, fmt)
        if i == 1:
            state = a.get_state()
            if calls == "same-hop" and "temporal_smoothing" in settings:
                assert state["flags"][1] == 1  # a silent stream crosses the checkpoint
            b.set_state(state, first_stream=first)
        if i >= 2:
            assert_bits_equal(_meter_call(b, xs[i], T, hop, fmt, first=first), want, (name, calls, dest, i))
    assert_bits_equal(b.get_state(first, S), a.get_state(), (name, calls, dest, "final"))


# ---- waveform: split runs ---------------------------------------------------------------------------------------------

WAVE = [  # name, settings, capture channels, PCM format, display outputs
    ("mix-f32", {"width": 800, "meter_buf": 150}, 2, "f32", {}),
    ("stereo-s16-offset-display", {"width": 300, "meter_buf": 50, "channel_mode": "stereo", "audio_sync_offset": 40}, 2,
     "s16", {"want_points": True, "want_pixels": True}),
    ("single-offset-gauss", {"width": 200, "meter_buf": 10, "channel_mode": "single", "audio_sync_offset": 40,
                             "filter_mode": "gauss"}, 1, "f32", {"want_points": True}),
    ("mono-as-stereo-s16-normalized", {"width": 640, "meter_buf": 20, "channel_mode": "stereo", "normalize_volume": True},
     1, "s16", {"want_points": True, "want_pixels": True}),
]
CLOCKS = [(False, False), (False, True), (True, False), (True, True)]


def _wave_calls(settings):
    ms, off = settings.get("meter_buf", 150), settings.get("audio_sync_offset", 0)
    big = int(SR * ms / 1000) + (SR * off // 1000 if off > 0 else 0) + 300  # more than the buffer: the clock catches up
    return [(3, 800), (5, 7), (2, big), (4, 800)]


def _wave_input(S, cc, T, hop, seed, fmt, settings):
    x = _samples(S, cc, T * hop, seed, fmt)
    rms = np.random.default_rng(seed).uniform(0.01, 0.3, (S, T)).astype(np.float32) \
        if settings.get("normalize_volume") else None
    return x, rms


def _embed(x, rms, lo, S_b, seed, fmt, settings):
    """The input of a larger engine: x (and rms) in slots [lo, lo + len(x)), other audio in the others."""
    S, cc, n = x.shape
    y = _samples(S_b, cc, n, seed, fmt)
    y[lo:lo + S] = x
    r = None
    if rms is not None:
        r = np.random.default_rng(seed).uniform(0.01, 0.3, (S_b, rms.shape[1])).astype(np.float32)
        r[lo:lo + S] = rms
    return y, r


@pytest.mark.parametrize("clock_a,clock_b", CLOCKS, ids=[f"{'dev' if a else 'host'}-{'dev' if b else 'host'}" for a, b in CLOCKS])
@pytest.mark.parametrize("name,settings,cc,fmt,want", WAVE, ids=[w[0] for w in WAVE])
def test_wave_split_run(name, settings, cc, fmt, want, clock_a, clock_b):
    from waveform_b200 import WaveEngine

    S, S_b, first = 3, 5, 1
    a = WaveEngine(settings, channels=cc, max_streams=S, device_clock=clock_a)
    b = WaveEngine(settings, channels=cc, max_streams=S_b, device_clock=clock_b)
    for i, (T, hop) in enumerate(_wave_calls(settings)):
        x, rms = _wave_input(S, cc, T, hop, 200 + i, fmt, settings)
        ref = a.process(x, T, hop, input_rms=rms, pcm_format=fmt, **want)
        if i == 1:
            b.set_state(a.get_state(), first_stream=first)
            b.set_clock(a.get_clock())
            assert b.get_clock() == a.get_clock()
        if i >= 2:
            y, r = _embed(x, rms, first, S_b, 300 + i, fmt, settings)
            got = b.process(y, T, hop, input_rms=r, pcm_format=fmt, **want)
            assert_bits_equal(_slots(got, first, first + S), ref, (name, i))
    assert_bits_equal(b.get_state(first, S), a.get_state(), (name, "final"))
    assert b.get_clock() == a.get_clock()


def test_wave_migration_into_a_busy_engine():
    """Two slots of a source engine move into slots 1, 2 of a larger engine whose streams carry other audio and whose clock
    walked other hops; the source's clock goes with them.  The moved slots continue as in the source; the others continue
    as in a twin of the destination that only took the clock."""
    from waveform_b200 import WaveEngine

    settings, cc, fmt = {"width": 300, "meter_buf": 50, "channel_mode": "stereo", "audio_sync_offset": 20}, 2, "f32"
    want = {"want_pixels": True}
    src = WaveEngine(settings, channels=cc, max_streams=2)
    dst, twin = (WaveEngine(settings, channels=cc, max_streams=5, device_clock=c) for c in (True, False))
    for i, (T, hop) in enumerate([(4, 800), (3, 441)]):
        src.process(_samples(2, cc, T * hop, 400 + i, fmt), T, hop)
    for i, (T, hop) in enumerate([(2, 97), (5, 800), (1, 3000)]):
        y = _samples(5, cc, T * hop, 450 + i, fmt)
        assert_bits_equal(dst.process(y, T, hop, **want), twin.process(y, T, hop, **want), ("busy", i))
    clk = src.get_clock()
    assert clk != dst.get_clock()
    dst.set_state(src.get_state(), first_stream=1)
    dst.set_clock(clk)
    twin.set_clock(clk)
    for i, (T, hop) in enumerate([(3, 800), (6, 7), (2, 800)]):
        x = _samples(2, cc, T * hop, 500 + i, fmt)
        y = _samples(5, cc, T * hop, 550 + i, fmt)
        y[1:3] = x
        got = dst.process(y, T, hop, **want)
        assert_bits_equal(_slots(got, 1, 3), src.process(x, T, hop, **want), ("moved", i))
        other = twin.process(y, T, hop, **want)
        for lo, hi in ((0, 1), (3, 5)):
            assert_bits_equal(_slots(got, lo, hi), _slots(other, lo, hi), ("others", i, lo))


# ---- graphs -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hop", [800, 700], ids=["one-pass", "general"])
def test_meter_graph_replays_read_restored_state(hop):
    """A captured meter call, with set_state between replays: the state of a donor engine that ran other audio.  Restores
    come after an odd and after an even number of replays (the graph's engine then reads the second and the first ring
    half), with the captured call's partials valid for its hop.  Every replay equals the eager call of a twin restored the
    same way; a replay right after a restore also equals the donor's own next call on the same input."""
    import torch
    from waveform_b200 import MeterEngine

    S, T, cc = 3, 3, 2
    settings = {"rms_mode": True, "audio_sync_offset": 30}
    a, b, donor = (MeterEngine(settings, channels=cc, max_streams=S) for _ in range(3))
    xin = torch.zeros((S, cc, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, want_pixels=True))
    for i in range(7):
        restore = i in (1, 4)  # after 1 and after 4 replays
        if restore:
            st = donor.get_state()
            a.set_state(st)
            b.set_state(st)
        else:
            donor.process(_samples(S, cc, 5 * hop, 600 + i, "f32"), 5, hop)
        x = _samples(S, cc, T * hop, 650 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(out, b.process(x, T, hop, want_pixels=True), ("replay", i))
        if restore:
            assert_bits_equal(out, donor.process(x, T, hop, want_pixels=True), ("donor", i))
    assert_bits_equal(a.get_state(), b.get_state(), "final")


def test_wave_graph_replays_read_restored_state_and_clock():
    """A captured device-clock waveform call, with set_state / set_clock between replays (a donor's slots and clock): every
    replay equals the eager call of a host-clock twin restored the same way, and a replay right after a restore also
    equals the donor's own next call on the same input."""
    import torch
    from waveform_b200 import WaveEngine

    S, T, hop, cc = 2, 2, 800, 2
    settings = {"width": 800, "meter_buf": 150, "audio_sync_offset": 40}
    a = WaveEngine(settings, channels=cc, max_streams=S, device_clock=True)
    b, donor = (WaveEngine(settings, channels=cc, max_streams=S) for _ in range(2))
    xin = torch.zeros((S, cc, T * hop), device="cuda")
    g, out = capture(lambda: a.process(xin, T, hop, want_pixels=True))
    for i in range(7):
        restore = i in (1, 4)
        if restore:
            st, clk = donor.get_state(), donor.get_clock()
            for e in (a, b):
                e.set_state(st)
                e.set_clock(clk)
        else:
            donor.process(_samples(S, cc, (1 + i) * 441, 700 + i, "f32"), 1 + i, 441)
        x = _samples(S, cc, T * hop, 750 + i, "f32")
        replay(g, [xin], [x])
        assert_bits_equal(out, b.process(x, T, hop, want_pixels=True), ("replay", i))
        if restore:
            assert_bits_equal(out, donor.process(x, T, hop, want_pixels=True), ("donor", i))
        assert a.get_clock() == b.get_clock()


# ---- round trips, defaults, resets, refusals ---------------------------------------------------------------------------

def test_round_trips_change_nothing():
    from waveform_b200 import MeterEngine, WaveEngine

    m, mt = (MeterEngine({"audio_sync_offset": 40}, channels=2, max_streams=3) for _ in range(2))
    w, wt = (WaveEngine({"width": 300, "meter_buf": 50, "audio_sync_offset": 40}, channels=2, max_streams=3,
                        device_clock=c) for c in (True, False))
    for i, (T, hop) in enumerate([(4, 800), (3, 900), (5, 7)]):
        x = _samples(3, 2, T * hop, 800 + i, "f32")
        assert_bits_equal(m.process(x, T, hop, want_pixels=True), mt.process(x, T, hop, want_pixels=True), ("meter", i))
        assert_bits_equal(w.process(x, T, hop), wt.process(x, T, hop), ("wave", i))
        m.set_state(m.get_state())
        m.set_state(m.get_state(1, 1), first_stream=1)
        w.set_state(w.get_state())
        w.set_clock(w.get_clock())
    assert_bits_equal(m.get_state(), mt.get_state(), "meter")
    assert_bits_equal(w.get_state(), wt.get_state(), "wave")


def test_fresh_state_and_resets():
    from waveform_b200 import MeterEngine, WaveEngine

    dbmin = _db_min()
    # without smoothing: with it the DB_MIN start-up value drives the EMA negative, and the first calls are silent
    m = MeterEngine({"audio_sync_offset": 40, "temporal_smoothing": "none"}, channels=2, max_streams=3)
    st = m.get_state()
    assert st["ring"].shape == (3, 2, m.window) and st["line"].shape == (3, 2, 1920)
    assert not st["ring"].any() and not st["line"].any() and not st["flags"].any()
    assert np.array_equal(st["ema"], np.full((3, 2), dbmin, np.float32))  # m_meter_buf := DB_MIN at start-up (sic)
    x = _samples(3, 2, 4 * 800, 900, "f32")
    m.process(x, 4, 800)
    before = m.get_state()
    assert before["line"].any() and not before["flags"].any()
    m.reset(1, 1)
    after = m.get_state()
    assert not after["ring"][1].any() and not after["ema"][1].any() and after["flags"][1] == 1
    assert np.array_equal(after["line"], before["line"])  # the reset leaves the delay lines alone
    for k in ("ring", "ema", "flags"):
        assert np.array_equal(after[k][[0, 2]], before[k][[0, 2]]), k
    # wf_meter_window floats per channel, oldest first: the ring is the newest samples of line ++ pcm
    full = np.concatenate([np.zeros((3, 2, m.window + 1920), np.float32), x], axis=2)
    assert np.array_equal(before["ring"][0], full[0, :, -1920 - m.window:-1920])
    assert np.array_equal(before["line"][0], full[0, :, -1920:])
    feed = MeterEngine({}, channels=2, max_streams=1, mode=2)
    assert feed.get_state()["ema"] is None

    for clock in (False, True):
        w = WaveEngine({"width": 300, "meter_buf": 50, "channel_mode": "stereo", "audio_sync_offset": 40}, channels=2,
                       max_streams=2, device_clock=clock)
        st = w.get_state()
        assert st["db"].shape == (2, 2, 300) and st["hold"].shape == (2, 2, 1920)
        assert np.array_equal(st["db"], np.full((2, 2, 300), dbmin, np.float32))
        assert not st["hold"].any() and not st["flags"].any()
        assert w.get_clock() == {"clock_ns": 10 ** 10, "audio_ts": 0, "waveform_ts": 0, "buffered": 300}
        x = _samples(2, 2, 3 * 800, 910, "f32")
        out = w.process(x, 3, 800)
        st = w.get_state()
        assert np.array_equal(bits(st["db"]), bits(out["out"][:, -1]))  # the last tick's rows
        assert np.array_equal(st["hold"], x[:, :, -1920:])
        w.reset()
        st = w.get_state()
        assert np.array_equal(st["db"], np.full((2, 2, 300), dbmin, np.float32)) and st["flags"].all()
    mono = WaveEngine({"width": 300}, channels=1, max_streams=1)
    assert mono.get_state()["db"].shape == (1, 1, 300) and mono.get_state()["hold"].shape == (1, 1, 0)


def test_out_of_range_and_refused_clocks_change_nothing():
    from waveform_b200 import MeterEngine, WaveEngine
    from waveform_b200.engine import WF_ERR_CAPACITY, WF_ERR_INVALID_ARG, WfError

    m, mt = (MeterEngine({}, channels=2, max_streams=3) for _ in range(2))
    w, wt = (WaveEngine({"width": 300, "meter_buf": 50, "audio_sync_offset": 10}, channels=2, max_streams=3,
                        device_clock=c) for c in (True, False))
    x = _samples(3, 2, 3 * 800, 950, "f32")
    m.process(x, 3, 800)
    mt.process(x, 3, 800)
    w.process(x, 3, 800)
    wt.process(x, 3, 800)
    for e in (m, w):
        for first, count in ((3, 1), (-1, 1), (2, 2), (0, 4)):
            with pytest.raises(WfError) as ei:
                e.get_state(first, count)
            assert ei.value.status == WF_ERR_CAPACITY
        with pytest.raises(WfError) as ei:
            e.set_state(e.get_state(1, 2), first_stream=2)
        assert ei.value.status == WF_ERR_CAPACITY
    clk = w.get_clock()
    step = 50 * 1000000 // 300
    D_ns = SR * 10 // 1000 * 10 ** 9 // SR
    bad = [{**clk, "buffered": max(300, 480) + 1},                          # more than the walk keeps
           {**clk, "audio_ts": clk["audio_ts"] + 1},                        # audio_ts != clock
           {**clk, "waveform_ts": clk["audio_ts"] - D_ns + step + 1},       # beyond one step past the stop
           {**clk, "audio_ts": 0, "clock_ns": clk["clock_ns"]},            # "no tick yet" with a moved waveform_ts
           {"clock_ns": 10 ** 10 + 5, "audio_ts": 0, "waveform_ts": 0, "buffered": 300},  # "no tick yet", moved clock
           {"clock_ns": 5, "audio_ts": 5, "waveform_ts": 0, "buffered": 480}]            # below the 10 s start
    for c in bad:
        for e in (w, wt):
            with pytest.raises(WfError) as ei:
                e.set_clock(c)
            assert ei.value.status == WF_ERR_INVALID_ARG
    assert w.get_clock() == clk == wt.get_clock()
    # exactly one step past the stop is a clock the walk can leave: the host walk and the device planner take it alike,
    # through ticks that emit nothing (hop 1: the stop stays within a step of waveform_ts) and ticks that emit
    edge = {**clk, "waveform_ts": clk["audio_ts"] - D_ns + step}
    w2, w3 = (WaveEngine({"width": 300, "meter_buf": 50, "audio_sync_offset": 10}, channels=2, max_streams=3,
                         device_clock=c) for c in (False, True))
    for e in (w2, w3):
        e.set_clock({"clock_ns": 10 ** 10, "audio_ts": 0, "waveform_ts": 0, "buffered": 300})  # a fresh engine's clock
        e.set_clock(edge)
    for i, (T, hop) in enumerate([(3, 1), (2, 800)]):
        z = _samples(3, 2, T * hop, 970 + i, "f32")
        assert_bits_equal(w3.process(z, T, hop, want_pixels=True), w2.process(z, T, hop, want_pixels=True), ("edge", i))
        assert w3.get_clock() == w2.get_clock()
        if i == 0:
            assert w2.get_clock()["waveform_ts"] == edge["waveform_ts"]  # no points yet: the clock's waveform_ts stayed
    assert_bits_equal(m.get_state(), mt.get_state(), "meter")
    y = _samples(3, 2, 4 * 800, 960, "f32")
    assert_bits_equal(w.process(y, 4, 800), wt.process(y, 4, 800), "after refusals")
    assert_bits_equal(m.process(y, 4, 800), mt.process(y, 4, 800), "meter after refusals")
