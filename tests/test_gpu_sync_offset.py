"""The audio sync offset (sync_offset_ms of wf_config / wf_meter_config / wf_wave_config) on the GPU.

Each engine's offset has an exact reference that needs no offset at all:
  * spectrum ring calls: plain calls over zeros(N + D) ++ samples on the delayed frames, with the start-up ticks (fewer
    than D samples arrived) passed as skip_mask;
  * level meter and RMS feed: the engine without an offset fed zeros(D) ++ stream;
and the compiled plugin fed packet by packet with its audio_sync_offset setting checks the models themselves (as
tests/test_sync_offset_cpu.py does on the CPU).  An offset <= 0, or a config of the previous size, gives today's bits.

Run on an H100:  python -m pytest tests/test_gpu_sync_offset.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from gpu_common import assert_bits_equal, bits, clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]
SR = 48000


def _delay(ms):
    return SR * ms // 1000 if ms > 0 else 0


def _signal(S, cc, n, seed, s16):
    x = synth_pcm(S, cc, n, seed=seed)
    x[:, :, n // 3: n // 3 + n // 5] = 0.0  # digital silence: the gate and m_last_silent
    return np.round(x * 32767.0).astype(np.int16) if s16 else x.astype(np.float32)


# ---- spectrum ------------------------------------------------------------------------------------------------------

def _feed(kind, fmt):
    import torch

    def feed(eng, pcm, T_, hop, ring, first_stream=0, skip=None):
        if kind == "device":
            o = eng.process(torch.from_numpy(pcm).cuda(), T_, hop, pcm_format=fmt, capture_ring=ring, want_peak=True,
                            first_stream=first_stream, skip_mask=None if skip is None else torch.from_numpy(skip).cuda())
            torch.cuda.synchronize()
            return {k: v.cpu().numpy() for k, v in o.items()}
        if kind == "pinned":
            pcm = torch.from_numpy(pcm).pin_memory().numpy()
        return dict(eng.process(pcm, T_, hop, pcm_format=fmt, capture_ring=ring, want_peak=True,
                                first_stream=first_stream, skip_mask=skip))
    return feed


def _spectrum_pair(settings, cc, S, calls, x, ms, feed, caller_mask=None, first_stream=0, max_streams=None):
    """Ring calls with the offset on one engine, plain calls on the delayed frames (start-up ticks as skip_mask) on
    another; asserts per call that outputs, kernel names, state and ring agree bit for bit."""
    from waveform_b200 import Engine

    ms_ = max_streams or S
    ring_eng = Engine({**settings, "audio_sync_offset": ms}, channels=cc, max_streams=ms_)
    plain_eng = Engine(settings, channels=cc, max_streams=ms_)
    N, D = ring_eng.fft_size, _delay(ms)
    assert ring_eng.sync_delay == D
    full = np.concatenate([np.zeros((S, cc, N + D), x.dtype), x], axis=2)
    pos = 0
    for i, (T_, hop) in enumerate(calls):
        new = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
        p0 = pos + hop
        plain = np.ascontiguousarray(full[:, :, p0: p0 + (T_ - 1) * hop + N])
        start = np.array([pos + (t + 1) * hop < D for t in range(T_)], np.uint8)[None, :].repeat(S, 0)
        caller = None if caller_mask is None else caller_mask(i, S, T_)
        ring_mask = caller
        plain_mask = None
        if pos < D or caller is not None:  # a ring call still owed samples skips through a mask: so does its reference
            plain_mask = start | (0 if caller is None else caller)
        got = feed(ring_eng, new, T_, hop, True, first_stream, ring_mask)
        want = feed(plain_eng, plain, T_, hop, False, first_stream, plain_mask)
        ctx = (settings, ms, T_, hop)
        assert_bits_equal(got, want, ctx)
        assert ring_eng.last_kernel_name() == plain_eng.last_kernel_name() + " ring", ctx
        assert_bits_equal(ring_eng.get_state(), plain_eng.get_state(), ctx)
        pos += T_ * hop
        want_ring = full[:, :, pos: pos + N + D].astype(np.float32)
        if x.dtype == np.int16:
            want_ring *= np.float32(2.0 ** -15)
        assert np.array_equal(ring_eng.get_ring(first_stream, S), want_ring), ctx
    return ring_eng


SPECTRUM = [(800, 1, False, "hann", "stft_warp2_kernel"), (2048, 1, False, "hann", "stft2048_"),
            (4096, 2, True, "blackman_harris", "stft_v3_kernel<4096,2,")]


def _calls(N):
    return [(3, 800), (1, 800), (2, N), (1, N + 400), (4, 512), (6, 1600), (2, 304), (1, N + 48000)]


@pytest.mark.parametrize("ms", [10, 170, 1000])
@pytest.mark.parametrize("kind", ["device", "host", "pinned"])
@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("N,cc,stereo,window,family", SPECTRUM)
def test_spectrum_ring_offset_equals_plain_on_delayed_frames(N, cc, stereo, window, family, fmt, kind, ms):
    """Start-up across several calls (D up to 48000 samples), hops below, at and above N and above N + D, silence inside."""
    settings = {"fft_size": N, "window": window, "silence_gate": True}
    if stereo:
        settings["channel_mode"] = "stereo"
    calls = _calls(N)
    x = _signal(3, cc, sum(t * h for t, h in calls), 11 + N + ms, fmt == "s16")
    eng = _spectrum_pair(settings, cc, 3, calls, x, ms, _feed(kind, fmt))
    assert eng.last_kernel_name().startswith(family) or family in eng.last_kernel_name()


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_spectrum_offset_caller_mask_and_slot_ranges(fmt):
    """The caller's skip_mask ORed with the start-up ticks; calls on slots [2, 5) of 8 leave the other slots alone."""
    rng = np.random.default_rng(5)

    def caller(i, S, T_):
        return (rng.uniform(size=(S, T_)) < 0.3).astype(np.uint8)

    calls = [(4, 800), (3, 800), (5, 1024), (2, 4000)]
    x = _signal(3, 1, sum(t * h for t, h in calls), 17, fmt == "s16")
    eng = _spectrum_pair({"fft_size": 2048, "silence_gate": True}, 1, 3, calls, x, 100, _feed("device", fmt),
                         caller_mask=caller, first_stream=2, max_streams=8)
    D = _delay(100)
    untouched = eng.get_ring()[[0, 1, 5, 6, 7]]
    assert untouched.shape == (5, 1, 2048 + D) and not untouched.any()
    eng.reset_state()  # leaves rings and start-up counts alone
    assert eng.get_ring(2, 3).shape == (3, 1, 2048 + D)


def test_spectrum_offset_set_ring_primes():
    """set_ring with N + D samples of real audio clears the start-up count: the next ring call skips nothing and equals a
    plain call over the primed audio."""
    import torch
    from waveform_b200 import Engine

    N, ms, hop, T_ = 2048, 170, 800, 6
    D = _delay(ms)
    settings = {"fft_size": N, "silence_gate": True}
    x = _signal(2, 1, N + D + T_ * hop, 31, False)
    ring = Engine({**settings, "audio_sync_offset": ms}, channels=1, max_streams=2)
    ring.set_ring(x[:, :, : N + D])
    got = ring.process(torch.from_numpy(x[:, :, N + D:]).contiguous().cuda(), T_, hop, capture_ring=True)
    plain = Engine(settings, channels=1, max_streams=2)
    want = plain.process(torch.from_numpy(x[:, :, hop: hop + (T_ - 1) * hop + N]).contiguous().cuda(), T_, hop)
    torch.cuda.synchronize()
    assert torch.equal(got["db"].view(torch.int32), want["db"].view(torch.int32))
    assert ring.last_kernel_name() == plain.last_kernel_name() + " ring"
    assert np.array_equal(ring.get_ring(), x[:, :, -(N + D):])
    with pytest.raises(ValueError):
        ring.set_ring(x[:, :, :N])


def test_spectrum_offset_mapped_buffers():
    """wf_host_alloc (zero-copy) live ticks with an offset give the device path's bits."""
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import load_library

    N, cc, ms = 2048, 1, 170
    settings = {"fft_size": N, "silence_gate": True, "audio_sync_offset": ms}
    calls = [(1, 800)] * 12 + [(2, 1600), (1, 4000)]
    x = _signal(1, cc, sum(t * h for t, h in calls), 41, False)
    L = load_library()
    dev = Engine(settings, channels=cc, max_streams=1)
    mapped = Engine(settings, channels=cc, max_streams=1)
    B = dev.bins
    cap = max(t * h for t, h in calls)
    pin, pout, psil = L.wf_host_alloc(cc * cap * 4), L.wf_host_alloc(4 * B * 4), L.wf_host_alloc(16)
    assert pin and pout and psil
    try:
        pos = 0
        for T_, hop in calls:
            new = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
            pos += T_ * hop
            o = dev.process(torch.from_numpy(new).cuda(), T_, hop, capture_ring=True)
            torch.cuda.synchronize()
            C.memmove(pin, new.ctypes.data, new.nbytes)
            mapped.process_raw(pin, 1, T_, hop, cc * T_ * hop, T_ * hop, out_db=pout, out_silent=psil, capture_ring=True)
            db = np.frombuffer((C.c_float * (T_ * B)).from_address(pout), np.float32).reshape(o["db"].shape)
            sil = np.frombuffer((C.c_uint8 * T_).from_address(psil), np.uint8).reshape(o["silent"].shape)
            assert np.array_equal(db.view(np.uint32), o["db"].cpu().numpy().view(np.uint32)), (T_, hop)
            assert np.array_equal(sil, o["silent"].cpu().numpy())
        assert np.array_equal(mapped.get_ring(), dev.get_ring())
    finally:
        for q in (pin, pout, psil):
            L.wf_host_free(q)


@pytest.mark.parametrize("ms", [10, 1000])
@pytest.mark.parametrize("N,cc,stereo,window", [(800, 1, False, "hann"), (2048, 1, False, "hann"),
                                                 (4096, 2, True, "blackman_harris")])
def test_spectrum_offset_against_the_plugin(N, cc, stereo, window, ms):
    """Ring calls with the offset against the compiled plugin fed packet by packet with audio_sync_offset, within the
    parity tolerance of tests/test_gpu_ring.py."""
    import torch
    from oracle import refbind
    from helpers import parity_report
    from waveform_b200 import Engine

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    settings = {"fft_size": N, "window": window, "silence_gate": True, "audio_sync_offset": ms}
    if stereo:
        settings["channel_mode"] = "stereo"
    calls = _calls(N)[:-1]
    x = _signal(1, cc, sum(t * h for t, h in calls), 51 + N, False)[0]
    pk = refbind.RefSource(settings, channels=cc)
    eng = Engine(settings, channels=cc, max_streams=1)
    dch = pk.display_channels
    pos = 0
    for T_, hop in calls:
        want, sil = [], []
        for t in range(T_):
            seg = x[:, pos + t * hop: pos + (t + 1) * hop]
            pk.advance(hop / pk.sample_rate)
            pk.push(seg[0], seg[1] if cc == 2 else None)
            pk.tick(1.0 / 60.0)
            want.append(np.stack([pk.decibels(c) for c in range(dch)]))
            sil.append(1 if pk.last_silent else 0)
        o = eng.process(torch.from_numpy(np.ascontiguousarray(x[None, :, pos: pos + T_ * hop])).cuda(), T_, hop,
                        capture_ring=True)
        got = o["db"][0].cpu().numpy()
        rep = parity_report(got, np.stack(want))
        assert rep["ok"], (N, ms, T_, hop, rep)
        assert np.array_equal(o["silent"][0].cpu().numpy(), np.array(sil, np.uint8)), (N, ms, T_, hop)
        pos += T_ * hop


@pytest.mark.parametrize("ms", [0, -500])
def test_spectrum_no_offset_is_todays_call(ms):
    """An offset <= 0 and a config of the previous size: same bits, kernel names and launches as no offset at all."""
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import WfConfig

    settings = {"fft_size": 2048, "silence_gate": True}
    x = _signal(4, 1, 6 * 800, 61, False)
    engines = [Engine(settings, channels=1, max_streams=4), Engine({**settings, "audio_sync_offset": ms}, channels=1,
                                                                   max_streams=4)]
    cfg = WfConfig.from_buffer_copy(engines[0].cfg)
    cfg.sync_offset_ms = 700  # beyond the previous struct's end: never read
    cfg.struct_size = WfConfig.sync_offset_ms.offset
    engines.append(Engine(config=cfg))
    outs, names, launches = [], [], []
    for e in engines:
        l0 = e.L.wf_launch_count(e.h)
        o = [e.process(torch.from_numpy(x[:, :, i * 1600: (i + 1) * 1600]).cuda(), 2, 800, capture_ring=True)
             for i in range(3)]
        torch.cuda.synchronize()
        outs.append(np.concatenate([oo["db"].cpu().numpy() for oo in o], axis=1))
        names.append(e.last_kernel_name())
        launches.append(e.L.wf_launch_count(e.h) - l0)
        assert e.get_ring().shape == (4, 1, 2048)
    assert all(np.array_equal(bits(o), bits(outs[0])) for o in outs)
    assert len(set(names)) == 1 and len(set(launches)) == 1


# ---- level meter and RMS feed ----------------------------------------------------------------------------------------

METER = [("peak", {"rms_mode": False, "meter_buf": 100}, 2, None), ("rms", {"rms_mode": True, "meter_buf": 150}, 2, None),
         ("rms-mono", {"rms_mode": True, "meter_buf": 20}, 1, None), ("feed", {}, 2, 2)]


@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("ms", [10, 170, 1000])
@pytest.mark.parametrize("name,settings,cc,mode", METER, ids=[m[0] for m in METER])
def test_meter_offset_is_a_zero_prefixed_stream(name, settings, cc, mode, ms, fmt):
    """Bit for bit the engine without an offset fed zeros(D) ++ stream, across calls, hops (4-aligned or not) and slot
    ranges, on device and host buffers."""
    import torch
    from waveform_b200 import MeterEngine

    D = _delay(ms)
    S = 5
    calls = [(5, 480), (3, 800), (2, 4800), (1, 9000), (7, 333), (4, 2048)]
    x = _signal(S, cc, sum(t * h for t, h in calls), 71 + ms, fmt == "s16")
    xd = np.concatenate([np.zeros((S, cc, D), x.dtype), x], axis=2)
    a = MeterEngine({**settings, "audio_sync_offset": ms}, channels=cc, max_streams=S + 2, mode=mode)
    b = MeterEngine(settings, channels=cc, max_streams=S + 2, mode=mode)
    pos = 0
    for i, (T_, hop) in enumerate(calls):
        pa = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
        pb = np.ascontiguousarray(xd[:, :, pos: pos + T_ * hop])
        if i % 2:
            ga = a.process(pa, T_, hop, first_stream=1, pcm_format=fmt)
            gb = b.process(pb, T_, hop, first_stream=1, pcm_format=fmt)
        else:
            ga = {k: v.cpu().numpy() for k, v in a.process(torch.from_numpy(pa).cuda(), T_, hop, first_stream=1,
                                                          pcm_format=fmt).items()}
            gb = {k: v.cpu().numpy() for k, v in b.process(torch.from_numpy(pb).cuda(), T_, hop, first_stream=1,
                                                          pcm_format=fmt).items()}
            torch.cuda.synchronize()
        assert_bits_equal(ga, gb, (name, ms, T_, hop))
        pos += T_ * hop
    a.reset(0, 3)  # leaves the delay lines alone: the next call still starts with the held-back samples
    b.reset(0, 3)
    ga = a.process(np.ascontiguousarray(x[:, :, :1600]), 2, 800, first_stream=1, pcm_format=fmt)
    held = np.concatenate([xd[:, :, pos: pos + D], x[:, :, :1600]], axis=2)  # the line: the last D samples so far
    gb = b.process(np.ascontiguousarray(held[:, :, :1600]), 2, 800, first_stream=1, pcm_format=fmt)
    assert_bits_equal(ga, gb, (name, ms, "after reset"))


@pytest.mark.parametrize("ms", [10, 1000])
@pytest.mark.parametrize("rms", [False, True])
def test_meter_offset_against_the_plugin(rms, ms):
    """PEAK values exactly, RMS within the existing 1e-5 relative, against the plugin fed packet by packet with audio_sync_offset."""
    from oracle import refbind
    from waveform_b200 import MeterEngine

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    settings = {"rms_mode": rms, "meter_buf": 150, "audio_sync_offset": ms}
    calls = [(5, 480), (3, 800), (2, 4800), (7, 333), (4, 2048)]
    x = _signal(1, 2, sum(t * h for t, h in calls), 81, False)
    ref = refbind.RefSource({"display_mode": "level_meter", **settings}, channels=2)
    eng = MeterEngine(settings, channels=2)
    pos = 0
    for T_, hop in calls:
        w = ref.run_meter(x[0, :, pos: pos + T_ * hop], T_, hop)
        g = eng.process(np.ascontiguousarray(x[:, :, pos: pos + T_ * hop]), T_, hop)
        if rms:
            np.testing.assert_allclose(g["lin"][0], w["lin"], rtol=1e-5, atol=0)  # tests/test_meter.py's RMS_TOL
        else:
            assert np.array_equal(g["lin"][0], w["lin"])  # the peaks; their dBFS goes through log10f (last-bit differences)
            assert np.max(np.abs(g["db"][0] - w["db"])) < 1e-4
        assert np.array_equal(g["silent"][0], w["silent"])
        pos += T_ * hop


def test_meter_no_offset_is_todays_call():
    from waveform_b200 import MeterEngine

    x = _signal(3, 2, 10 * 800, 91, False)
    outs, launches = [], []
    for ms in (None, 0, -1000):
        e = MeterEngine({} if ms is None else {"audio_sync_offset": ms}, channels=2, max_streams=3)
        l0 = e.L.wf_meter_launch_count(e.h)
        outs.append(e.process(x, 10, 800))
        launches.append(e.L.wf_meter_launch_count(e.h) - l0)
    for o in outs[1:]:
        assert_bits_equal(o, outs[0], "no offset")
    assert len(set(launches)) == 1


# ---- waveform --------------------------------------------------------------------------------------------------------

WAVE = [({"width": 800, "meter_buf": 150}, 2), ({"width": 800, "meter_buf": 150, "channel_mode": "stereo"}, 2),
        ({"width": 300, "meter_buf": 50}, 1), ({"width": 640, "meter_buf": 500, "channel_mode": "stereo"}, 1)]


@pytest.mark.parametrize("ms", [10, 170, 1000])
@pytest.mark.parametrize("settings,cc", WAVE)
def test_wave_offset_against_the_plugin(settings, cc, ms):
    """D below and above the buffered span (m_waveform_samples), changing hops, two calls per hop, with display
    outputs: the plugin's point pattern and silent flags exactly, dB values to 1e-4 dB (tests/test_wave.py)."""
    from oracle import refbind
    from waveform_b200 import WaveEngine

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    S = 2
    calls = [(6, 480), (5, 800), (1, 4800), (12, 97), (8, 2000), (3, 441)]
    x = _signal(S, cc, sum(t * h for t, h in calls), 101 + ms, False)
    x[1, :, 2000: 9000] = 1.0
    refs = [refbind.RefSource({"display_mode": "waveform", **settings, "audio_sync_offset": ms}, channels=cc)
            for _ in range(S)]
    eng = WaveEngine({**settings, "audio_sync_offset": ms}, channels=cc, max_streams=S)
    pos = 0
    for T_, hop in calls:
        want = [r.run_wave(x[s, :, pos: pos + T_ * hop], T_, hop) for s, r in enumerate(refs)]
        ref = np.stack([w["out"] for w in want])
        ref_sil = np.stack([w["silent"] for w in want])
        o = eng.process(np.ascontiguousarray(x[:, :, pos: pos + T_ * hop]), T_, hop, want_points=True, want_pixels=True)
        out, sil = o["out"], o["silent"]
        assert np.array_equal(sil, ref_sil), (ms, hop)
        lo = ref < -700.0
        assert np.array_equal(out < -700.0, lo), (ms, hop)
        untouched = ref == np.float32(-758.59564)
        assert np.array_equal(out[untouched], ref[untouched])
        assert np.max(np.abs(out[~lo] - ref[~lo]), initial=0.0) < 1e-4, (ms, hop)
        pos += T_ * hop


@pytest.mark.parametrize("s16", [False, True])
@pytest.mark.parametrize("settings,cc", WAVE)
def test_wave_offset_chunked_and_per_tick_kernels_agree(settings, cc, s16, monkeypatch):
    import torch
    from waveform_b200 import WaveEngine

    S, ms = 5, 170
    calls = [(13, 480), (40, 800), (2, 4800)]
    x = _signal(S, cc, sum(t * h for t, h in calls), 111, s16)
    fmt = "s16" if s16 else "f32"
    outs = {}
    for chunk in ("1", "0"):
        set_knobs(monkeypatch, {"WF_WAVE_CHUNK": chunk})
        eng = WaveEngine({**settings, "audio_sync_offset": ms}, channels=cc, max_streams=S)
        pos, got = 0, []
        for T_, hop in calls:
            o = eng.process(torch.from_numpy(np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])).cuda(), T_, hop,
                            want_points=True, want_pixels=True, pcm_format=fmt)
            torch.cuda.synchronize()
            got.append({k: v.cpu().numpy() for k, v in o.items()})
            pos += T_ * hop
        outs[chunk] = got
    for a, b in zip(outs["1"], outs["0"]):
        assert_bits_equal(a, b, "chunked vs per-tick")


def test_wave_no_offset_is_todays_call():
    from waveform_b200 import WaveEngine

    x = _signal(2, 2, 30 * 800, 121, False)
    outs, launches = [], []
    for ms in (None, 0, -20):
        e = WaveEngine({"width": 800} if ms is None else {"width": 800, "audio_sync_offset": ms}, channels=2, max_streams=2)
        l0 = e.L.wf_wave_launch_count(e.h)
        outs.append(e.process(x, 30, 800, want_points=True))
        launches.append(e.L.wf_wave_launch_count(e.h) - l0)
    for o in outs[1:]:
        assert_bits_equal(o, outs[0], "no offset")
    assert len(set(launches)) == 1
