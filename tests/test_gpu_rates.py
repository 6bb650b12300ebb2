"""Every engine at 44.1 kHz and at the automatic FFT sizes of the common frame rates, on the GPU.

The grid, sizes and tick counts are tests/test_rates_cpu.py's.  At 44.1 kHz the plugin's tick brings more samples than the
automatic size (735 > 720 at 60 fps), so a capture-ring call reads each frame in place hop - N samples into its tick, at
an odd offset whenever the hop is odd; several automatic sizes (1824, 1760, 912, 432, 304, 176, 2000, 992) have no
warp-per-stream plan and run on stft_anyn_kernel with radices 3, 5, 11, 19 and 31; the 150 ms meter window (6608) is no
multiple of the hop; the waveform's clock runs on 44100.

Run on an H100:  python -m pytest tests/test_gpu_rates.py -m gpu -q
"""
from __future__ import annotations

import subprocess
from pathlib import Path

import numpy as np
import pytest

from fp64_spectrum import Fp64Spectrum, compare
from gpu_common import clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import parity_report, synth_pcm
from refdata import frame_peak, reference, sample_index
from test_rates_cpu import FPS, GRID, auto_size, fps_value, frames_to_ns, grid_id, sync_delay, tick_counts

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]
ROOT = Path(__file__).resolve().parents[1]

# ---- routing: the rule of wf_engine.cu choose_route, restated for these sizes -------------------------------------------

# sizes with a compiled warp-per-stream plan (wf_warp2_*.cu)
WARP2_SIZES = {192, 288, 320, 352, 384, 400, 448, 480, 512, 528, 576, 640, 704, 720, 768, 800, 832, 880, 896, 960, 1024,
               1152, 1280, 1344, 1408, 1456, 1536, 1600, 1664, 1728, 1792, 1920, 2048}
POW2_SIZES = {128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768}


def expected_kernel(N, cc, stereo, hop):
    """The start of the kernel name a spectrum call without display outputs runs.  A non-power-of-two size goes to the
    warp-per-stream kernel when it has a plan, the call is one-channel mono and its frames are 16-byte aligned (hop a
    multiple of 4 samples: the strides and a ring call's in-place offset hop - N then are too), else to the any-N kernel."""
    if N in POW2_SIZES:
        return ("stft_fused_kernel<", "stft_wide_kernel<")
    if cc == 1 and not stereo and hop % 4 == 0 and N in WARP2_SIZES:
        return ("stft_warp2_kernel<",)
    return (f"stft_anyn_kernel<{cc}> N={N}",)


def test_routing_rule_facts():
    """No GPU needed: the any-N sizes of the grid are the ones without a warp-per-stream plan, and every 44.1 kHz hop of
    60 fps and 59.94 fps that is odd keeps one-channel 720 off the warp-per-stream kernel."""
    anyn = sorted({auto_size(sr, f) for sr, f in GRID} - WARP2_SIZES - POW2_SIZES)
    assert anyn == [176, 304, 432, 912, 992, 1760, 1824, 2000]
    assert expected_kernel(720, 1, False, 735)[0].startswith("stft_anyn_kernel<1>")
    assert expected_kernel(720, 1, False, 736) == ("stft_warp2_kernel<",)
    assert expected_kernel(720, 2, False, 736)[0].startswith("stft_anyn_kernel<2>")


# ---- 1. spectrum at every automatic size ----------------------------------------------------------------------------------

LAYOUTS = {"one": (1, False), "mix": (2, False), "stereo": (2, True)}
S = 3
SEEN: dict[tuple, str] = {}      # (rate, fps, layout, mode, hop) -> kernel name


def _spectrum_settings(N, all_options, stereo):
    s = {"fft_size": N, "window": "hann", "silence_gate": True}
    if all_options:
        s = {"fft_size": N, "window": "blackman_harris", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0,
             "fast_peaks": True, "normalize_volume": True, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5}
    if stereo:
        s["channel_mode"] = "stereo"
    return s


def _grid_calls(sr, fps):
    """(ticks, hop) per call: the frame rate's tick counts alternating across calls (the same hop throughout at an integer
    rate)."""
    hops = sorted(set(tick_counts(sr, fps, 1001)))
    a, b = hops[0], hops[-1]
    return [(3, a), (2, b), (1, a), (4, b)] if a != b else [(3, a), (2, a), (1, a), (4, a)]


def _grid_signal(N, cc, n, seed):
    x = synth_pcm(S, cc, n, seed=seed)
    x[1, :, n // 3: n // 3 + 2 * N + 1500] = 0.0        # a silence stretch longer than two frames: the gate and the hold
    if cc == 2:
        x[2, 1, n // 2:] = 0.0                           # one channel goes quiet
    x[2] *= np.float32(2.0 ** -12)
    return x


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("point", GRID, ids=[grid_id(p) for p in GRID])
def test_spectrum_at_the_automatic_size(point, layout):
    """Plain device calls, host (numpy) calls and capture-ring calls over the same frames, plain and all options, with
    seconds = 1 / fps: each stream within 1e-6 of float64 (fp64_spectrum.compare) with the same silent flags, the ring
    calls bit for bit the plain device calls, and each call on the kernel the routing rule names."""
    import torch
    from waveform_b200 import Engine

    sr, fps = point
    cc, stereo = LAYOUTS[layout]
    N = auto_size(sr, fps)
    seconds = 1.0 / fps_value(fps)
    calls = _grid_calls(sr, fps)
    T = sum(t for t, _ in calls)
    total = sum(t * h for t, h in calls)
    x = _grid_signal(N, cc, total, 0x44 + N + cc)
    full = np.concatenate([np.zeros((S, cc, N), np.float32), x], axis=2)     # the ring's start-up zeros ++ the stream
    worst = 0.0
    for all_opt in (False, True):
        settings = _spectrum_settings(N, all_opt, stereo)
        rms = (0.02 + 0.3 * np.random.default_rng(N).uniform(size=(S, T))).astype(np.float32) if all_opt else None
        engines = {m: Engine(settings, sample_rate=sr, channels=cc, max_streams=S) for m in ("device", "host", "ring")}
        g = np.float32(engines["device"].gravity(seconds))
        db_min = float(engines["device"].db_min)
        got = {m: [] for m in engines}
        sil = {m: [] for m in engines}
        fs = [Fp64Spectrum(settings, channels=cc, sample_rate=sr) for _ in range(S)]   # state carried across calls
        truth = [[] for _ in range(S)]
        pos, t0 = 0, 0
        for T_, hop in calls:
            plain = np.ascontiguousarray(full[:, :, pos + hop: pos + hop + (T_ - 1) * hop + N])
            new = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
            r = None if rms is None else np.ascontiguousarray(rms[:, t0: t0 + T_])
            outs = {
                "device": engines["device"].process(torch.from_numpy(plain).cuda(), T_, hop, seconds=seconds,
                                                    input_rms=None if r is None else torch.from_numpy(r).cuda()),
                "host": engines["host"].process(plain, T_, hop, seconds=seconds, input_rms=r),
                "ring": engines["ring"].process(torch.from_numpy(new).cuda(), T_, hop, seconds=seconds,
                                                input_rms=None if r is None else torch.from_numpy(r).cuda(),
                                                capture_ring=True),
            }
            torch.cuda.synchronize()
            names = {m: e.last_kernel_name() for m, e in engines.items()}
            want = expected_kernel(N, cc, stereo, hop)
            for m, name in names.items():
                SEEN[(sr, fps, layout, m, hop)] = name
                assert name.startswith(want), (m, name, want, hop)
            assert names["ring"] == names["device"] + " ring", names
            for m, o in outs.items():
                got[m].append(o["db"].cpu().numpy() if m != "host" else o["db"])
                sil[m].append(o["silent"].cpu().numpy() if m != "host" else o["silent"])
            for s in range(S):   # float64 over the same frames
                truth[s].append(fs[s].run(plain[s], T_, hop, g, input_rms=None if r is None else r[s]))
            pos += T_ * hop
            t0 += T_
        got = {m: np.concatenate(v, axis=1) for m, v in got.items()}
        sil = {m: np.concatenate(v, axis=1) for m, v in sil.items()}
        assert np.array_equal(got["ring"].view(np.uint32), got["device"].view(np.uint32)), (point, layout, all_opt)
        assert np.array_equal(sil["ring"], sil["device"])
        for s in range(S):
            tr = {k: np.concatenate([c[k] for c in truth[s]]) for k in ("db", "silent", "db_eps", "flush", "weight")}
            for m in ("device", "host"):
                err, bad_floor = compare(got[m][s], tr, db_min)
                ctx = (point, layout, all_opt, m, s)
                assert not bad_floor, ("DB_MIN above the flush level", ctx)
                assert np.array_equal(sil[m][s].astype(bool), tr["silent"]), ctx
                assert err.max() < 1e-6, (float(err.max()), ctx)
                worst = max(worst, float(err.max()))
    print(f"rates {grid_id(point)} {layout} N={N}: {sorted(set(SEEN[k] for k in SEEN if k[:3] == (sr, fps, layout)))} "
          f"max normwise vs float64 {worst:.2e}")


# ---- 2. ring and sync offset against the plugin at 44.1 kHz ------------------------------------------------------------

@pytest.mark.parametrize("ms", [0, 7])
@pytest.mark.parametrize("N", [720, 1456, 2048])
@pytest.mark.parametrize("fps", [(60, 1), (60000, 1001)], ids=["60", "59.94"])
def test_ring_against_the_plugin_at_44100(fps, N, ms):
    """Ring calls, packet by packet from the first tick, against the compiled plugin fed the same packets with its clock
    advanced by each packet's whole-ns span: parity_report's criterion and identical silent flags."""
    import torch
    from oracle import refbind
    from waveform_b200 import Engine

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    sr = 44100
    hops = tick_counts(sr, fps, 40)
    calls = []
    for h in hops:   # consecutive equal tick counts share a call, up to 4 ticks
        if calls and calls[-1][1] == h and calls[-1][0] < 4:
            calls[-1] = (calls[-1][0] + 1, h)
        else:
            calls.append((1, h))
    cc = 2
    settings = {"fft_size": N, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg", "silence_gate": True}
    if ms:
        settings["audio_sync_offset"] = ms
    total = sum(hops)
    x = synth_pcm(1, cc, total, seed=0x2E6 + N + ms)[0]
    x[:, total // 4: total // 4 + 3 * 735] = 0.0
    x[:, total // 2: total // 2 + 735] *= 1e-4
    eng = Engine(settings, sample_rate=sr, channels=cc, max_streams=1)
    ref = refbind.RefSource(settings, sample_rate=sr, channels=cc, fps=fps)
    seconds = 1.0 / fps_value(fps)
    got_db, got_sil, want_db, want_sil = [], [], [], []
    pos = 0
    for T_, hop in calls:
        new = torch.from_numpy(np.ascontiguousarray(x[None, :, pos: pos + T_ * hop])).cuda()
        o = eng.process(new, T_, hop, seconds=seconds, capture_ring=True)
        torch.cuda.synchronize()
        got_db.append(o["db"][0].cpu().numpy())
        got_sil.append(o["silent"][0].cpu().numpy())
        for t in range(T_):
            a, b = pos + t * hop, pos + (t + 1) * hop
            ref.L.wfref_advance_clock_ns(ref.h, frames_to_ns(sr, b) - frames_to_ns(sr, a))
            ref.push(x[0, a:b], x[1, a:b])
            ref.tick(seconds)
            want_db.append(ref.decibels(0)[None])
            want_sil.append(1 if ref.last_silent else 0)
        pos += T_ * hop
    got_db, want_db = np.concatenate(got_db), np.stack(want_db)
    rep = parity_report(got_db, want_db, db_min=float(eng.db_min))
    assert rep["ok"], rep
    assert np.array_equal(np.concatenate(got_sil), np.array(want_sil, np.uint8))
    assert eng.last_kernel_name().endswith(" ring")
    if ms:
        assert eng.sync_delay == sync_delay(sr, ms) == 308


# ---- 3. level meter and RMS feed at 44.1 kHz ----------------------------------------------------------------------------

METER_CASES = [({"meter_buf": 150, "rms_mode": True}, 2), ({"meter_buf": 100, "rms_mode": False}, 2),
               ({"meter_buf": 150, "rms_mode": False, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.4}, 1),
               ({}, 2)]   # {} : the RMS feed
RMS_TOL = 1e-5


def _close(a, b, rel, floor=1e-30):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return np.all(np.abs(a - b) <= rel * np.maximum(np.abs(b), floor))


@pytest.mark.parametrize("buf", ["device", "host"])
@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("hop", [735, 736, 1470])
@pytest.mark.parametrize("case", range(len(METER_CASES)))
def test_meter_at_44100_against_the_oracle(case, hop, fused, buf, monkeypatch):
    """Peaks, their EMA and the silent flags bit for bit against the oracle; RMS values to 1e-5 relative (the fp32 sum's
    order, tests/test_meter.py).  Several calls, so that the carried state crosses call boundaries."""
    import torch
    from oracle.oraclebind import OracleMeter
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    set_knobs(monkeypatch, {"WF_METER_FUSED": fused})
    settings, cc = METER_CASES[case]
    feed = not settings
    if feed and hop > 1024:
        # the oracle restates capture_audio, which squares the first 1024 samples of a longer packet again for each
        # further part; OBS never delivers one, and test_meter_rms_against_float64_at_44100 holds the feed at this hop
        pytest.skip("RMS feed: packets of at most 1024 samples")
    S_, T = 4, 60
    pcm = synth_pcm(S_, cc, T * hop, seed=0x3A + hop)
    pcm[1, :, 20 * hop: 45 * hop] = 0.0                 # decay, the silent flag, wake-up
    pcm[2, :, 10 * hop: 50 * hop] *= np.float32(0.05)
    eng = MeterEngine(settings, sample_rate=44100, channels=cc, max_streams=S_, mode=METER_INPUT_RMS if feed else None)
    assert eng.window == (44096 if feed else int(44100 * settings["meter_buf"] / 1000) & -16)
    outs, t0 = [], 0
    for n in (1, 7, 22, 30):
        x = np.ascontiguousarray(pcm[:, :, t0 * hop: (t0 + n) * hop])
        if buf == "device":
            o = eng.process(torch.from_numpy(x).cuda(), n, hop)
            torch.cuda.synchronize()
            o = {k: v.cpu().numpy() for k, v in o.items()}
        else:
            o = eng.process(x, n, hop)
        outs.append(o)
        t0 += n
    got = {k: np.concatenate([o[k] for o in outs], axis=1) for k in outs[0]}
    for s in range(S_):
        orc = OracleMeter(settings, sample_rate=44100, channels=cc).run(pcm[s], T, hop, meter=not feed, rms=feed)
        if feed:
            assert _close(got["rms"][s], orc["rms"], RMS_TOL), s
            continue
        assert np.array_equal(got["silent"][s], orc["silent"]), s
        if settings["rms_mode"]:
            # the smoothed RMS level is a dB value that crosses zero: 1e-5 relative, at least 2e-4 dB (test_meter.py)
            assert _close(got["lin"][s], orc["lin"], RMS_TOL, floor=20.0), s
        else:
            assert np.array_equal(got["lin"][s], orc["lin"]), s          # max and the EMA are exact
            assert np.max(np.abs(got["db"][s] - orc["db"])) < 1e-4


@pytest.mark.parametrize("mode", ["rms", "peak", "feed"])
def test_meter_mapped_buffers_at_44100(mode):
    """Zero-copy host buffers (wf_host_alloc) give the device path's bits at 44.1 kHz with alternating tick counts."""
    import ctypes as C

    import torch
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS, WfMeterBatch

    settings = {} if mode == "feed" else {"meter_buf": 150, "rms_mode": mode == "rms"}
    cc, S_ = 2, 2
    kw = dict(sample_rate=44100, channels=cc, max_streams=S_, mode=METER_INPUT_RMS if mode == "feed" else None)
    dev, mapped = MeterEngine(settings, **kw), MeterEngine(settings, **kw)
    L = dev.L
    hops = tick_counts(44100, (60000, 1001), 24)
    x = synth_pcm(S_, cc, sum(hops), seed=77)
    cap = max(hops)
    pin, pout, psil = L.wf_host_alloc(S_ * cc * cap * 4), L.wf_host_alloc(S_ * cc * 4), L.wf_host_alloc(S_)
    assert pin and pout and psil
    try:
        pos = 0
        for hop in hops:
            new = np.ascontiguousarray(x[:, :, pos: pos + hop])
            pos += hop
            want = dev.process(torch.from_numpy(new).cuda(), 1, hop)
            torch.cuda.synchronize()
            want = {k: v.cpu().numpy() for k, v in want.items()}
            C.memmove(pin, new.ctypes.data, new.nbytes)
            b = WfMeterBatch()
            b.struct_size = C.sizeof(WfMeterBatch)
            b.n_streams, b.n_ticks, b.hop, b.first_stream, b.seconds = S_, 1, hop, 0, 1.0 / 59.94
            b.pcm, b.stream_stride, b.channel_stride = pin, cc * hop, hop
            if mode == "feed":
                b.out_lin = pout
            else:
                b.out_lin, b.out_silent = pout, psil
            mapped._check(L.wf_meter_process(mapped.h, C.byref(b)))
            lin = np.frombuffer((C.c_float * (S_ * (1 if mode == "feed" else cc))).from_address(pout), np.float32)
            ref = want["rms"] if mode == "feed" else want["lin"]
            assert np.array_equal(lin.reshape(ref.shape).view(np.uint32), ref.view(np.uint32)), hop
            if mode != "feed":
                sil = np.frombuffer((C.c_uint8 * S_).from_address(psil), np.uint8)
                assert np.array_equal(sil.reshape(want["silent"].shape), want["silent"])
    finally:
        for q in (pin, pout, psil):
            L.wf_host_free(q)


@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("kind,hop", [("rms", 735), ("rms", 736), ("feed", 735), ("feed", 1470)])
def test_meter_rms_against_float64_at_44100(kind, hop, fused, monkeypatch):
    """As tests/test_gpu_fp64.py's test_meter_rms_against_float64, with the 44.1 kHz windows W = 6608 (150 ms) and
    44096 (the RMS feed): on every tick the GPU's relative error against float64 is at most the oracle's + 4 ulp."""
    from oracle.oraclebind import OracleMeter
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    set_knobs(monkeypatch, {"WF_METER_FUSED": fused})
    S_, ch, n_ticks = 3, 2, 400 if kind == "rms" else 900
    settings = {} if kind == "feed" else {"meter_buf": 150, "rms_mode": True, "temporal_smoothing": "none"}
    eng = MeterEngine(settings, sample_rate=44100, channels=ch, max_streams=S_,
                      mode=METER_INPUT_RMS if kind == "feed" else None)
    W = eng.window
    assert W == (44096 if kind == "feed" else 6608)
    pcm = synth_pcm(S_, ch, n_ticks * hop, seed=0x5EED + hop)
    pcm[1, :, : n_ticks // 4 * hop] *= np.float32(2.0 ** -20)
    pcm[1, :, 3 * n_ticks // 4 * hop:] *= np.float32(2.0 ** -20)
    pcm[2, :, n_ticks // 3 * hop: n_ticks // 3 * hop + W + 2 * hop] = 0.0
    calls = [1, 7, 92, n_ticks - 100]
    got, t0 = [], 0
    for n in calls:
        out = eng.process(np.ascontiguousarray(pcm[:, :, t0 * hop:(t0 + n) * hop]), n, hop)
        got.append(out["rms"] if kind == "feed" else out["lin"])
        t0 += n
    got = np.concatenate(got, axis=1).astype(np.float64)
    ulp4 = 4 * 2.0 ** -24
    for s in range(S_):
        if kind == "feed":
            sq = np.square(np.abs(pcm[s]).max(axis=0).astype(np.float32)).astype(np.float64)[None]
            orc = OracleMeter({}, sample_rate=44100, channels=ch).run(pcm[s], n_ticks, hop, meter=False, rms=True)["rms"][:, None]
        else:
            sq = np.square(pcm[s].astype(np.float64))
            orc = OracleMeter(settings, sample_rate=44100, channels=ch).run(pcm[s], n_ticks, hop)["lin"]
        ends = (np.arange(n_ticks) + 1) * hop
        truth = np.stack([np.sqrt(np.array([sq[c, max(0, e - W): e].sum() for c in range(sq.shape[0])]) / W) for e in ends])
        g = got[s] if kind != "feed" else got[s][:, None]
        scale = np.maximum(truth, 1e-30)
        e_gpu = np.abs(g - truth) / scale
        e_orc = np.abs(orc.astype(np.float64) - truth) / scale
        live = truth > 0
        over = live & (e_gpu > e_orc + ulp4)
        assert not over.any(), (s, np.argwhere(over)[:5].tolist(), float(e_gpu[over].max()))
        assert np.all(g[~live] == 0.0)


# ---- 4. waveform at 44.1 kHz -----------------------------------------------------------------------------------------------

WAVE_CASES = [({"width": 800, "meter_buf": 150}, 2), ({"width": 800, "meter_buf": 150, "channel_mode": "stereo"}, 2),
              ({"width": 300, "meter_buf": 50, "channel_mode": "stereo", "normalize_volume": True}, 1),
              ({"width": 301, "meter_buf": 40, "filter_mode": "gauss", "interp_mode": "lanczos"}, 2)]
WAVE_KEYS = ("width", "meter_buf", "channel_mode", "normalize_volume")


def _wave_signal(S_, cc, n, seed):
    x = synth_pcm(S_, cc, n, seed=seed)
    x[1, :, n // 5: n // 3] = 1.0        # a row of exactly 0 dB entries ...
    x[1, :, n // 3: n // 2] = 0.0        # ... then zeros: the all-zero silent rule
    if cc == 2:
        x[2, 1] = 0.0
    return x


def _wave_vs_oracle(out, ref, ctx):
    lo = ref < -700.0
    assert np.array_equal(out < -700.0, lo), ctx
    untouched = ref == np.float32(-758.59564)
    assert np.array_equal(out[untouched], ref[untouched]), ctx
    raw = (~lo) & (np.abs(ref) <= 1.0) & (ref == out)
    assert np.max(np.abs(out[lo] - ref[lo]), initial=0.0) < 1e-3, ctx
    assert np.max(np.abs(out[~lo & ~raw] - ref[~lo & ~raw]), initial=0.0) < 1e-4, ctx


@pytest.mark.parametrize("ms", [0, 13])
@pytest.mark.parametrize("case", range(len(WAVE_CASES)))
def test_wave_at_44100(case, ms, monkeypatch):
    """Host-clock and device-clock engines, per-tick and chunked kernels, display outputs on, 59.94 fps tick counts one per
    call and then 60 fps calls of several ticks: rows and silent flags against the oracle (ms = 0; with an offset, against
    the compiled plugin), points and pixels against the display restatement; all four engines bit for bit alike."""
    import torch
    from oracle.oraclebind import OracleWave
    from test_display_modes import _tables, wave_display
    from waveform_b200 import WaveEngine

    settings, cc = WAVE_CASES[case]
    sr, S_ = 44100, 3
    calls = [(1, h) for h in tick_counts(sr, (60000, 1001), 20)] + [(6, 735), (1, 1470), (9, 735), (2, 367)]
    total = sum(t * h for t, h in calls)
    x = _wave_signal(S_, cc, total, 0x77 + case)
    rms = (0.05 + 0.2 * np.random.default_rng(case).uniform(size=(S_, sum(t for t, _ in calls)))).astype(np.float32) \
        if settings.get("normalize_volume") else None
    ws = {**settings, **({"audio_sync_offset": ms} if ms else {})}
    runs = {}
    for chunk in ("1", "0"):
        set_knobs(monkeypatch, {"WF_WAVE_CHUNK": chunk})
        for clock in (False, True):
            eng = WaveEngine(ws, sample_rate=sr, channels=cc, max_streams=S_, device_clock=clock)
            outs, pos, t0 = [], 0, 0
            for T_, hop in calls:
                xi = torch.from_numpy(np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])).cuda()
                ri = None if rms is None else torch.from_numpy(np.ascontiguousarray(rms[:, t0: t0 + T_])).cuda()
                o = eng.process(xi, T_, hop, input_rms=ri, want_points=True, want_pixels=True)
                torch.cuda.synchronize()
                outs.append({k: v.cpu().numpy() for k, v in o.items()})
                pos += T_ * hop
                t0 += T_
            runs[(chunk, clock)] = {k: np.concatenate([o[k] for o in outs], axis=1) for k in outs[0]}
    base = runs[("0", False)]
    for key, r in runs.items():
        for k in base:
            assert np.array_equal(r[k].view(np.uint8), base[k].view(np.uint8)), (key, k)
    # rows and flags: the oracle (no offset) or the plugin (offset)
    ref = np.zeros_like(base["out"])
    ref_sil = np.zeros_like(base["silent"])
    for s in range(S_):
        if ms:
            from oracle import refbind

            if not refbind.available():
                pytest.skip("the compiled reference (oracle/_ref) is not built")
            src = refbind.RefSource({"display_mode": "waveform", **ws}, sample_rate=sr, channels=cc)
        else:
            src = OracleWave({k: v for k, v in settings.items() if k in WAVE_KEYS}, sample_rate=sr, channels=cc)
        pos, t0 = 0, 0
        for T_, hop in calls:
            seg = np.ascontiguousarray(x[s, :, pos: pos + T_ * hop])
            rr = None if rms is None else rms[s, t0: t0 + T_]
            w = src.run_wave(seg, T_, hop, rms=rr) if ms else src.run(seg, T_, hop, rms=rr)
            ref[s, t0: t0 + T_], ref_sil[s, t0: t0 + T_] = w["out"], w["silent"]
            pos += T_ * hop
            t0 += T_
    assert np.array_equal(base["silent"], ref_sil)
    _wave_vs_oracle(base["out"], ref, (settings, ms))
    pts, px, mn = wave_display(base["out"], _tables(settings, cc), settings)
    assert np.abs(base["points"] - pts).max() < 1e-3
    assert np.abs(base["pixels"] - px).max() < 2e-4
    assert np.array_equal(base["min"][..., 1], mn[..., 1])


# ---- 5. the seam at 44.1 kHz ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fps", [(60, 1), (60000, 1001)], ids=["60", "59.94"])
def test_wavsource_cuda_matches_wavsource_generic_at_44100(fps):
    """WAVSourceCUDA against WAVSourceGeneric, both built from the plugin's own sources, with auto_fft_size (720) and
    volume normalisation (the live RMS feed), fed OBS's 1024-frame packets on their own clock and ticked at the frame rate."""
    from oracle import refbind

    if not (refbind.available() and refbind.cuda_seam_available()):
        pytest.skip("oracle/_ref libraries not built (needs the reference sources)")
    sr, cc = 44100, 2
    settings = {"auto_fft_size": True, "window": "blackman", "normalize_volume": True, "channel_mode": "stereo"}
    gen = refbind.RefSource(settings, impl=refbind.IMPL_GENERIC, sample_rate=sr, channels=cc, fps=fps)
    cuda = refbind.RefSource(settings, impl=refbind.IMPL_CUDA, sample_rate=sr, channels=cc, fps=fps)
    assert gen.fft_size == cuda.fft_size == 720
    ticks, packet = 120, 1024
    pcm = synth_pcm(1, cc, ticks * 800, seed=31)[0] * np.float32(0.3)
    pcm[:, 30000:45000] = 0.0
    num, den = fps
    out = {}
    for name, src in (("gen", gen), ("cuda", cuda)):
        clock, sent, rows, sil, rms = 0, 0, [], [], []
        for t in range(ticks):
            now = (t + 1) * 10**9 * den // num
            while frames_to_ns(sr, sent + packet) <= now and sent + packet <= pcm.shape[1]:
                end = frames_to_ns(sr, sent + packet)
                src.L.wfref_advance_clock_ns(src.h, end - clock)
                clock = end
                src.push(pcm[0, sent: sent + packet], pcm[1, sent: sent + packet])
                sent += packet
            src.L.wfref_advance_clock_ns(src.h, now - clock)
            clock = now
            src.tick(float(np.float32(den) / np.float32(num)))
            rows.append(np.stack([src.decibels(0), src.decibels(1)]))
            sil.append(src.last_silent)
            rms.append(src.L.wfref_input_rms(src.h))
        out[name] = (np.stack(rows), np.array(sil), np.array(rms))
    assert np.array_equal(out["gen"][2], out["cuda"][2]) and out["gen"][2][-1] > 0
    assert np.array_equal(out["gen"][1], out["cuda"][1])
    g, c = out["gen"][0], out["cuda"][0]
    d = np.abs(g.astype(np.float64) - c.astype(np.float64))
    assert d.max() < 2e-3 and np.median(d) < 2e-5, (d.max(), np.median(d))


def test_live_adapter_at_44100(tmp_path):
    """The C++ host mirror (SpectrumSourceCUDA) at 44.1 kHz, N = 720, 1024-frame packets, 60 fps, with the live RMS feed,
    against the compiled plugin driven with the same schedule (its outputs stored, tests/refdata.py)."""
    from test_gpu_host import _build_driver

    sr, N, cc, stereo, normalize = 44100, 720, 2, 1, 1
    packet, fps, ticks, ns = 1024, 60, 60, 44100
    pcm = synth_pcm(1, cc, ns, seed=21)[0]
    pcm[:, 20000:] = 0.0
    B, dch = N // 2, 2
    t_at, b_at = sample_index((ticks,), 8, N), sample_index((B,), 64, N + 1)

    def live():
        from oracle import refbind

        ref = refbind.RefSource({"fft_size": N, "channel_mode": "stereo", "normalize_volume": True},
                                impl=refbind.IMPL_GENERIC, sample_rate=sr, channels=cc)
        now = clock = 10 * 10**9
        tick_ns, pkt_ns = 10**9 // fps, packet * 10**9 // sr
        next_pkt, pos, rows, sil = now, 0, [], []
        for _ in range(ticks):
            now += tick_ns
            while next_pkt + pkt_ns <= now and pos + packet <= ns:
                next_pkt += pkt_ns
                ref.L.wfref_advance_clock_ns(ref.h, next_pkt - clock)
                clock = next_pkt
                ref.push(pcm[0, pos:pos + packet], pcm[1, pos:pos + packet])
                pos += packet
            ref.L.wfref_advance_clock_ns(ref.h, now - clock)
            clock = now
            ref.tick(np.float32(1.0) / np.float32(fps))
            rows.append(np.stack([ref.decibels(c) for c in range(2)]))
            sil.append(ref.last_silent)
        rows = np.stack(rows)
        return {"silent": np.array(sil, np.uint8), "db": rows[t_at][..., b_at], "peak": frame_peak(rows[t_at], -758.0)}

    ref = reference(f"rates/live_adapter/{sr}_{N}", live)
    exe = _build_driver(tmp_path)
    inp, outp = tmp_path / "pcm.f32", tmp_path / "out.f32"
    pcm.astype(np.float32).tofile(inp)
    r = subprocess.run([str(exe), str(inp), str(cc), str(ns), str(N), str(packet), str(fps), str(ticks), str(outp),
                        str(stereo), str(normalize), str(sr)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(outp, dtype=np.uint8).reshape(ticks, dch * B * 4 + 1)
    got = raw[:, :-1].copy().view(np.float32).reshape(ticks, dch, B)
    assert np.array_equal(raw[:, -1], ref["silent"])
    rep = parity_report(got[t_at][..., b_at], ref["db"], peak=ref["peak"])
    assert rep["ok"], rep
