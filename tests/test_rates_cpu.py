"""Every engine at the sample rates and frame rates OBS really runs: 44.1 and 48 kHz, at the common video frame rates.

48 kHz at 60 fps is the one configuration where every fast path's preconditions hold (hop = N = 800, a 150 ms meter window
of exactly 9 hops).  At 44.1 kHz the automatic FFT size is 735 & -16 = 720 while each 60 fps tick brings 735 samples, the
meter window (6608) is no multiple of the hop, and every clock computation runs on 44100.  This file writes the (rate, fps)
grid down once (tests/test_gpu_rates.py imports it) and checks, without a GPU, what depends on the rate on the host side
and in the oracle:
  - the automatic FFT size of every grid point, the compiled plugin's own m_fft_size;
  - the engine's setup tables against the plugin's at 44.1 and 48 kHz;
  - the oracle (spectrum, level meter, RMS feed, waveform) against the plugin at 44.1 kHz;
  - the engine's waveform tick plan against the oracle at 44.1, 48, 96 and 22.05 kHz;
  - the audio sync offset's models against the plugin at 44.1 kHz, where ms * 44.1 is fractional.
What the compiled plugin computed is stored in tests/golden/reference_outputs.npz (tests/refdata.py)."""
from __future__ import annotations

import numpy as np
import pytest

from helpers import parity_report, synth_pcm
from refdata import digest, frame_peak, reference, sample_index

# ---- the grid ---------------------------------------------------------------------------------------------------------

RATES = (44100, 48000)
FPS = ((24000, 1001), (24, 1), (25, 1), (30000, 1001), (30, 1), (48, 1), (50, 1), (60000, 1001), (60, 1), (90, 1),
       (100, 1), (120, 1), (144, 1), (165, 1), (240, 1))
GRID = [(sr, fps) for sr in RATES for fps in FPS]


def fps_id(fps) -> str:
    num, den = fps
    return f"{num}" if den == 1 else f"{num}-{den}"


def grid_id(point) -> str:
    return f"{point[0]}-{fps_id(point[1])}"


def fps_value(fps) -> float:
    return float(fps[0]) / float(fps[1])


def auto_size(sr: int, fps) -> int:
    """m_fft_size under auto_fft_size: size_t(samples_per_sec / fps) & -16, at least 128, with fps a double as OBS's."""
    return max(int(sr / fps_value(fps)) & -16, 128)


def tick_counts(sr: int, fps, n: int) -> list[int]:
    """New samples per video frame for the first n frames: at a fractional frame rate they alternate between two
    neighbours (735 / 736 at 44.1 kHz and 59.94 fps, 533 / 534 at 48 kHz and 90 fps)."""
    num, den = fps
    return [(k + 1) * sr * den // num - k * sr * den // num for k in range(n)]


def frames_to_ns(sr: int, frames: int) -> int:
    """audio_frames_to_ns: the timestamp span of `frames` samples, truncated to whole ns."""
    return frames * 10**9 // sr


def sync_delay(sr: int, ms: int) -> int:
    """Samples an audio sync offset of ms milliseconds holds back (ns_to_audio_frames of a positive offset, else 0)."""
    return ms * 10**6 * sr // 10**9 if ms > 0 else 0


def test_grid_facts():
    """The grid's sizes and tick counts are the ones DESIGN.md §2 lists."""
    sizes = {sr: sorted({auto_size(sr, f) for f in FPS}) for sr in RATES}
    assert sizes[44100] == [176, 256, 304, 352, 432, 480, 720, 880, 912, 1456, 1760, 1824]
    assert sizes[48000] == [192, 288, 320, 400, 480, 528, 800, 960, 992, 1600, 1920, 2000]
    for sr, fps in GRID:
        c = tick_counts(sr, fps, 1001)
        q = int(sr / fps_value(fps))
        assert set(c) <= {q, q + 1} and sum(c) == 1001 * sr * fps[1] // fps[0]
        assert (len(set(c)) == 2) == (sr * fps[1] % fps[0] != 0), (sr, fps)
    assert set(tick_counts(44100, (60000, 1001), 8)) == {735, 736}
    assert set(tick_counts(48000, (90, 1), 3)) == {533, 534}


def _ref(**kw):
    from oracle import refbind

    return refbind.RefSource(**kw)


# ---- 1. automatic sizes -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("point", GRID, ids=[grid_id(p) for p in GRID])
def test_automatic_fft_size_is_the_plugins(point):
    from waveform_b200.engine import make_config, preview_tables

    sr, fps = point
    N = auto_size(sr, fps)
    r = reference(f"rates/auto_size/{grid_id(point)}",
                  lambda: {"fft_size": _ref(settings={"auto_fft_size": True}, sample_rate=sr, channels=1, fps=fps).fft_size})
    assert int(r["fft_size"]) == N
    info = preview_tables(make_config({"fft_size": N}, sr, 1))["info"]
    assert info.fft_size == N and info.bins == N // 2


# ---- 2. setup tables at 44.1 and 48 kHz -------------------------------------------------------------------------------

TABLE_CASES = [
    ({"fft_size": 720, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg"}, 2),
    ({"fft_size": 1824, "display_mode": "bars", "interp_mode": "lanczos", "bar_width": 4, "bar_gap": 1,
      "rolloff_q": 1.0, "rolloff_rate": 6.0}, 1),
    ({"fft_size": 912, "log_scale": False, "interp_mode": "point", "slope": 0.5, "cutoff_low": 20, "cutoff_high": 20000}, 1),
    ({"fft_size": 432, "mirror_freq_axis": True, "interp_mode": "catmull_rom", "filter_mode": "gauss", "filter_radius": 2.5,
      "cutoff_low": 100, "cutoff_high": 12000, "rolloff_q": 1.5, "rolloff_rate": 9.0}, 2),
    ({"fft_size": 2000, "display_mode": "bars", "interp_mode": "catmull_rom", "log_scale": False, "mirror_freq_axis": True,
      "cutoff_high": 21000, "channel_mode": "stereo"}, 2),
    ({"fft_size": 176, "window": "power_of_sine", "sine_exponent": 3, "interp_mode": "lanczos", "rolloff_q": 0.7,
      "rolloff_rate": 3.0, "cutoff_low": 50, "cutoff_high": 16000, "width": 300}, 1),
    ({"fft_size": 4096, "window": "blackman_harris", "display_mode": "bars", "interp_mode": "point", "cutoff_low": 30,
      "cutoff_high": 22000, "rolloff_q": 2.0, "rolloff_rate": 12.0, "filter_mode": "gauss"}, 1),
    ({"fft_size": 1456, "window": "hamming", "log_scale": True, "interp_mode": "lanczos", "slope": 1.0,
      "cutoff_low": 10, "cutoff_high": 17500, "mirror_freq_axis": True, "width": 1280}, 1),
]
TABLE_NAMES = ("window", "slope", "rolloff", "interp_indices", "band_widths", "interp_weights", "gauss")


def _as_table(a, dtype=np.float32):
    return np.zeros(0, dtype) if a is None else np.ascontiguousarray(a, dtype).ravel()


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("case", range(len(TABLE_CASES)))
def test_engine_tables_equal_the_plugins_at_each_rate(case, sr):
    """wf_tables.cpp against WAVSource::update() at this rate: window, slope, roll-off (hz_per_bin = sr / N), the
    interpolation indices (cutoff * N / sr) and weights, the bar band widths and the Gaussian, bit for bit."""
    from waveform_b200.engine import make_config, preview_tables

    settings, cc = TABLE_CASES[case]

    def live():
        r = _ref(settings=settings, sample_rate=sr, channels=cc)
        _, weights = r.interp_kernel()
        t = {"window": r.window(), "slope": r.slope(), "rolloff": r.rolloff(), "interp_indices": r.interp_indices(),
             "band_widths": r.band_widths(), "interp_weights": weights, "gauss": r.gauss_kernel()[0]}
        return {"fft_size": r.fft_size, "window_sum": np.float32(r.window_sum), "db_min": np.float32(r.db_min),
                **{k: digest(_as_table(v, np.int32 if k == "band_widths" else np.float32)) for k, v in t.items()}}

    ref = reference(f"rates/tables/{sr}/case{case}", live)
    t = preview_tables(make_config(settings, sr, cc))
    assert t["info"].fft_size == int(ref["fft_size"])
    for name in TABLE_NAMES:
        got = _as_table(t[name] if t[name].size else None, np.int32 if name == "band_widths" else np.float32)
        assert np.array_equal(digest(got), ref[name]), (name, sr, settings)
    assert np.float32(t["info"].window_sum) == ref["window_sum"] and np.float32(t["info"].db_min) == ref["db_min"]
    if settings.get("rolloff_q"):   # the roll-off table depends on the rate, so the two rates must differ
        other = preview_tables(make_config(settings, 48000 if sr == 44100 else 44100, cc))["rolloff"]
        assert not np.array_equal(other, t["rolloff"])


# ---- 3. the oracle against the plugin at 44.1 kHz ---------------------------------------------------------------------

SR = 44100
HOPS = (735, 736, 1470, 367, 306)      # 60 fps, its 59.94 neighbour, 30 fps, 120 fps, 144 fps
TICKS, BINS = 4, 32


def _spectrum_input(N, cc, T, hop, seed):
    x = synth_pcm(1, cc, (T - 1) * hop + N, seed=seed)[0]
    x[:, 5 * hop: 5 * hop + 3 * N] = 0.0
    if cc == 2:
        x[1, 11 * hop:] = 0.0
    return x


def _oracle_vs_plugin(key, settings, cc, hop, T, seconds, seed, sr=SR):
    """The oracle against the plugin over T ticks of `hop` samples at this rate: tables bit for bit, the spectra of a fixed
    sample of ticks and bins within test_oracle_vs_reference's parity criterion, silent flags and display points."""
    from oracle.oraclebind import OracleSource

    rms = (0.05 + 0.3 * np.random.default_rng(seed).uniform(size=T)).astype(np.float32) \
        if settings.get("normalize_volume") else None
    ticks = sample_index((T,), TICKS, seed)

    def live():
        ref = _ref(settings=settings, sample_rate=sr, channels=cc)
        N, c = ref.fft_size, ref.capture_channels
        a = ref.run_stft(_spectrum_input(N, c, T, hop, seed), T, hop, seconds=seconds, rms=rms, want_points=True)
        bins = sample_index((N // 2,), BINS, seed + 1)
        pts = sample_index((a["points"].shape[-1],), BINS, seed + 2)
        return {"fft_size": N, "capture_channels": c, "db_min": ref.db_min, "frames": a["frames"],
                "rolloff": digest(_as_table(ref.rolloff())), "interp_indices": digest(ref.interp_indices()),
                "silent": a["silent"], "db": a["db"][ticks][..., bins], "peak": frame_peak(a["db"][ticks], ref.db_min),
                "num_points": a["points"].shape[-1], "points": a["points"][ticks][..., pts]}

    r = reference(key, live)
    N, c = int(r["fft_size"]), int(r["capture_channels"])
    assert int(r["frames"]) == T
    orc = OracleSource(settings, sample_rate=sr, channels=cc)
    b = orc.run_stft(_spectrum_input(N, c, T, hop, seed), T, hop, seconds=seconds, rms=rms, want_points=True)
    assert np.array_equal(digest(_as_table(orc.rolloff())), r["rolloff"])
    assert np.array_equal(digest(orc.interp_indices()), r["interp_indices"])
    bins = sample_index((N // 2,), BINS, seed + 1)
    pts = sample_index((int(r["num_points"]),), BINS, seed + 2)
    rep = parity_report(b["db"][ticks][..., bins], r["db"], db_min=float(r["db_min"]), peak=r["peak"])
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(r["silent"], b["silent"])
    d = np.abs(r["points"].astype(np.float64) - b["points"][ticks][..., pts].astype(np.float64))
    assert d.max() < 5e-3 and np.median(d) < 1e-4


SPECTRUM_CASES = [
    ({"fft_size": 720, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg"}, 2, 735),
    ({"fft_size": 720, "window": "hann", "rolloff_q": 1.0, "rolloff_rate": 6.0, "silence_gate": True}, 1, 736),
    ({"fft_size": 1456, "window": "blackman_harris", "channel_mode": "stereo", "slope": 0.5, "fast_peaks": True}, 2, 1470),
    ({"fft_size": 352, "window": "hamming", "normalize_volume": True, "display_mode": "bars", "interp_mode": "lanczos"}, 2, 367),
    ({"fft_size": 304, "window": "power_of_sine", "sine_exponent": 2, "interp_mode": "catmull_rom", "cutoff_high": 20000,
      "rolloff_q": 1.5, "rolloff_rate": 9.0}, 1, 306),
]


@pytest.mark.parametrize("case", range(len(SPECTRUM_CASES)))
def test_spectrum_oracle_is_the_plugins_at_44100(case):
    settings, cc, hop = SPECTRUM_CASES[case]
    _oracle_vs_plugin(f"rates/spectrum/case{case}", settings, cc, hop, 24, 1.0 / 60.0, 300 + case)


@pytest.mark.parametrize("seed", range(16))
def test_spectrum_oracle_randomised_rates_and_settings(seed):
    """Differential fuzz over the grid: a random rate and frame rate give the automatic size and the hop (one of the frame
    rate's tick counts); the settings are drawn as in test_oracle_vs_reference."""
    rng = np.random.default_rng(8800 + seed)
    sr = int(rng.choice(RATES))
    fps = FPS[int(rng.integers(len(FPS)))]
    N = auto_size(sr, fps)
    hop = int(rng.choice(tick_counts(sr, fps, 4)))
    mode = str(rng.choice(["mono", "mono", "stereo"]))
    cc = 2 if mode == "stereo" or rng.uniform() < 0.5 else 1
    settings = {"fft_size": N, "channel_mode": mode,
                "window": str(rng.choice(["none", "hann", "hamming", "blackman", "blackman_harris"])),
                "temporal_smoothing": str(rng.choice(["none", "exp_moving_avg", "tv_exp_moving_avg"])),
                "gravity": float(rng.choice([0.2, 0.5, 0.65, 0.9])), "floor": int(rng.choice([-30, -45, -65])),
                "display_mode": str(rng.choice(["curve", "bars"])),
                "interp_mode": str(rng.choice(["point", "lanczos", "catmull_rom"])),
                "log_scale": bool(rng.uniform() < 0.8)}
    if rng.uniform() < 0.4:
        settings.update(slope=float(rng.choice([0.25, 1.0])), fast_peaks=bool(rng.uniform() < 0.5))
    if rng.uniform() < 0.5:
        settings.update(rolloff_q=float(rng.choice([0.7, 1.0, 2.0])), rolloff_rate=float(rng.choice([3.0, 9.0])))
    if rng.uniform() < 0.3:
        settings.update(cutoff_low=int(rng.choice([20, 60])), cutoff_high=int(rng.choice([12000, 20000])))
    if rng.uniform() < 0.2:
        settings["normalize_volume"] = True
    _oracle_vs_plugin(f"rates/spectrum/seed{seed}", settings, cc, hop, 16, 1.0 / fps_value(fps), 900 + seed, sr=sr)


METER_CASES = [({"meter_buf": 150, "rms_mode": True}, 2),            # the default: W = 6608, not a multiple of 735
               ({"meter_buf": 100, "rms_mode": False, "fast_peaks": True}, 2),
               ({"meter_buf": 20, "rms_mode": True, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.4}, 1)]


def _meter_pcm(cc, T, hop, seed):
    pcm = synth_pcm(1, cc, T * hop, seed=seed)[0]
    pcm[:, (T // 2) * hop: (3 * T // 4) * hop] = 0.0
    return pcm


@pytest.mark.parametrize("hop", HOPS)
@pytest.mark.parametrize("case", range(len(METER_CASES)))
def test_meter_oracle_is_bit_exact_vs_the_plugin_at_44100(case, hop):
    from oracle.oraclebind import OracleMeter

    settings, cc = METER_CASES[case]
    T = 48
    pcm = _meter_pcm(cc, T, hop, 40 + case)

    def live():
        r = _ref(settings={"display_mode": "level_meter", **settings}, sample_rate=SR, channels=cc)
        out = r.run_meter(pcm, T, hop)
        return {"window": r.fft_size, **{k: digest(out[k]) for k in ("db", "lin", "silent")}}

    ref = reference(f"rates/meter/case{case}/{hop}", live)
    o = OracleMeter(settings, sample_rate=SR, channels=cc)
    assert o.window == int(ref["window"]) == int(SR * settings["meter_buf"] / 1000) & -16
    out = o.run(pcm, T, hop)
    for k in ("db", "lin", "silent"):
        assert np.array_equal(digest(out[k]), ref[k]), k


@pytest.mark.parametrize("hop", (735, 736, 367, 306, 1000))
@pytest.mark.parametrize("cc", [1, 2])
def test_rms_feed_oracle_is_bit_exact_vs_the_plugin_at_44100(cc, hop):
    """The RMS feed's window is 44100 & -16 = 44096 samples (packets of at most 1024 samples, as OBS delivers them)."""
    from oracle.oraclebind import OracleMeter

    T = 90
    pcm = _meter_pcm(cc, T, hop, 60 + cc)

    def live():
        r = _ref(settings={"normalize_volume": True, "fft_size": 720}, sample_rate=SR, channels=cc)
        return {"rms": digest(r.run_meter(pcm, T, hop)["rms"])}

    ref = reference(f"rates/rms_feed/{cc}/{hop}", live)
    out = OracleMeter({}, sample_rate=SR, channels=cc).run(pcm, T, hop, meter=False, rms=True)["rms"]
    assert np.array_equal(digest(out), ref["rms"])


WAVE_CASES = [({"width": 800, "meter_buf": 150}, 2),
              ({"width": 300, "meter_buf": 50, "channel_mode": "stereo"}, 2),
              ({"width": 640, "meter_buf": 500, "channel_mode": "stereo", "normalize_volume": True}, 1),
              ({"width": 1000, "meter_buf": 20}, 1)]


def _wave_pcm(cc, T, hop, seed):
    pcm = synth_pcm(1, cc, T * hop, seed=seed)[0]
    pcm[:, 20 * hop: 30 * hop] = 0.0
    pcm[:, 33 * hop: 35 * hop] = 1.0
    return pcm


@pytest.mark.parametrize("hop", HOPS)
@pytest.mark.parametrize("case", range(len(WAVE_CASES)))
def test_wave_oracle_is_bit_exact_vs_the_plugin_at_44100(case, hop):
    """tick_waveform at 44.1 kHz: a window of samples_per_sec * meter_ms / 1000 samples (6615 at 150 ms) and the
    timestamp walk on frames_to_ns / ns_to_frames with 44100."""
    from oracle.oraclebind import OracleWave

    settings, cc = WAVE_CASES[case]
    T = 50
    pcm = _wave_pcm(cc, T, hop, 70 + case)
    rms = (0.05 + 0.2 * np.random.default_rng(case).uniform(size=T)).astype(np.float32) \
        if settings.get("normalize_volume") else None

    def live():
        r = _ref(settings={"display_mode": "waveform", **settings}, sample_rate=SR, channels=cc)
        out = r.run_wave(pcm, T, hop, rms=rms)
        return {"out": digest(out["out"]), "silent": digest(out["silent"])}

    ref = reference(f"rates/wave/case{case}/{hop}", live)
    out = OracleWave(settings, sample_rate=SR, channels=cc).run(pcm, T, hop, rms=rms)
    assert np.array_equal(digest(out["out"]), ref["out"])
    assert np.array_equal(digest(out["silent"]), ref["silent"])


# ---- 4. the engine's waveform plan --------------------------------------------------------------------------------------

def wave_plan(width, meter_ms, D, hops, sr):
    """tick_waveform's timestamp walk (src/source_generic.cpp:290-339,358) for packets of the given sizes stamped "now", with
    the sync offset's reserve of D samples: per tick, the stream index of every new point's sample (negative: a start-up or
    delay zero)."""
    ws = int(float(sr) * (meter_ms / 1000.0))
    step = meter_ms * 1000000 // width
    clock, wts, buffered, pos = 10 * 10**9, 0, width, 0
    out = []
    for hop in hops:
        clock += frames_to_ns(sr, hop)
        ats = clock
        pos += hop
        total = min(buffered + hop, ws + D)
        buffered = total
        pts = []
        if total > D:
            start, stop = ats - frames_to_ns(sr, total), ats - frames_to_ns(sr, D)
            if wts < start:
                wts = start
            if wts > stop and wts - stop > step:
                wts = start
            for i in range(width):
                ts = wts + i * step
                if ts >= stop:
                    break
                index = min(max((ats - ts) * sr // 10**9, D + 1), total)
                pts.append(pos - index)
            wts += len(pts) * step
            buffered = D
        out.append(np.array(pts, np.int64))
    return out


def _ramp(n):
    return ((np.arange(n, dtype=np.float64) + 1.0) * 2.0 ** -20).astype(np.float32)[None, :]  # exact, never 0


def _picked(pts, ramp):
    return np.where(pts >= 0, ramp[0, np.maximum(pts, 0)], np.float32(0.0))


WAVE_PLAN_SETTINGS = [(800, 150), (300, 50), (1000, 20), (640, 500)]


@pytest.mark.parametrize("sr", [44100, 48000, 96000, 22050])
@pytest.mark.parametrize("width,meter_ms", WAVE_PLAN_SETTINGS)
def test_engine_wave_plan_equals_the_oracle_at_each_rate(width, meter_ms, sr):
    """wf_wave_preview_plan (which points a tick emits, which sample each takes) against the oracle's ramp read-back: a mono
    capture shown as two channels leaves the raw new samples in the second channel.  At 44.1 and 48 kHz every tick count
    of the grid; at 96 and 22.05 kHz those of 60 and 59.94 fps."""
    from oracle.oraclebind import OracleWave
    from waveform_b200.engine import make_wave_config, preview_wave_plan

    T = 40
    settings = {"width": width, "meter_buf": meter_ms, "channel_mode": "stereo"}
    fpss = FPS if sr in RATES else ((60, 1), (60000, 1001))
    hops = sorted({h for f in fpss for h in tick_counts(sr, f, 4)})
    for hop in hops:
        ramp = _ramp(T * hop)
        got = OracleWave(settings, sample_rate=sr, channels=1).run(ramp, T, hop)["out"][:, 1, :]
        counts, src = preview_wave_plan(make_wave_config(settings, sr, channels=1), T, hop)
        assert counts.sum() == len(src) and counts.max() <= width
        model = wave_plan(width, meter_ms, 0, [hop] * T, sr)
        assert np.array_equal(counts, [len(p) for p in model]), (sr, hop)
        o = 0
        for t in range(T):
            c = int(counts[t])
            assert np.array_equal(got[t, width - c:], _picked(src[o: o + c], ramp)), (sr, hop, t)
            o += c


@pytest.mark.parametrize("point", [(44100, (60000, 1001)), (44100, (30000, 1001)), (48000, (60000, 1001)),
                                   (44100, (24000, 1001))], ids=grid_id)
def test_wave_plan_model_with_alternating_tick_counts(point):
    """A fractional frame rate's alternating tick counts, one tick per call: the model (the engine's walk, restated) against
    the oracle's ramp read-back tick by tick."""
    from oracle.oraclebind import OracleWave

    sr, fps = point
    width, meter_ms = 800, 150
    hops = tick_counts(sr, fps, 90)
    ramp = _ramp(sum(hops))
    o = OracleWave({"width": width, "meter_buf": meter_ms, "channel_mode": "stereo"}, sample_rate=sr, channels=1)
    plan = wave_plan(width, meter_ms, 0, hops, sr)
    pos = 0
    for t, hop in enumerate(hops):
        got = o.run(np.ascontiguousarray(ramp[:, pos: pos + hop]), 1, hop)["out"][0, 1]
        c = len(plan[t])
        assert np.array_equal(got[width - c:], _picked(plan[t], ramp)), (t, hop, c)
        pos += hop


# ---- 5. the audio sync offset at 44.1 kHz -------------------------------------------------------------------------------

OFFSETS_MS = [1, 7, 13, 999]   # ms * 44.1 is fractional for each


def test_sync_delay_truncates_at_44100():
    for ms, want in ((1, 44), (7, 308), (13, 573), (999, 44055), (-5, 0)):
        assert sync_delay(SR, ms) == want


def _advance(ref, sr, before, after):
    """The plugin's clock by the span of the samples it has been handed: whole ns of each packet's end (a per-packet
    rounding of hop / sr would drift from the packets' own timestamps)."""
    ref.L.wfref_advance_clock_ns(ref.h, frames_to_ns(sr, after) - frames_to_ns(sr, before))


def _ring_calls(N):
    return [(3, 735), (1, 736), (2, N), (1, N + 441), (4, 512), (6, 1470), (2, 367), (2, 22050), (3, 735)]


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("N,cc,stereo", [(720, 1, False), (1456, 2, True)])
def test_spectrum_offset_model_is_the_plugins_at_44100(N, cc, stereo, ms):
    """The plugin fed packet by packet with an offset: a tick is short of audio while fewer than D samples have arrived in
    all, and then leaves m_decibels and m_last_silent as they were; every other tick's frame is the oldest N of the newest
    N + D samples of zeros(N + D) ++ stream.  Held against the oracle fed the model's frames."""
    from oracle.oraclebind import OracleSource

    D = sync_delay(SR, ms)
    calls = _ring_calls(N)
    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=0x44 + N + ms)[0]
    x[:, total // 3: total // 3 + N] = 0.0
    settings = {"fft_size": N, "window": "hann", "silence_gate": True, **({"channel_mode": "stereo"} if stereo else {})}
    bins = sample_index((N // 2,), BINS, N)

    def live():
        pk = _ref(settings={**settings, "audio_sync_offset": ms}, sample_rate=SR, channels=cc)
        dch = pk.display_channels
        prev = np.stack([pk.decibels(c) for c in range(dch)])
        db, peak, sil, same, pos = [], [], [], [], 0
        for T_, hop in calls:
            for t in range(T_):
                seg = x[:, pos: pos + hop]
                _advance(pk, SR, pos, pos + hop)
                pk.push(seg[0], seg[1] if cc == 2 else None)
                pk.tick(1.0 / 60.0)
                row = np.stack([pk.decibels(c) for c in range(dch)])
                same.append(np.array_equal(row, prev))
                db.append(row[:, bins])
                peak.append(frame_peak(row, pk.db_min))
                sil.append(pk.last_silent)
                prev = row
                pos += hop
        return {"db": np.stack(db), "peak": np.stack(peak), "silent": np.array(sil, np.uint8),
                "same": np.array(same, np.uint8), "db_min": pk.db_min}

    r = reference(f"rates/sync_spectrum/{N}/{ms}", live)
    timeline = np.concatenate([np.zeros((cc, N + D), np.float32), x], axis=1)
    orc = OracleSource(settings, sample_rate=SR, channels=cc)
    arrived, k, run = 0, 0, []
    for T_, hop in calls:
        for t in range(T_):
            arrived += hop
            if arrived < D:      # short of audio: nothing changes
                assert r["same"][k] and (k == 0 or r["silent"][k] == r["silent"][k - 1]), (k, ms)
            else:
                orc.tick([timeline[c, arrived: arrived + N] for c in range(cc)], 1.0 / 60.0)
                rows = np.stack([orc.decibels(c) for c in range(2 if stereo else 1)])
                run.append((k, rows[:, bins], orc.last_silent))
            k += 1
    assert run, "no tick with audio"
    idx = [i for i, _, _ in run]
    rep = parity_report(np.stack([v for _, v, _ in run]), r["db"][idx], db_min=float(r["db_min"]), peak=r["peak"][idx])
    assert rep["ok"], (rep, ms)
    assert np.array_equal(np.array([s for _, _, s in run], np.uint8), r["silent"][idx])
    if D > 735:
        assert len(run) < k


METER_SYNC_CASES = [({"display_mode": "level_meter", "rms_mode": False, "meter_buf": 100}, 2),
                    ({"display_mode": "level_meter", "rms_mode": True, "meter_buf": 150}, 2),
                    ({"fft_size": 720, "normalize_volume": True, "channel_mode": "stereo"}, 2)]   # the RMS feed


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("case", range(len(METER_SYNC_CASES)))
def test_meter_offset_is_a_zero_prefixed_stream_at_44100(case, ms):
    """tick_meter / update_input_rms with the offset consume all but the newest D samples: the plugin with the offset equals
    the oracle fed zeros(D) ++ stream (peaks and flags exactly; RMS sums in another ring order, to a few 1e-6)."""
    from oracle.oraclebind import OracleMeter

    settings, cc = METER_SYNC_CASES[case]
    D = sync_delay(SR, ms)
    feed = bool(settings.get("normalize_volume"))
    calls = [(5, 735), (3, 736), (9, 1024), (2, 367), (7, 306), (4, 1000)] if feed else \
        [(5, 735), (3, 736), (2, 4410), (1, 9000), (7, 306), (4, 1470)]
    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=0x4E + ms)[0]
    x[:, total // 4: total // 4 + 6000] = 0.0

    def live():
        off = _ref(settings={**settings, "audio_sync_offset": ms}, sample_rate=SR, channels=cc)
        outs, pos = [], 0
        for T_, hop in calls:
            outs.append(off.run_meter(x[:, pos: pos + T_ * hop], T_, hop))
            pos += T_ * hop
        return {k: np.concatenate([o[k] for o in outs]) for k in (("rms",) if feed else ("db", "lin", "silent"))}

    r = reference(f"rates/sync_meter/case{case}/{ms}", live)
    xd = np.concatenate([np.zeros((cc, D), np.float32), x], axis=1)
    meter = {k: v for k, v in settings.items() if k in ("rms_mode", "meter_buf")}
    o = OracleMeter(meter, sample_rate=SR, channels=cc)
    outs, pos = [], 0
    for T_, hop in calls:
        outs.append(o.run(xd[:, pos: pos + T_ * hop], T_, hop, meter=not feed, rms=feed))
        pos += T_ * hop
    peak = settings.get("rms_mode") is False
    for k in (("rms",) if feed else ("db", "lin", "silent")):
        got = np.concatenate([v[k] for v in outs])
        if peak or k == "silent":
            assert np.array_equal(got, r[k]), (k, ms)
        else:
            np.testing.assert_allclose(got, r[k], rtol=1e-5, atol=1e-9 if k != "db" else 1e-4, err_msg=f"{k} {ms}")


WAVE_TAIL = 48    # newest entries of each tick's row kept in the record (at most that many of its new points)


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("width,meter_ms", [(800, 150), (300, 50)])
def test_wave_offset_plan_is_the_plugins_at_44100(width, meter_ms, ms):
    """The waveform with the offset's reserve of D samples: the model's points (and the engine's plan of a first call)
    against the plugin's ramp read-back, tick by tick, with 59.94 fps tick counts and a few odd packets."""
    from waveform_b200.engine import make_wave_config, preview_wave_plan

    D = sync_delay(SR, ms)
    settings = {"display_mode": "waveform", "width": width, "meter_buf": meter_ms, "channel_mode": "stereo"}
    hops = tick_counts(SR, (60000, 1001), 40) + [4410, 300, 97, 97] + [1470] * 6 + [44100, 441]
    ramp = _ramp(sum(hops))

    def live():
        r = _ref(settings={**settings, "audio_sync_offset": ms}, sample_rate=SR, channels=1)
        tail, pos = [], 0
        for hop in hops:
            tail.append(r.run_wave(ramp[:, pos: pos + hop], 1, hop)["out"][0, 1, width - WAVE_TAIL:])
            pos += hop
        return {"tail": np.stack(tail)}

    rec = reference(f"rates/sync_wave/{width}_{meter_ms}/{ms}", live)["tail"]
    plan = wave_plan(width, meter_ms, D, hops, SR)
    emitted = 0
    for t in range(len(hops)):   # the tick's new points are the raw samples; older entries have been through dBFS
        c = min(len(plan[t]), WAVE_TAIL)
        emitted += c
        assert np.array_equal(rec[t][WAVE_TAIL - c:], _picked(plan[t][len(plan[t]) - c:], ramp)), (t, hops[t], c)
    assert emitted > 0
    cfg = make_wave_config({k: v for k, v in settings.items() if k != "display_mode"} | {"audio_sync_offset": ms},
                           SR, channels=1)
    for hop in (735, 736, 1470):
        counts, src = preview_wave_plan(cfg, 40, hop)
        model = wave_plan(width, meter_ms, D, [hop] * 40, SR)
        assert np.array_equal(counts, [len(p) for p in model]), hop
        assert np.array_equal(src, np.concatenate(model).clip(min=-1)), hop
