"""The oracle against the UNMODIFIED reference (oracle/_ref/libwaveform_ref.so, compiled from its sources), including
the AVX2 path the plugin really executes.  What the reference computed on these inputs is stored in
tests/golden/reference_outputs.npz (tests/refdata.py): tables as digests, spectra and points as a fixed sample."""
import numpy as np
import pytest

from helpers import parity_report, synth_pcm
from oracle.oraclebind import OracleSource
from refdata import digest, frame_peak, reference, sample_index

TABLES = ("window", "slope", "rolloff", "interp_indices")
TICKS, BINS = 4, 32  # sampled ticks per case and bins (or points) per tick and channel


def _ref(impl=None, **kw):
    from oracle import refbind

    return refbind.RefSource(impl=refbind.IMPL_GENERIC if impl is None else impl, **kw)


CASES = [
    ({"fft_size": 1024, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 1),
    ({"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2),
    ({"fft_size": 2048, "window": "hann"}, 1),
    ({"fft_size": 2048, "window": "hamming", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "fast_peaks": True}, 2),
    ({"fft_size": 8192, "window": "blackman", "interp_mode": "lanczos", "filter_mode": "gauss", "filter_radius": 2.5}, 2),
    ({"fft_size": 800, "window": "power_of_sine", "sine_exponent": 3, "temporal_smoothing": "tv_exp_moving_avg",
      "gravity": 0.4, "log_scale": False, "interp_mode": "point"}, 1),
    ({"fft_size": 2048, "window": "none", "temporal_smoothing": "none", "display_mode": "bars", "interp_mode": "point",
      "normalize_volume": True}, 2),
    ({"fft_size": 1024, "display_mode": "bars", "interp_mode": "lanczos", "bar_width": 4, "bar_gap": 1,
      "filter_mode": "gauss", "mirror_freq_axis": True}, 2),
    ({"fft_size": 16384, "window": "hann"}, 1),
    ({"fft_size": 1024, "channel_mode": "stereo", "gravity": 0.2, "floor": -30}, 2),
]


@pytest.mark.parametrize("settings,channels", CASES)
def test_oracle_matches_compiled_reference(settings, channels):
    _compare(f"oracle_vs_reference/case{CASES.index((settings, channels))}", settings, channels)


@pytest.mark.parametrize("seed", range(40))
def test_randomised_settings_oracle_vs_compiled_reference(seed):
    """Differential fuzz of the oracle against the unmodified reference over the settings space the GPU fuzz
    (tests/test_gpu_scale.py::test_randomised_configs_against_oracle) draws from, plus the display options: every table bit for bit,
    every tick's spectrum within the parity criterion, silent flags and points."""
    rng = np.random.default_rng(4000 + seed)
    N = int(rng.choice([128, 512, 1024, 2048, 4096, 8192, 800, 720, 1600, 1920, 1456, 352, 2000, 4160, 1088]))
    mode = str(rng.choice(["mono", "mono", "stereo"]))
    channels = 2 if mode == "stereo" or rng.uniform() < 0.25 else 1
    settings = {"fft_size": N, "channel_mode": mode,
                "window": str(rng.choice(["none", "hann", "hamming", "blackman", "blackman_harris", "power_of_sine"])),
                "temporal_smoothing": str(rng.choice(["none", "exp_moving_avg", "exp_moving_avg", "tv_exp_moving_avg"])),
                "gravity": float(rng.choice([0.2, 0.5, 0.65, 0.9])), "floor": int(rng.choice([-30, -45, -65])),
                "display_mode": str(rng.choice(["curve", "curve", "bars"])),
                "interp_mode": str(rng.choice(["point", "lanczos", "catmull_rom"])),
                "log_scale": bool(rng.uniform() < 0.8)}
    if settings["window"] == "power_of_sine":
        settings["sine_exponent"] = int(rng.choice([1, 2, 3, 4]))
    if rng.uniform() < 0.3:
        settings.update(slope=float(rng.choice([0.25, 1.0])), fast_peaks=bool(rng.uniform() < 0.5))
    if rng.uniform() < 0.3:
        settings.update(rolloff_q=1.0, rolloff_rate=float(rng.choice([3.0, 9.0])))
    if rng.uniform() < 0.3:
        settings.update(filter_mode="gauss", filter_radius=float(rng.choice([1.5, 2.5])))
    if rng.uniform() < 0.2:
        settings["normalize_volume"] = True
    if settings["display_mode"] == "bars" and rng.uniform() < 0.5:
        settings.update(bar_width=int(rng.choice([2, 4, 24])), bar_gap=int(rng.choice([0, 1, 6])))
    hop_div = int(rng.choice([1, 2, 4]))
    _compare(f"oracle_vs_reference/seed{seed}", settings, channels, T=int(rng.choice([6, 14, 30])), hop_div=hop_div, seed=seed)


def _input(N, cc, T, hop, seed):
    x = synth_pcm(1, cc, (T - 1) * hop + N, seed=seed)[0]
    x[:, 6 * hop: 6 * hop + 4 * N] = 0
    if cc == 2:
        x[1, 12 * hop:] = 0  # one channel goes silent: exercises the stale-dB quirk
    return x


def _samples(N, n_points, seed):
    """The sampled bins and display points of a case (seeded: the same positions when recording and when testing)."""
    return sample_index((N // 2,), BINS, seed + 1), sample_index((n_points,), BINS, seed + 2)


def _compare(key, settings, channels, T=30, hop_div=2, seed=11):
    rms = (0.05 + 0.3 * np.random.default_rng(1).uniform(size=T)).astype(np.float32) if settings.get("normalize_volume") else None
    ticks = sample_index((T,), TICKS, seed)

    def live():
        ref = _ref(settings=settings, channels=channels)
        N, cc = ref.fft_size, ref.capture_channels
        a = ref.run_stft(_input(N, cc, T, N // hop_div, seed), T, N // hop_div, rms=rms, want_points=True)
        bins, pts = _samples(N, a["points"].shape[-1], seed)
        taps, kernel = ref.interp_kernel()
        return {"fft_size": N, "capture_channels": cc, "db_min": ref.db_min, "window_sum": ref.window_sum,
                **{name: digest(getattr(ref, name)()) for name in TABLES}, "taps": taps, "kernel": digest(kernel),
                "silent": a["silent"], "db": a["db"][ticks][..., bins], "peak": frame_peak(a["db"][ticks], ref.db_min),
                "num_points": a["points"].shape[-1], "points": a["points"][ticks][..., pts]}

    r = reference(key, live)
    N, cc = int(r["fft_size"]), int(r["capture_channels"])
    hop = N // hop_div
    orc = OracleSource(settings, channels=channels)
    b = orc.run_stft(_input(N, cc, T, hop, seed), T, hop, rms=rms, want_points=True)
    for name in TABLES:
        assert np.array_equal(digest(getattr(orc, name)()), r[name]), name
    assert np.float32(orc.window_sum) == r["window_sum"]
    taps, kernel = orc.interp_kernel()
    assert taps == int(r["taps"]) and np.array_equal(digest(kernel), r["kernel"])
    bins, pts = _samples(N, int(r["num_points"]), seed)
    assert b["points"].shape[-1] == int(r["num_points"])
    rep = parity_report(b["db"][ticks][..., bins], r["db"], db_min=float(r["db_min"]), peak=r["peak"])
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(r["silent"], b["silent"])
    d = np.abs(r["points"].astype(np.float64) - b["points"][ticks][..., pts].astype(np.float64))
    assert d.max() < 5e-3 and np.median(d) < 1e-4


def test_avx2_path_is_within_the_same_tolerance():
    """What the plugin runs on any recent x86 (WAVSourceAVX2, FMA EMA, sqrt(fma)) vs the generic parity target."""
    s = {"fft_size": 2048, "window": "hann"}

    def live():
        from oracle import refbind

        x = synth_pcm(1, 1, 20 * 2048, seed=5)[0]
        g, a = _ref(settings=s, channels=1), _ref(refbind.IMPL_AVX2, settings=s, channels=1)
        rg, ra = g.run_stft(x, 20, 2048), a.run_stft(x, 20, 2048)
        ticks, bins = sample_index((20,), TICKS, 5), sample_index((1024,), BINS, 6)
        return {"db_min": g.db_min, "generic": rg["db"][ticks][..., bins], "avx2": ra["db"][ticks][..., bins],
                "peak": frame_peak(rg["db"][ticks], g.db_min)}

    r = reference("oracle_vs_reference/avx2", live)
    rep = parity_report(r["avx2"], r["generic"], db_min=float(r["db_min"]), peak=r["peak"])
    assert rep["ok"], rep


def test_av_sync_offset_selects_older_frame():
    """Positive audio/video delay: tick_spectrum takes the OLDEST N of the last delay+N samples
    (src/source_generic.cpp:50-59)."""
    s = {"fft_size": 1024, "window": "hann", "temporal_smoothing": "none", "audio_sync_offset": 0}
    N = 1024
    x = synth_pcm(1, 1, 4 * N, seed=9)[0]

    def live():
        ref = _ref(settings=s, channels=1)
        ref.advance(4 * N / ref.sample_rate)
        ref.push(x[0])                      # packet ends "now"
        ref.tick()
        return {"latest": ref.decibels(0)}

    latest = reference("oracle_vs_reference/av_sync", live)["latest"]
    o = OracleSource({k: v for k, v in s.items() if k != "audio_sync_offset"}, channels=1)
    o.tick([x[0, -N:]])
    assert parity_report(latest, o.decibels(0))["ok"]


PX_CASES = [
    ({"fft_size": 1024, "display_mode": "curve", "interp_mode": "lanczos", "height": 300}, 1),
    ({"fft_size": 2048, "display_mode": "bars", "interp_mode": "catmull_rom", "rounded_caps": True, "min_bar_height": 5,
      "bar_width": 10, "bar_gap": 2}, 1),
    ({"fft_size": 1024, "display_mode": "curve", "channel_mode": "stereo", "channel_spacing": 20, "mirror_freq_axis": True,
      "filter_mode": "gauss", "height": 400}, 2),
    ({"fft_size": 1024, "display_mode": "bars", "channel_mode": "stereo", "channel_spacing": 10, "rounded_caps": True,
      "mirror_freq_axis": True, "interp_mode": "point"}, 2),
]


@pytest.mark.parametrize("settings,channels", PX_CASES)
def test_display_stage_matches_reference_render(settings, channels):
    """dB -> pixel lerp/clamp, mirroring and (miny, minpos): the oracle against WAVSource::render() itself
    (src/source.cpp:1346-1565 run verbatim behind the fake graphics API)."""
    T = 6

    def live():
        ref = _ref(settings=settings, channels=channels)
        N, cc = ref.fft_size, ref.capture_channels
        x = synth_pcm(1, cc, T * N, seed=4)[0]
        for t in range(T):
            ref.advance(N / ref.sample_rate)
            ref.push(x[0, t * N:(t + 1) * N], x[1, t * N:(t + 1) * N] if cc > 1 else None)
            ref.tick()
        ref.render()
        return {"fft_size": N, "capture_channels": cc,
                "decibels": np.stack([ref.decibels(c) for c in range(ref.display_channels)]),
                "render_buf": np.stack([ref.render_buf(c) for c in range(ref.display_channels)])}

    r = reference(f"oracle_vs_reference/render{PX_CASES.index((settings, channels))}", live)
    N, cc = int(r["fft_size"]), int(r["capture_channels"])
    orc = OracleSource(settings, channels=channels)
    x = synth_pcm(1, cc, T * N, seed=4)[0]
    for t in range(T):
        orc.tick([x[c, t * N:(t + 1) * N] for c in range(cc)])
    px, miny, minpos = orc.render_pixels()
    for c in range(len(r["render_buf"])):
        assert np.abs(r["render_buf"][c] - px[c]).max() < 5e-4
    # fed with the reference's own m_decibels only the interpolation's summation order differs: on an AVX machine
    # render() takes apply_interp_filter_fma3 (src/source.cpp:1383-1387), the oracle restates the generic template
    px2, _ = orc.pixels_of(r["decibels"])
    for c in range(len(r["render_buf"])):
        assert np.abs(r["render_buf"][c] - px2[c]).max() < 1e-4
