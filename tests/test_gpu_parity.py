"""GPU parity tests proper: the CUDA path (through the C-ABI) against the oracle on identical PCM.

Run on an H100:  python -m pytest tests -m gpu -x -q
"""
from __future__ import annotations

import numpy as np
import pytest

from helpers import check_points, parity_report, synth_pcm

pytestmark = pytest.mark.gpu


def _oracle_batch(settings, channels, pcm, T, hop, rms=None, want_points=False):
    from oracle.oraclebind import OracleSource

    S = pcm.shape[0]
    db, pts, sil = [], [], []
    for s in range(S):
        o = OracleSource(settings, channels=channels)
        r = o.run_stft(pcm[s], T, hop, rms=None if rms is None else rms[s], want_points=want_points)
        db.append(r["db"])
        pts.append(r["points"])
        sil.append(r["silent"])
    return np.stack(db), (np.stack(pts) if want_points else None), np.stack(sil)


def _engine(settings, channels, S):
    from waveform_b200 import Engine

    return Engine(settings, channels=channels, max_streams=S)


CASES = [
    # (settings, channels, hop_div)  — BASELINE configs 1..5 shapes first
    ({"fft_size": 1024, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 1, 1),  # config 1
    ({"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2, 4),                       # config 2
    ({"fft_size": 2048, "window": "hann"}, 1, 1),                                                            # config 3
    ({"fft_size": 8192, "window": "hann", "interp_mode": "lanczos"}, 1, 4),                                  # config 4
    ({"fft_size": 16384, "window": "hann"}, 1, 1),                                                           # config 5
    ({"fft_size": 2048, "window": "hamming", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "fast_peaks": True}, 2, 2),
    ({"fft_size": 2048, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.4}, 1, 2),
    ({"fft_size": 2048, "window": "none", "temporal_smoothing": "none"}, 1, 1),
    ({"fft_size": 2048, "window": "power_of_sine", "sine_exponent": 3, "slope": 1.0, "fast_peaks": True}, 1, 1),
    ({"fft_size": 8192, "window": "blackman", "interp_mode": "lanczos", "filter_mode": "gauss", "filter_radius": 2.5}, 2, 2),
    ({"fft_size": 128, "window": "none", "temporal_smoothing": "none"}, 1, 1),
    ({"fft_size": 256, "interp_mode": "point"}, 1, 2),
    ({"fft_size": 512, "display_mode": "bars", "interp_mode": "point", "bar_width": 8, "bar_gap": 2}, 2, 2),
    ({"fft_size": 1024, "display_mode": "bars", "interp_mode": "lanczos", "bar_width": 4, "bar_gap": 1,
      "filter_mode": "gauss", "mirror_freq_axis": True}, 2, 2),
    ({"fft_size": 4096, "log_scale": False, "interp_mode": "catmull_rom"}, 1, 2),
    ({"fft_size": 32768, "window": "hann"}, 1, 2),
    # sizes that are not powers of two (SURVEY §8f rank 1): the automatic size at 48 kHz/60 fps, slider steps of 64
    ({"fft_size": 800, "window": "hann"}, 1, 1),
    ({"fft_size": 1920, "window": "blackman", "channel_mode": "stereo"}, 2, 2),
    ({"fft_size": 192, "window": "hamming", "temporal_smoothing": "none"}, 1, 1),
    ({"fft_size": 4160, "window": "hann", "interp_mode": "lanczos", "filter_mode": "gauss"}, 2, 4),
    ({"fft_size": 8128, "window": "hann"}, 1, 2),
    ({"fft_size": 1456, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 1, 1),
    # the plugin's "large FFT" range: work buffers live in L2 instead of shared memory
    ({"fft_size": 65536, "window": "hann"}, 1, 4),
    ({"fft_size": 40000, "window": "blackman_harris", "interp_mode": "lanczos"}, 1, 2),
]


@pytest.mark.parametrize("settings,channels,hop_div", CASES)
def test_spectrum_parity_vs_oracle(settings, channels, hop_div):
    S, T = (5, 10) if settings["fft_size"] <= 32768 else (3, 5)
    eng = _engine(settings, channels, S)
    N = eng.fft_size
    hop = N // hop_div
    cc = eng.capture_channels
    pcm = synth_pcm(S, cc, (T - 1) * hop + N, zero_frames=[(1, 3, 7)], frame_len=N, hop=hop)
    out = eng.process(pcm, T, hop, want_points=True)
    ref_db, ref_pts, ref_sil = _oracle_batch(settings, channels, pcm, T, hop, want_points=True)
    rep = parity_report(out["db"], ref_db, db_min=eng.db_min)
    assert rep["ok"], rep
    assert rep["normwise"] < 1e-6, rep
    assert np.array_equal(out["silent"], ref_sil)
    # display points: the interpolation / Gaussian arithmetic itself (relative to the row's dB scale) ...
    assert check_points(settings, channels, out["db"], out["points"]) < 2e-6
    # ... and end to end against the oracle's points (dominated by the spectrum's own fp32 noise on faint bins)
    d = np.abs(out["points"].astype(np.float64) - ref_pts.astype(np.float64))
    assert np.median(d) < 1e-4 and np.nanmax(d) < 2e-2, (np.median(d), float(np.nanmax(d)))


GOLD = sorted((__import__("pathlib").Path(__file__).parent / "golden").glob("case_*.npz"))


@pytest.mark.parametrize("path", GOLD, ids=[p.stem for p in GOLD])
def test_cuda_engine_against_reference_golden_vectors(path):
    """The CUDA path against what the UNMODIFIED reference produced (fixtures generated by tests/golden/make_golden.py)."""
    import json
    z = np.load(path, allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    eng = _engine(settings, int(z["channels"]), 1)
    rms = z["rms"][None, :] if z["rms"].size else None
    out = eng.process(z["pcm"][None], int(z["n_frames"]), int(z["hop"]), seconds=float(z["seconds"]), input_rms=rms,
                      want_points=True)
    rep = parity_report(out["db"][0], z["db"], db_min=float(z["db_min"]))
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(out["silent"][0], z["silent"])
    assert check_points(settings, int(z["channels"]), out["db"], out["points"]) < 2e-6
    d = np.abs(out["points"][0].astype(np.float64) - z["points"].astype(np.float64))
    assert np.median(d) < 1e-4 and d.max() < 2e-2, (d.max(), np.median(d))


def test_fast2048_matches_generic_and_oracle(monkeypatch):
    """The hand-specialised N=2048 kernel and the generic kernel implement the same semantics."""
    import torch
    from waveform_b200 import Engine

    settings = {"fft_size": 2048, "window": "hann"}
    S, T, N = 37, 9, 2048
    pcm = synth_pcm(S, 1, T * N, zero_frames=[(2, 2, 6), (5, 0, 9)], frame_len=N, hop=N)
    fast = Engine(settings, channels=1, max_streams=S).process(torch.from_numpy(pcm).cuda(), T, N)
    monkeypatch.setenv("WF_FORCE_GENERIC", "1")
    gen = Engine(settings, channels=1, max_streams=S).process(torch.from_numpy(pcm).cuda(), T, N)
    monkeypatch.delenv("WF_FORCE_GENERIC")
    torch.cuda.synchronize()
    f, g = fast["db"].cpu().numpy(), gen["db"].cpu().numpy()
    ref_db, _, ref_sil = _oracle_batch(settings, 1, pcm, T, N)
    for name, got in (("fast", f), ("generic", g)):
        rep = parity_report(got, ref_db)
        assert rep["ok"] and rep["normwise"] < 1e-6, (name, rep)
    assert np.array_equal(fast["silent"].cpu().numpy(), ref_sil)
    assert np.array_equal(gen["silent"].cpu().numpy(), ref_sil)


def test_silence_gate_and_hold():
    """Digital silence: outputs decay under the EMA, then freeze once below floor-10 dB
    (src/source_generic.cpp:63-95); m_last_silent flips at the same tick as in the reference."""
    settings = {"fft_size": 2048, "window": "hann", "gravity": 0.3, "floor": -40}
    S, T, N = 3, 40, 2048
    pcm = synth_pcm(S, 1, T * N)
    pcm[:, :, 4 * N:] = 0.0
    pcm[2, :, 30 * N: 32 * N] = 0.1  # wakes up again
    eng = _engine(settings, 1, S)
    out = eng.process(pcm, T, N)
    ref_db, _, ref_sil = _oracle_batch(settings, 1, pcm, T, N)
    assert ref_sil.sum() > 0, "test must exercise the gate"
    assert np.array_equal(out["silent"], ref_sil)
    rep = parity_report(out["db"], ref_db, db_min=eng.db_min)
    assert rep["ok"], rep
    # held frames are bit-identical copies of the previous output
    s, t = np.argwhere(ref_sil == 1)[1]
    assert np.array_equal(out["db"][s, t], out["db"][s, t - 1])


def test_stereo_one_channel_silent_quirk():
    """One channel silent while the other plays: the reference re-applies dbfs() to the stale dB values of the
    skipped channel (SURVEY.md appendix A quirk); the engine reproduces it."""
    settings = {"fft_size": 1024, "window": "hann", "channel_mode": "stereo", "gravity": 0.2, "floor": -30}
    S, T, N = 2, 30, 1024
    pcm = synth_pcm(S, 2, T * N)
    pcm[:, 1, 3 * N:] = 0.0
    eng = _engine(settings, 2, S)
    out = eng.process(pcm, T, N)
    ref_db, _, ref_sil = _oracle_batch(settings, 2, pcm, T, N)
    assert np.array_equal(out["silent"], ref_sil)
    rep = parity_report(out["db"], ref_db, db_min=eng.db_min)
    assert rep["ok"], rep
    assert (ref_db[:, -1, 1] <= eng.db_min + 1).all()  # the quirk drove channel 1 to DB_MIN


def test_state_continues_across_calls_and_checkpoint():
    """EMA state persists in the engine between calls; get_state/set_state round-trips it."""
    settings = {"fft_size": 2048, "window": "hann"}
    S, T, N = 4, 12, 2048
    pcm = synth_pcm(S, 1, T * N)
    whole = _engine(settings, 1, S).process(pcm, T, N)["db"]
    eng = _engine(settings, 1, S)
    a = eng.process(pcm[:, :, : 5 * N], 5, N)["db"]
    state = eng.get_state()
    eng2 = _engine(settings, 1, S)
    eng2.set_state(state)
    b = eng2.process(pcm[:, :, 5 * N:], T - 5, N)["db"]
    assert np.array_equal(np.concatenate([a, b], axis=1), whole)


def test_reset_state_matches_timeout_branch():
    settings = {"fft_size": 2048, "window": "hann"}
    S, T, N = 2, 6, 2048
    pcm = synth_pcm(S, 1, T * N)
    eng = _engine(settings, 1, S)
    eng.process(pcm, T, N)
    eng.reset_state()
    st = eng.get_state()
    assert (st["tsmooth"] == 0).all() and (st["flags"] == 1).all()
    assert np.allclose(st["hold_db"], eng.db_min)
    from oracle.oraclebind import OracleSource
    o = OracleSource(settings, channels=1)
    o.run_stft(pcm[0], T, N)
    o.reset()
    r = o.run_stft(pcm[0], T, N)
    out = eng.process(pcm, T, N)
    assert parity_report(out["db"][0], r["db"])["ok"]


def test_volume_normalisation_and_skip_mask():
    settings = {"fft_size": 2048, "window": "hann", "normalize_volume": True, "volume_target": -8, "max_gain": 30}
    S, T, N = 3, 8, 2048
    pcm = synth_pcm(S, 1, T * N)
    rng = np.random.default_rng(5)
    rms = (0.02 + 0.3 * rng.uniform(size=(S, T))).astype(np.float32)
    eng = _engine(settings, 1, S)
    out = eng.process(pcm, T, N, input_rms=rms)
    ref_db, _, _ = _oracle_batch(settings, 1, pcm, T, N, rms=rms)
    d = np.abs(out["db"].astype(np.float64) - ref_db)
    assert d.max() < 2e-3 and np.median(d) < 2e-5, (d.max(), np.median(d))
    # bin 0 is not compensated (loop starts at i = 1, src/source_generic.cpp:165)
    plain = _engine({"fft_size": 2048, "window": "hann"}, 1, S).process(pcm, T, N)["db"]
    assert np.allclose(out["db"][..., 0], plain[..., 0], atol=1e-4)


def test_unaligned_hop_and_host_device_paths_agree():
    import torch
    settings = {"fft_size": 2048, "window": "hann"}
    S, T, N, hop = 3, 7, 2048, 801  # odd hop -> scalar-load path of the generic kernel
    pcm = synth_pcm(S, 1, (T - 1) * hop + N)
    host = _engine(settings, 1, S).process(pcm, T, hop)["db"]
    dev = _engine(settings, 1, S).process(torch.from_numpy(pcm).cuda(), T, hop)["db"].cpu().numpy()
    assert np.array_equal(host, dev)
    ref_db, _, _ = _oracle_batch(settings, 1, pcm, T, hop)
    assert parity_report(host, ref_db)["ok"]


def test_known_answers():
    """Analytic vectors (SURVEY.md §8c): impulse, exact-bin sine, DC, silence."""
    N = 2048
    eng = _engine({"fft_size": N, "window": "none", "temporal_smoothing": "none"}, 1, 1)
    x = np.zeros((1, 1, N), np.float32)
    x[0, 0, 0] = 1.0
    db = eng.process(x, 1, N)["db"][0, 0, 0]
    assert np.allclose(db, 20 * np.log10(2.0 / N), atol=1e-4)
    x[:] = 0.25  # DC c -> bin 0 = 20 log10(2c)
    db = _engine({"fft_size": N, "window": "none", "temporal_smoothing": "none"}, 1, 1).process(x, 1, N)["db"][0, 0, 0]
    assert abs(db[0] - 20 * np.log10(0.5)) < 1e-4
    n = np.arange(N)
    x[0, 0] = np.sin(2 * np.pi * 100 * n / N).astype(np.float32)
    db = _engine({"fft_size": N, "window": "hann", "temporal_smoothing": "none"}, 1, 1).process(x, 1, N)["db"][0, 0, 0]
    assert abs(db[100]) < 1e-2 and abs(db[99] + 6.02) < 2e-2 and abs(db[101] + 6.02) < 2e-2
    x = np.zeros((1, 1, 2 * N), np.float32)
    e = _engine({"fft_size": N, "window": "hann"}, 1, 1)
    o = e.process(x, 3, N // 4)
    assert (o["db"] == e.db_min).all() and (o["silent"] == 1).all()


def test_peak_normalise_and_errors():
    import torch
    from waveform_b200 import Engine, WfError

    settings = {"fft_size": 2048, "window": "hann"}
    S, T, N = 6, 4, 2048
    pcm = synth_pcm(S, 1, T * N)
    eng = _engine(settings, 1, S)
    out = eng.process(torch.from_numpy(pcm).cuda(), T, N, want_peak=True)
    db = out["db"].cpu().numpy()
    peak = out["peak"].cpu().numpy()
    assert np.allclose(peak, db[..., 1:].max(axis=(0, 2, 3)), atol=0)
    data = out["db"].clone()
    eng.peak_normalize(data, out["peak"], target_db=-3.0, max_gain=20.0)
    eng.synchronize()
    gain = np.minimum(-3.0 - peak, 20.0)
    exp = db.copy()
    exp[..., 1:] += gain[None, :, None, None]
    assert np.allclose(data.cpu().numpy(), exp, atol=1e-5)
    with pytest.raises(WfError) as ei:
        Engine({"fft_size": 70000}, channels=1)   # beyond the plugin's 65536 maximum: an explicit error, never a guess
    assert ei.value.status == -2
    with pytest.raises(WfError) as ei:
        eng.process(np.zeros((S + 1, 1, N), np.float32), 1, N)
    assert ei.value.status == -6


@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_subwarp_groups_diverge_independently(N):
    """N <= 1024 packs several streams into one warp.  A gated (silent) stream next to active ones, with the peak
    reduction and display points requested, exercises warp primitives under group-divergent control flow
    (regression: collectives must name only the calling group's lanes; found by compute-sanitizer)."""
    import torch
    settings = {"fft_size": N, "window": "hann", "floor": -40, "gravity": 0.3}
    S, T = 9, 24
    pcm = synth_pcm(S, 1, T * N)
    pcm[0] = 0.0
    pcm[4, :, 5 * N:] = 0.0
    eng = _engine(settings, 1, S)
    out = eng.process(torch.from_numpy(pcm).cuda(), T, N, want_points=True, want_peak=True)
    torch.cuda.synchronize()
    ref_db, ref_pts, ref_sil = _oracle_batch(settings, 1, pcm, T, N, want_points=True)
    got = out["db"].cpu().numpy()
    assert np.array_equal(out["silent"].cpu().numpy(), ref_sil) and ref_sil.sum() > T
    assert parity_report(got, ref_db, db_min=eng.db_min)["ok"]
    assert np.allclose(out["peak"].cpu().numpy(), got[..., 1:].max(axis=(0, 2, 3)))
    assert check_points(settings, 1, got, out["points"].cpu().numpy()) < 2e-6


@pytest.mark.parametrize("settings,channels", [
    ({"fft_size": 1024, "display_mode": "curve", "interp_mode": "lanczos", "height": 300}, 1),
    ({"fft_size": 2048, "display_mode": "bars", "interp_mode": "catmull_rom", "rounded_caps": True, "min_bar_height": 5,
      "bar_width": 10, "bar_gap": 2}, 1),
    ({"fft_size": 1024, "display_mode": "curve", "channel_mode": "stereo", "channel_spacing": 20, "mirror_freq_axis": True,
      "filter_mode": "gauss", "height": 400}, 2),
    ({"fft_size": 4096, "display_mode": "bars", "channel_mode": "stereo", "channel_spacing": 10, "rounded_caps": True,
      "mirror_freq_axis": True, "interp_mode": "point"}, 2),
    ({"fft_size": 800, "display_mode": "curve", "interp_mode": "catmull_rom", "height": 225}, 1),
])
def test_display_stage_pixels(settings, channels):
    """SURVEY §8(f) rank 3: dB -> pixel heights, mirroring and (miny, minpos) in the kernel epilogue, against the oracle's
    restatement of render_curve / render_bars (itself checked against WAVSource::render in test_oracle_vs_reference)."""
    from oracle.oraclebind import OracleSource
    S, T = 4, 6
    eng = _engine(settings, channels, S)
    N = eng.fft_size
    pcm = synth_pcm(S, eng.capture_channels, T * N)
    out = eng.process(pcm, T, N, want_points=True, want_pixels=True)
    o = OracleSource(settings, channels=channels)
    exp_px, exp_min = o.pixels_of(out["db"])
    assert np.abs(out["pixels"] - exp_px).max() < 2e-4, float(np.abs(out["pixels"] - exp_px).max())
    assert np.abs(out["min"][..., 0] - exp_min[..., 0]).max() < 2e-4
    same = out["min"][..., 1] == exp_min[..., 1]
    assert same.mean() > 0.9  # an exact tie between two points can flip under a 1e-5 px difference
    assert check_points(settings, channels, out["db"], out["points"]) < 2e-6


# ---- the cluster ("wide") kernel: R CTAs per stream working on R ticks at once (csrc/wf_wide.cuh) ----------------

WIDE_CASES = [
    # (settings, channels, hop_div, T) — T not a multiple of R, stereo, mono-mix, display stages, gate-heavy
    ({"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2, 4, 13),
    ({"fft_size": 8192, "window": "hann", "interp_mode": "lanczos", "filter_mode": "gauss"}, 1, 4, 11),
    ({"fft_size": 16384, "window": "hann", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "fast_peaks": True}, 2, 2, 9),
    ({"fft_size": 4096, "display_mode": "bars", "interp_mode": "catmull_rom", "mirror_freq_axis": True}, 2, 2, 10),
    ({"fft_size": 32768, "window": "hann"}, 1, 2, 5),
]


@pytest.mark.parametrize("v3", ["1", "0"])
@pytest.mark.parametrize("R", [2, 4, 8])
@pytest.mark.parametrize("settings,channels,hop_div,T", WIDE_CASES)
def test_wide_kernel_is_bit_identical_to_one_group_kernel(settings, channels, hop_div, T, R, v3, monkeypatch):
    """Distributing a stream's bins over a cluster must not change a single bit: the recurrences are only
    distributed, never reassociated.  Also checks both against the oracle.  v3 = "1": the CTA-per-tick kernel
    (csrc/wf_v3.cuh, cluster size 1 vs R; 16384 has no size-1 variant, so 2 vs R); "0": the first-generation pair
    (wf_kernels.cuh vs wf_wide.cuh)."""
    import torch
    from waveform_b200 import Engine

    S = 3
    monkeypatch.setenv("WF_V3", v3)
    monkeypatch.setenv("WF_WIDE_R", "1")
    e1 = Engine(settings, channels=channels, max_streams=S)
    monkeypatch.setenv("WF_WIDE_R", str(R))
    e2 = Engine(settings, channels=channels, max_streams=S)
    N = e1.fft_size
    hop = N // hop_div
    cc = e1.capture_channels
    pcm = synth_pcm(S, cc, (T - 1) * hop + N, zero_frames=[(1, 2, 6)], frame_len=N, hop=hop)
    x = torch.from_numpy(pcm).cuda()
    a = e1.process(x, T, hop, want_points=True, want_peak=True)
    b = e2.process(x, T, hop, want_points=True, want_peak=True)
    torch.cuda.synchronize()
    for key in ("db", "points", "silent", "peak"):
        assert np.array_equal(a[key].cpu().numpy(), b[key].cpu().numpy()), key
    sa, sb = e1.get_state(), e2.get_state()
    for key in ("tsmooth", "hold_db", "flags"):
        assert np.array_equal(sa[key], sb[key]), key
    ref_db, _, ref_sil = _oracle_batch(settings, channels, pcm, T, hop)
    rep = parity_report(b["db"].cpu().numpy(), ref_db, db_min=e2.db_min)
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(b["silent"].cpu().numpy(), ref_sil)


@pytest.mark.parametrize("v3", ["1", "0"])
@pytest.mark.parametrize("R", [1, 2, 8])
def test_wide_kernel_gate_hold_and_wakeup(R, v3, monkeypatch):
    """Silence inside a round of R ticks: decay, freeze below floor-10 dB, wake-up — the lazily evaluated cluster-wide
    reduction must flip m_last_silent on the same tick as the reference (src/source_generic.cpp:63-95)."""
    monkeypatch.setenv("WF_V3", v3)
    monkeypatch.setenv("WF_WIDE_R", str(R))
    settings = {"fft_size": 4096, "window": "hann", "gravity": 0.3, "floor": -40, "channel_mode": "stereo"}
    S, T, N = 3, 37, 4096
    pcm = synth_pcm(S, 2, T * N)
    pcm[:, :, 3 * N:] = 0.0
    pcm[1, 1, 5 * N: 9 * N] = 0.05   # one channel keeps playing for a while
    pcm[2, :, 29 * N: 31 * N] = 0.1  # wakes up again
    eng = _engine(settings, 2, S)
    out = eng.process(pcm, T, N)
    ref_db, _, ref_sil = _oracle_batch(settings, 2, pcm, T, N)
    assert ref_sil.sum() > 0, "test must exercise the gate"
    assert np.array_equal(out["silent"], ref_sil)
    rep = parity_report(out["db"], ref_db, db_min=eng.db_min)
    assert rep["ok"], rep
    # state carries over a call boundary that falls inside the silent stretch
    eng2 = _engine(settings, 2, S)
    a = eng2.process(pcm[:, :, : 6 * N], 6, N)
    b = eng2.process(pcm[:, :, 6 * N:], T - 6, N)
    assert np.array_equal(np.concatenate([a["db"], b["db"]], axis=1), out["db"])
    assert np.array_equal(np.concatenate([a["silent"], b["silent"]], axis=1), out["silent"])
