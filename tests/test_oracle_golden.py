"""The oracle (plain-C restatement) against the golden vectors generated from the UNMODIFIED reference
(tests/golden/make_golden.py).  CPU only; this is what pins the oracle when oracle/_ref is not around."""
import json
from pathlib import Path

import numpy as np
import pytest

from helpers import parity_report
from oracle.oraclebind import OracleSource

GOLD = sorted((Path(__file__).parent / "golden").glob("case_*.npz"))


def _load(path):
    z = np.load(path, allow_pickle=False)
    return z, json.loads(str(z["settings"]))


@pytest.mark.parametrize("path", GOLD, ids=[p.stem for p in GOLD])
def test_oracle_reproduces_reference_golden(path):
    z, settings = _load(path)
    o = OracleSource(settings, channels=int(z["channels"]))
    rms = z["rms"] if z["rms"].size else None
    r = o.run_stft(z["pcm"], int(z["n_frames"]), int(z["hop"]), seconds=float(z["seconds"]), rms=rms, want_points=True)
    # tables: bit-exact with what WAVSource::update() built
    for name, got in (("window", o.window()), ("slope", o.slope()), ("rolloff", o.rolloff()),
                      ("interp_indices", o.interp_indices())):
        exp = z[name]
        if exp.size == 0:
            assert got is None
        else:
            assert np.array_equal(got, exp), name
    assert np.float32(o.window_sum) == z["window_sum"]
    assert np.float32(o.db_min) == z["db_min"]
    taps, w = o.interp_kernel()
    if z["interp_weights"].size:
        assert np.array_equal(w, z["interp_weights"])
    bw = o.band_widths()
    if z["band_widths"].size:
        assert np.array_equal(bw, z["band_widths"])
    gk, _, gs = o.gauss_kernel()
    if z["gauss"].size:
        assert np.array_equal(gk, z["gauss"]) and np.float32(gs) == z["gauss_sum"]
    # spectra: the FFT arithmetic differs from FFTW's codelets in the last bits -> parity metric, not bit equality
    rep = parity_report(r["db"], z["db"], db_min=float(z["db_min"]))
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(r["silent"], z["silent"])
    d = np.abs(r["points"].astype(np.float64) - z["points"].astype(np.float64))
    assert d.max() < 5e-3 and np.median(d) < 1e-4, (d.max(), np.median(d))


def test_known_answers_oracle():
    """Analytic vectors (SURVEY.md §8c)."""
    N = 1024
    o = OracleSource({"fft_size": N, "window": "none", "temporal_smoothing": "none"}, channels=1)
    x = np.zeros((1, N), np.float32)
    x[0, 0] = 1.0
    db = o.run_stft(x, 1, N)["db"][0, 0]
    assert np.allclose(db, 20 * np.log10(2.0 / N), atol=1e-4)          # impulse: flat spectrum
    x[:] = 0.25
    db = OracleSource({"fft_size": N, "window": "none", "temporal_smoothing": "none"}, channels=1).run_stft(x, 1, N)["db"][0, 0]
    assert abs(db[0] - 20 * np.log10(0.5)) < 1e-4                       # DC c -> 20 log10(2c)
    n = np.arange(N)
    x[0] = np.sin(2 * np.pi * 64 * n / N)
    db = OracleSource({"fft_size": N, "window": "hann", "temporal_smoothing": "none"}, channels=1).run_stft(x, 1, N)["db"][0, 0]
    assert abs(db[64]) < 2e-2 and abs(db[63] + 6.02) < 3e-2             # exact-bin sine under Hann
    # EMA step response y_t = g y_{t-1} + (1-g) x
    g = 0.65
    o = OracleSource({"fft_size": N, "window": "none", "gravity": g}, channels=1)
    x[:] = 0.25
    dbs = o.run_stft(np.tile(x, (1, 6)), 6, N)["db"][:, 0, 0]
    y, exp = 0.0, []
    for _ in range(6):
        y = g * y + (1 - g) * 0.5
        exp.append(20 * np.log10(y))
    assert np.allclose(dbs, exp, atol=1e-4)
    # silence -> DB_MIN and gated
    z = np.zeros((1, 3 * N), np.float32)
    o = OracleSource({"fft_size": N}, channels=1)
    r = o.run_stft(z, 3, N)
    assert (r["db"] == np.float32(o.db_min)).all() and r["silent"].all()


def test_r2c_against_float64_dft():
    from oracle.oraclebind import r2c
    rng = np.random.default_rng(3)
    for n in (128, 736, 800, 1024, 2048, 4096, 16384):
        x = rng.standard_normal(n).astype(np.float32)
        t = np.fft.rfft(x.astype(np.float64))
        assert np.abs(r2c(x) - t).max() / np.abs(t).max() < 5e-7


STALL = sorted((Path(__file__).parent / "golden").glob("stall_*.npz"))


def stall_calls(z):
    """Engine-call view of a stall fixture: [(pcm_view [cc, samples], n_frames, skip[n_frames])]."""
    hop, N = int(z["hop"]), json.loads(str(z["settings"]))["fft_size"]
    out = []
    for c in json.loads(str(z["calls"])):
        n = int(c["n_frames"])
        out.append((z["pcm"][:, c["offset"]: c["offset"] + (n - 1) * hop + N], n, np.array(c["skip"], np.uint8)))
    return out


@pytest.mark.parametrize("path", STALL, ids=[p.stem for p in STALL])
def test_oracle_reproduces_reference_not_enough_audio(path):
    """'Not enough audio' ticks (src/source_generic.cpp:55-61) as the compiled reference produced them when audio was
    stamped ahead of the tick clock; the oracle is driven with frame = NULL on the skipped ticks."""
    z, settings = _load(path)
    o = OracleSource(settings, channels=int(z["channels"]))
    hop, N = int(z["hop"]), settings["fft_size"]
    t = 0
    assert sum(int(s.sum()) for _, _, s in stall_calls(z)) >= 2, "fixture must contain skipped ticks"
    for pcm, n, skip in stall_calls(z):
        for i in range(n):
            frames = [None if skip[i] else pcm[ch, i * hop: i * hop + N] for ch in range(pcm.shape[0])]
            o.tick(frames, float(z["seconds"]))
            got = np.stack([o.decibels(ch) for ch in range(o.display_channels)])
            rep = parity_report(got, z["db"][t], db_min=float(z["db_min"]))
            assert rep["ok"], (t, rep)
            assert o.last_silent == bool(z["silent"][t]), t
            t += 1
    assert t == int(z["n_frames"])


def test_fp64_arbiter_reference_and_oracle():
    """SURVEY §4(ii)/§7: the error of the reference's FFTW path (golden vectors) and of the oracle's own fp32 FFT against
    a double-precision ground truth computed from the same float32 window table.  Both are ~1e-7 normwise; the GPU
    variant of this test (tests/test_gpu_scale.py) holds the CUDA path to the same yardstick."""
    from fp64_spectrum import Fp64Spectrum

    z, settings = _load(Path(__file__).parent / "golden" / "case_c3_mono_2048_hann.npz")
    T, hop = int(z["n_frames"]), int(z["hop"])
    o = OracleSource(settings, channels=1)
    truth = Fp64Spectrum(settings, channels=1).run(z["pcm"], T, hop, o.gravity(float(z["seconds"])))["db"][:, 0]
    got = o.run_stft(z["pcm"], T, hop, seconds=float(z["seconds"]))["db"][:, 0]
    lin = lambda d: np.power(10.0, np.asarray(d, np.float64) / 20.0)
    peak = lin(truth).max(axis=-1, keepdims=True)
    err_ref = (np.abs(lin(z["db"][:, 0]) - lin(truth)) / peak).max()
    err_port = (np.abs(lin(got) - lin(truth)) / peak).max()
    assert err_ref < 1e-6 and err_port < 1e-6, (err_ref, err_port)
