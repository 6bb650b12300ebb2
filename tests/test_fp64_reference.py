"""The float64 restatement of tick_spectrum (tests/fp64_spectrum.py) against the oracle and the compiled reference's own
outputs (tests/golden/), and both float32 implementations' error against it.  CPU only.

The reference's error on the fp64_* fixtures is the yardstick the GPU kernels are held to (tests/test_gpu_fp64.py)."""
import json
from pathlib import Path

import numpy as np
import pytest

from fp64_spectrum import Fp64Spectrum, normwise_vs_truth
from helpers import parity_report
from oracle.oraclebind import OracleSource

GOLDEN = Path(__file__).parent / "golden"
FP64 = sorted(GOLDEN.glob("fp64_*.npz"))


def _load(path):
    z = np.load(path, allow_pickle=False)
    return z, json.loads(str(z["settings"]))


def _truth(z, settings, rms=None, skip=None):
    o = OracleSource(settings, channels=int(z["channels"]))
    f = Fp64Spectrum(settings, channels=int(z["channels"]))
    T, hop = int(z["n_frames"]), int(z["hop"])
    return f.run(z["pcm"], T, hop, o.gravity(float(z["seconds"])), input_rms=rms, skip_mask=skip)


@pytest.mark.parametrize("path", FP64, ids=[p.stem for p in FP64])
def test_fp64_restatement_matches_oracle_and_reference(path):
    """Within the parity criterion of both float32 implementations, with identical silent flags; and each of them is within
    1e-6 normwise of the float64 truth on every frame (the figures are printed: `pytest -s`)."""
    z, settings = _load(path)
    T, hop = int(z["n_frames"]), int(z["hop"])
    truth = _truth(z, settings)
    orc = OracleSource(settings, channels=int(z["channels"])).run_stft(z["pcm"], T, hop, seconds=float(z["seconds"]))
    db_min = float(z["db_min"])
    for name, db, sil in (("oracle", orc["db"], orc["silent"]), ("reference", z["db"], z["silent"])):
        rep = parity_report(truth["db"], db, db_min=db_min)
        assert rep["ok"] and rep["normwise"] < 1e-6, (name, rep)
        assert np.array_equal(truth["silent"], sil.astype(bool)), name
    err_orc = normwise_vs_truth(orc["db"], truth["db"], db_min).max()
    err_ref = normwise_vs_truth(z["db"], truth["db"], db_min).max()
    print(f"{path.stem}: N={settings['fft_size']} normwise vs float64: reference {err_ref:.2e}, oracle {err_orc:.2e}")
    assert err_ref < 1e-6 and err_orc < 1e-6, (err_ref, err_orc)


# The reference's other golden cases exercise what the fp64_* cases leave at their defaults: slope, roll-off, fast peaks,
# volume normalisation, the 2 -> 1 channel mix, stereo, TV-exponential gravity, the silence gate and hold.
CASES = sorted(GOLDEN.glob("case_*.npz"))


@pytest.mark.parametrize("path", CASES, ids=[p.stem for p in CASES])
def test_fp64_restatement_matches_reference_all_options(path):
    z, settings = _load(path)
    truth = _truth(z, settings, rms=z["rms"] if z["rms"].size else None)
    rep = parity_report(truth["db"], z["db"], db_min=float(z["db_min"]))
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(truth["silent"], z["silent"].astype(bool))


STALL = sorted(GOLDEN.glob("stall_*.npz"))


@pytest.mark.parametrize("path", STALL, ids=[p.stem for p in STALL])
def test_fp64_restatement_matches_reference_not_enough_audio(path):
    """Skipped ticks (skip_mask): the channel keeps its stale m_decibels row, which goes through dbfs() again."""
    z, settings = _load(path)
    cc, hop = int(z["channels"]), int(z["hop"])
    f = Fp64Spectrum(settings, channels=cc)
    g = OracleSource(settings, channels=cc).gravity(float(z["seconds"]))
    dbs, sil = [], []
    for c in json.loads(str(z["calls"])):
        n = int(c["n_frames"])
        r = f.run(z["pcm"][:, c["offset"]:], n, hop, g, skip_mask=np.array(c["skip"], np.uint8))
        dbs.append(r["db"])
        sil.append(r["silent"])
    rep = parity_report(np.concatenate(dbs), z["db"], db_min=float(z["db_min"]))
    assert rep["ok"], rep
    assert np.array_equal(np.concatenate(sil), z["silent"].astype(bool))


def test_fp64_restatement_known_answers():
    """Analytic values: an impulse has a flat spectrum 2/N, DC c gives 2c at bin 0, an exact-bin sine of amplitude a
    gives a at its bin (rectangular window), and the EMA is g·old + (1-g)·new with the float32 gravity."""
    N = 1024
    f = Fp64Spectrum({"fft_size": N, "window": "none", "temporal_smoothing": "none"}, channels=1)
    x = np.zeros(N, np.float32)
    x[0] = 1.0
    db, _ = f.tick([x], 0.0)
    assert np.allclose(db[0], 20 * np.log10(2.0 / N), atol=1e-12, rtol=0)
    x[:] = 0.25
    db, _ = f.tick([x], 0.0)
    assert abs(db[0, 0] - 20 * np.log10(0.5)) < 1e-12
    n = np.arange(N)
    x = (0.5 * np.sin(2 * np.pi * 3 * n / N)).astype(np.float32)
    db, _ = f.tick([x], 0.0)
    assert abs(db[0, 3] - 20 * np.log10(0.5)) < 1e-6
    g = np.float32(0.65)
    f = Fp64Spectrum({"fft_size": N, "window": "none", "gravity": 0.65}, channels=1)
    x = np.full(N, 0.25, np.float32)
    y = 0.0
    for _ in range(4):
        db, _ = f.tick([x], g)
        y = float(g) * y + float(np.float32(1) - g) * 0.5
        assert abs(db[0, 0] - 20 * np.log10(y)) < 1e-12
    assert abs(f.state[0, 0] - y) < 1e-15
