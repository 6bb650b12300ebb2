"""The drop-in boundary as a COMPILED artefact: waveform_b200/host/source_cuda.hpp (class WAVSourceCUDA, the binding
INTEGRATION.md §1 shows) built against the UNMODIFIED reference sources (source.cpp & co.) + the fake libobs, driven through
the plugin's own update() / capture_output_bus() / tick(), tick for tick against WAVSourceGeneric driven the same way.

Everything above tick_spectrum() (settings, ring buffers, A/V sync, update_input_rms, the timeout branch) is the
reference's own code in both runs; only the per-frame pipeline differs (FFTW + scalar loops vs libwfstft.so)."""
import numpy as np
import pytest

from helpers import parity_report, synth_pcm

pytestmark = pytest.mark.gpu


def _pair(settings, channels):
    from oracle import refbind

    if not (refbind.available() and refbind.cuda_seam_available()):
        pytest.skip("oracle/_ref libraries not built (needs the reference sources)")
    return (refbind.RefSource(settings, impl=refbind.IMPL_GENERIC, channels=channels),
            refbind.RefSource(settings, impl=refbind.IMPL_CUDA, channels=channels))


SEAM_CASES = [
    ({"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2, 800),      # BASELINE configs[1] shape
    ({"fft_size": 2048, "window": "hann"}, 1, 800),                                             # headline kernel family, 1 stream
    ({"fft_size": 1024, "window": "hamming", "slope": 0.75, "rolloff_q": 1.5, "rolloff_rate": 9.0, "fast_peaks": True}, 2, 512),
    ({"fft_size": 800, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5}, 1, 800),
    ({"fft_size": 8192, "window": "hann", "gravity": 0.3, "floor": -40}, 1, 1600),
]


@pytest.mark.parametrize("settings,channels,hop", SEAM_CASES)
def test_wavsource_cuda_matches_wavsource_generic_tick_for_tick(settings, channels, hop):
    gen, cuda = _pair(settings, channels)
    N, T = gen.fft_size, 40
    assert cuda.fft_size == N and cuda.capture_channels == gen.capture_channels
    cc = gen.capture_channels
    pcm = synth_pcm(1, cc, (T - 1) * hop + N, seed=5)[0]
    pcm[:, 12 * hop: 30 * hop] = 0.0          # decays, freezes (floor -40 case), then wakes up again
    a = gen.run_stft(pcm, T, hop)
    b = cuda.run_stft(pcm, T, hop)
    assert a["frames"] == b["frames"] == T
    assert np.array_equal(a["silent"], b["silent"])
    rep = parity_report(b["db"], a["db"], db_min=gen.db_min)
    # two independent fp32 FFTs (FFTW's codelets vs the CUDA passes), each ~4e-7 from a double-precision DFT
    # (tests/test_gpu_scale.py::test_fp64_arbiter_*): up to 1.3e-6 from each other over 40 ticks
    assert rep["ok"] and rep["normwise"] < 2e-6, rep


def test_wavsource_cuda_volume_normalisation_live_rms_and_hide_show():
    """m_input_rms comes from the reference's own capture_audio / update_input_rms in both runs (not forced): the RMS feed
    works live through the seam.  Then hide() -> the timeout branch (reset once, DB_MIN, m_last_silent) -> show()."""
    settings = {"fft_size": 2048, "window": "hann", "normalize_volume": True, "channel_mode": "stereo"}
    gen, cuda = _pair(settings, 2)
    hop, N = 800, 2048
    pcm = synth_pcm(1, 2, 80 * hop + N, seed=9)[0] * 0.3
    out = {}
    for name, src in (("gen", gen), ("cuda", cuda)):
        rows, sil, rms = [], [], []
        for t in range(80):
            if t == 40:
                src.set_showing(False)
            if t == 50:
                src.set_showing(True)
            src.advance(hop / 48000.0)
            src.push(pcm[0, t * hop:(t + 1) * hop], pcm[1, t * hop:(t + 1) * hop])
            src.tick(1.0 / 60.0)
            rows.append(np.stack([src.decibels(0), src.decibels(1)]))
            sil.append(src.last_silent)
            rms.append(src.L.wfref_input_rms(src.h))
        out[name] = (np.stack(rows), np.array(sil), np.array(rms))
    assert np.array_equal(out["gen"][2], out["cuda"][2]) and out["gen"][2][-1] > 0      # identical live RMS feed
    assert np.array_equal(out["gen"][1], out["cuda"][1]) and out["gen"][1][40:50].all()  # hidden -> m_last_silent
    g, c = out["gen"][0], out["cuda"][0]
    assert (c[40:50] == gen.db_min).all()
    d = np.abs(g.astype(np.float64) - c.astype(np.float64))
    assert d.max() < 2e-3 and np.median(d) < 2e-5, (d.max(), np.median(d))               # dB domain (gain added after dbfs)
    rep = parity_report(c[50:], g[50:], db_min=gen.db_min)                                # EMA restarted from zero after show()
    assert rep["same_floor"]
