"""The C++ host-side mirror (waveform_b200/host/SpectrumSourceCUDA: ring buffers, A/V sync, timeout, live ticks through
the C-ABI) against the compiled reference driven with the SAME packet / tick schedule (what the reference computed is
stored under tests/golden/, tests/refdata.py: silent flags in full, the spectra of a fixed sample of ticks and bins)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from helpers import parity_report, synth_pcm
from refdata import frame_peak, reference, sample_index

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _build_driver(tmp_path):
    exe = tmp_path / "live_driver"
    lib = ROOT / "waveform_b200" / "lib"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT/'include'}", f"-I{ROOT/'waveform_b200'/'host'}",
                    str(ROOT / "tests" / "host" / "live_driver.cpp"), str(ROOT / "waveform_b200" / "host" / "spectrum_source.cpp"),
                    f"-L{lib}", "-lwfstft", f"-Wl,-rpath,{lib}", "-o", str(exe)], check=True)
    return exe


def _reference_live(settings, cc, pcm, N, packet, fps, ticks):
    from oracle import refbind

    ref = refbind.RefSource(settings, impl=refbind.IMPL_GENERIC, channels=cc)
    L, h = ref.L, ref.h
    now = 10 * 10**9
    tick_ns, pkt_ns = 10**9 // fps, packet * 10**9 // 48000
    next_pkt, pos = now, 0
    clock = now
    ns = pcm.shape[1]
    out, sil = [], []

    def set_clock(t):
        nonlocal clock
        assert t >= clock
        L.wfref_advance_clock_ns(h, t - clock)
        clock = t

    for _ in range(ticks):
        now += tick_ns
        while next_pkt + pkt_ns <= now and pos + packet <= ns:
            next_pkt += pkt_ns
            set_clock(next_pkt)
            ref.push(pcm[0, pos:pos + packet], pcm[1, pos:pos + packet] if cc > 1 else None)
            pos += packet
        set_clock(now)
        ref.tick(np.float32(1.0) / np.float32(fps))
        out.append(np.stack([ref.decibels(c) for c in range(ref.display_channels)]))
        sil.append(ref.last_silent)
    return np.stack(out), np.array(sil, dtype=np.uint8)


def _reference(N, cc, stereo, normalize, pcm, packet, fps, ticks):
    settings = {"fft_size": N, "channel_mode": "stereo" if stereo else "mono"}
    if normalize:  # the RMS feed runs live in both: capture_audio pre-accumulate + update_input_rms (not forced)
        settings["normalize_volume"] = True
    t_at, b_at = sample_index((ticks,), 8, N), sample_index((N // 2,), 64, N + 1)

    def live():
        ref, ref_sil = _reference_live(settings, cc, pcm, N, packet, fps, ticks)
        return {"silent": ref_sil, "db": ref[t_at][..., b_at], "peak": frame_peak(ref[t_at], -758.0)}

    return reference(f"live_adapter/{N}_{cc}_{stereo}_{normalize}", live), t_at, b_at


def _input(cc, ns):
    pcm = synth_pcm(1, cc, ns, seed=21)[0]
    pcm[:, 20000:] = 0.0  # goes silent: EMA decay, then the gate
    return pcm


CASES = [(4096, 2, 1, 0), (2048, 1, 0, 0), (1024, 2, 0, 0), (2048, 2, 1, 1), (800, 1, 0, 1)]
PACKET, FPS, TICKS, SAMPLES = 480, 60, 45, 48000


@pytest.mark.parametrize("N,cc,stereo,normalize", CASES)
def test_live_adapter_matches_reference_plugin(tmp_path, N, cc, stereo, normalize):
    exe = _build_driver(tmp_path)
    packet, fps, ticks = PACKET, FPS, TICKS
    ns = SAMPLES
    pcm = _input(cc, ns)
    inp, outp = tmp_path / "pcm.f32", tmp_path / "out.f32"
    pcm.astype(np.float32).tofile(inp)
    r = subprocess.run([str(exe), str(inp), str(cc), str(ns), str(N), str(packet), str(fps), str(ticks), str(outp),
                        str(stereo), str(normalize)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    B = N // 2
    dch = 2 if stereo else 1
    raw = np.fromfile(outp, dtype=np.uint8).reshape(ticks, dch * B * 4 + 1)
    got = raw[:, :-1].copy().view(np.float32).reshape(ticks, dch, B)
    got_sil = raw[:, -1]
    ref, t_at, b_at = _reference(N, cc, stereo, normalize, pcm, packet, fps, ticks)
    assert np.array_equal(got_sil, ref["silent"])
    rep = parity_report(got[t_at][..., b_at], ref["db"], peak=ref["peak"])
    assert rep["ok"], rep
