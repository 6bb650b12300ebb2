#!/usr/bin/env python
"""Measurements for the SURVEY §8(f) 'next' rows already built:
  rank 1  non-power-of-two N (any-N kernel): device-resident throughput + fraction of the measured HBM roofline
  rank 2  live adapter: per-tick latency of wf_process (1 source, 1 tick, host buffers) next to the reference's
          own tick_spectrum on one host core (oracle/_ref)."""
import json, sys, time
from pathlib import Path
import numpy as np
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch
from waveform_b200 import Engine
from helpers import synth_pcm

PEAK = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0
print("== rank 1: non-power-of-two sizes, device-resident, S=4096 streams x T=16 ticks, hop=N")
for N in (800, 720, 960, 1600, 1920, 2000, 4160):
    S, T = 4096, 16
    eng = Engine({"fft_size": N, "window": "hann"}, channels=1, max_streams=S)
    pcm = (torch.rand((S, 1, T * N), device="cuda") - 0.5) * 0.5
    out = torch.empty((S, T, 1, N // 2), device="cuda")
    st = torch.cuda.Stream()
    step = lambda: eng.process_raw(pcm.data_ptr(), S, T, N, T * N, T * N, out_db=out.data_ptr(), stream=st.cuda_stream, sync=False)
    for _ in range(3): step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(10): step()
    e1.record(st); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    b = S * T * (N * 4 + N // 2 * 4)
    print(f"  N={N:5d}: {S*T/ms/1e3:8.2f} M frames/s  {ms*1e3:8.1f} us/launch  {b/ms/1e6:7.1f} GB/s  frac_of_measured_hbm {b/ms/1e6/PEAK:.3f}")

print("== rank 2: live tick latency (1 stereo source, N=4096): capture_audio + tick through the plugin's own code, per tick")
N = 4096
try:
    from oracle import refbind
    impls = [(refbind.IMPL_GENERIC, "WAVSourceGeneric (reference, 1 core)"), (refbind.IMPL_AVX2, "WAVSourceAVX2    (reference, 1 core)")]
    if refbind.cuda_seam_available():
        impls.append((refbind.IMPL_CUDA, "WAVSourceCUDA    (this repo: host/source_cuda.hpp -> libwfstft.so, zero-copy pinned staging)"))
    for N in (4096, 2048):
        print(f"  -- N={N}")
        for impl, name in impls:
            r = refbind.RefSource({"fft_size": N, "channel_mode": "stereo"}, impl=impl, channels=2)
            pcm = synth_pcm(1, 2, 1001 * 800 + N)[0]
            r.run_stft(pcm, 200, 800, want_db=False)   # warm-up
            t0 = time.perf_counter(); r.run_stft(pcm[:, 200 * 800:], 800, 800, want_db=False); dt = time.perf_counter() - t0
            print(f"  {name}: {dt/800*1e6:.1f} us per tick")
except Exception as ex:
    print("  reference unavailable:", ex)
eng = Engine({"fft_size": 4096, "channel_mode": "stereo"}, channels=2, max_streams=1)
x = synth_pcm(1, 2, 4096)
lat = []
for i in range(300):
    t0 = time.perf_counter(); eng.process(x, 1, 4096); lat.append(time.perf_counter() - t0)
lat = np.array(lat[50:]) * 1e6
print(f"  (python Engine.process, pageable numpy buffers, staged copies: median {np.median(lat):.1f} us  p95 {np.percentile(lat,95):.1f} us)")

# where a live tick's time goes: the C call alone (no plugin plumbing), zero-copy pinned buffers from wf_host_alloc
import ctypes as C
for (N, ch, mode) in ((4096, 2, "stereo"), (2048, 1, "mono")):
    e = Engine({"fft_size": N, "channel_mode": mode}, channels=ch, max_streams=1)
    L = e.L
    cc, dch, B = e.capture_channels, e.display_channels, e.bins
    pin = L.wf_host_alloc(cc * N * 4); pout = L.wf_host_alloc(dch * B * 4); pfl = L.wf_host_alloc(16)
    src = synth_pcm(1, cc, N)[0].ravel()
    C.memmove(pin, src.ctypes.data, src.nbytes)
    wall, kern = [], []
    for i in range(400):
        t0 = time.perf_counter()
        e.process_raw(pin, 1, 1, N, cc * N, N, out_db=pout, out_silent=pfl + 1, skip_mask=pfl)
        wall.append(time.perf_counter() - t0)
        if i % 8 == 0:
            kern.append(e.last_kernel_ms() * 1e3)
    wall = np.array(wall[50:]) * 1e6
    print(f"  wf_process alone, zero-copy, N={N} {mode}: wall median {np.median(wall):.1f} us p95 {np.percentile(wall,95):.1f} us; "
          f"kernel (events) median {np.median(kern):.1f} us; {e.last_kernel_name()}")
    L.wf_host_free(pin); L.wf_host_free(pout); L.wf_host_free(pfl)
