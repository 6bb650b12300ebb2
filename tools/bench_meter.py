#!/usr/bin/env python
"""Device-resident throughput of the level meter / RMS feed (wf_meter_*) and of the waveform mode (wf_wave_*): ticks/s and
fraction of the HBM roofline (algorithmic bytes: meter = 4 B per sample in, outputs negligible; waveform = 4 B per sample in
+ width*4 B per display channel and tick out)."""
import json, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch
from waveform_b200 import MeterEngine, WaveEngine
from waveform_b200.engine import METER_INPUT_RMS

PEAK = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0
for name, settings, ch, S, T, hop, mode in [
        ("meter RMS 150 ms stereo", {"meter_buf": 150, "rms_mode": True}, 2, 4096, 64, 800, None),
        ("meter peak 100 ms mono", {"meter_buf": 100, "rms_mode": False}, 1, 8192, 64, 800, None),
        ("RMS feed (1 s window) stereo", {}, 2, 4096, 64, 800, METER_INPUT_RMS)]:
    eng = MeterEngine(settings, channels=ch, max_streams=S, mode=mode)
    pcm = (torch.rand((S, ch, T * hop), device="cuda") - 0.5) * 0.5
    st = torch.cuda.Stream()
    for _ in range(3):
        eng.process(pcm, T, hop, stream=st.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    K = 10
    e0.record(st)
    for _ in range(K):
        eng.process(pcm, T, hop, stream=st.cuda_stream)
    e1.record(st); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    nbytes = S * ch * T * hop * 4
    print(f"{name:32s} {S*T/ms/1e3:8.2f} M ticks/s  {ms*1e3:8.1f} us/call  {nbytes/ms/1e6:7.1f} GB/s  frac {nbytes/ms/1e6/PEAK:.3f}  window {eng.window}")

for name, settings, ch, S, T, hop in [("waveform 800 pts / 150 ms, 2ch mixed", {"width": 800, "meter_buf": 150}, 2, 4096, 64, 800),
                                      ("waveform 800 pts stereo", {"width": 800, "meter_buf": 150, "channel_mode": "stereo"}, 2, 4096, 64, 800)]:
    eng = WaveEngine(settings, channels=ch, max_streams=S)
    pcm = (torch.rand((S, ch, T * hop), device="cuda") - 0.5) * 0.5
    st = torch.cuda.Stream()
    for _ in range(3):
        eng.process(pcm, T, hop, stream=st.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    K = 10
    e0.record(st)
    for _ in range(K):
        eng.process(pcm, T, hop, stream=st.cuda_stream)
    e1.record(st); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    nbytes = S * T * (ch * hop * 4 + eng.display_channels * eng.cfg.width * 4)
    kms = eng.last_kernel_ms()
    print(f"{name:36s} {S*T/ms/1e3:8.2f} M ticks/s  {ms*1e3:8.1f} us/call  {nbytes/ms/1e6:7.1f} GB/s  frac {nbytes/ms/1e6/PEAK:.3f}"
          f"  (kernel alone {kms*1e3:.1f} us, frac {nbytes/kms/1e6/PEAK:.3f})")
