"""float32 vs int16 PCM input (pcm_format) on the level meter, the RMS feed and the waveform, timed in alternation in one
process.

Shapes (those of tools/bench_meter.py; 64 ticks of 800 samples per call):
    meter_rms     RMS meter, 150 ms window, stereo, 4096 streams (one-pass kernel)
    meter_peak    peak meter, 100 ms window, mono, 8192 streams
    feed          the RMS feed (1 s window), stereo, 4096 streams
    wave_mix      waveform, 800 points over 150 ms, two channels mixed to one, 4096 streams
    wave_stereo   waveform, 800 points over 150 ms, stereo, 4096 streams
    meter_pin     meter_rms with the PCM in pinned host memory, end to end (H2D of the PCM, kernels, D2H of the outputs
                  into numpy arrays; host clock around the blocking call)
For each shape and format: median / min / max over the rounds of the kernel time (CUDA events around the kernel section,
*_last_kernel_ms), ticks/s, and the algorithmic bytes over the median time (meter: 4 or 2 B per sample in, outputs
negligible; waveform: the same plus width * 4 B per display channel and tick out).  The two formats' outputs are compared
bit for bit at the timed size.  The card's name, power limit and maximum SM clock are read in the same process.

    python tools/bench_meter_wave_s16.py [--rounds 9] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from waveform_b200 import MeterEngine, WaveEngine  # noqa: E402
from waveform_b200.engine import METER_INPUT_RMS  # noqa: E402

T, HOP = 64, 800
# name: (kind, settings, channels, streams, meter mode, pinned host)
SHAPES = {
    "meter_rms": ("meter", {"meter_buf": 150, "rms_mode": True}, 2, 4096, None, False),
    "meter_peak": ("meter", {"meter_buf": 100, "rms_mode": False}, 1, 8192, None, False),
    "feed": ("meter", {}, 2, 4096, METER_INPUT_RMS, False),
    "wave_mix": ("wave", {"width": 800, "meter_buf": 150}, 2, 4096, None, False),
    "wave_stereo": ("wave", {"width": 800, "meter_buf": 150, "channel_mode": "stereo"}, 2, 4096, None, False),
    "meter_pin": ("meter", {"meter_buf": 150, "rms_mode": True}, 2, 4096, None, True),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [v.strip() for v in q.split(",")]
    except Exception:  # no nvidia-smi: the name from torch, the rest unknown
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def _host(v):
    return v.cpu().numpy() if hasattr(v, "cpu") else v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    name, power, sm_clock = card()
    print(json.dumps({"gpu": name, "power_limit": power, "max_sm_clock": sm_clock}), flush=True)
    for key in a.shapes.split(","):
        kind, settings, cc, S, mode, pinned = SHAPES[key]
        g = torch.Generator().manual_seed(S + cc)
        x16 = torch.randint(-16384, 16384, (S, cc, T * HOP), dtype=torch.int16, generator=g)
        x32 = x16.to(torch.float32) * 2.0 ** -15
        if kind == "meter":
            engines = {f: MeterEngine(settings, channels=cc, max_streams=S, device=0, mode=mode) for f in ("f32", "s16")}
        else:
            engines = {f: WaveEngine(settings, channels=cc, max_streams=S, device=0) for f in ("f32", "s16")}
        if pinned:  # numpy views of page-locked memory: the host path, staged through the engine's device buffers
            pcm = {"f32": x32.pin_memory().numpy(), "s16": x16.pin_memory().numpy()}
        else:
            pcm = {"f32": x32.cuda(), "s16": x16.cuda()}
        times = {f: [] for f in pcm}
        outs = {}
        for r in range(a.warmup + a.rounds):
            for f in ("f32", "s16"):
                e = engines[f]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[f] = e.process(pcm[f], T, HOP, pcm_format=f)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                if r >= a.warmup:
                    times[f].append(wall if pinned else e.last_kernel_ms())
        same = all(np.array_equal(_host(outs["f32"][k]).view(np.uint8), _host(outs["s16"][k]).view(np.uint8)) for k in outs["f32"])
        for f in ("f32", "s16"):
            t = np.array(times[f])
            med = float(np.median(t))
            nbytes = S * cc * T * HOP * (2 if f == "s16" else 4)
            if kind == "wave":
                nbytes += S * T * engines[f].display_channels * engines[f].cfg.width * 4
            print(json.dumps({"shape": key, "format": f, "streams": S, "channels": cc, "ticks": T, "hop": HOP,
                              "pinned_host_end_to_end": pinned, "median_ms": round(med, 4),
                              "min_ms": round(float(t.min()), 4), "max_ms": round(float(t.max()), 4),
                              "ticks_per_s": round(S * T / (med * 1e-3)),
                              "algorithmic_GB_per_s": round(nbytes / (med * 1e-3) / 1e9, 1),
                              "bit_equal_outputs": bool(same)}), flush=True)


if __name__ == "__main__":
    main()
