"""Kernel time of the waveform engine with and without its display stage (render_curve on the GPU).

At the plugin defaults (800 points, 150 ms, a packet of 800 samples per tick, Catmull-Rom, no Gaussian) and device-resident
buffers, three calls are timed in alternation on one engine per channel layout:
    out      the scrolling dB rows only (what the engine computed before it had a display stage)
    out+px   the rows and the pixel rows + (miny, minpos)
    px       the pixel rows + (miny, minpos) only (out = NULL)
It prints one JSON line per (layout, variant): median / min / max kernel time over the repeats (CUDA events around the
kernel, wf_wave_last_kernel_ms) and the algorithmic bandwidth: PCM of the call in, the requested outputs out.  The card's
name and power limit are read in the same process.

    python tools/bench_wave_display.py [--streams 4096] [--ticks 32] [--repeats 20]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from waveform_b200 import WaveEngine  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (v.strip() for v in q.split(","))
        return name, power
    except Exception:  # no nvidia-smi: the name from torch, power unknown
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--ticks", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    S, T, hop, width = a.streams, a.ticks, 800, 800
    name, power = card()
    variants = {"out": dict(want_db=True, want_pixels=False), "out+px": dict(want_db=True, want_pixels=True),
                "px": dict(want_db=False, want_pixels=True)}
    for layout in ("mono", "stereo"):
        eng = WaveEngine({"width": width, "meter_buf": 150, "channel_mode": layout}, channels=2, max_streams=S)
        dch = eng.display_channels
        pcm = torch.from_numpy(np.random.default_rng(1).uniform(-0.5, 0.5, size=(S, 2, T * hop)).astype(np.float32)).cuda()
        times = {k: [] for k in variants}
        for r in range(a.warmup + a.repeats):
            for k, kw in variants.items():
                eng.process(pcm, T, hop, **kw)
                ms = eng.last_kernel_ms()
                if r >= a.warmup:
                    times[k].append(ms)
        row = S * T * dch * width * 4
        for k, kw in variants.items():
            t = np.array(times[k])
            nbytes = S * 2 * T * hop * 4 + (row if kw["want_db"] else 0) + ((row + S * T * 8) if kw["want_pixels"] else 0)
            med = float(np.median(t))
            print(json.dumps({"layout": layout, "variant": k, "streams": S, "ticks": T, "width": width, "hop": hop,
                              "kernel_ms_median": round(med, 4), "kernel_ms_min": round(float(t.min()), 4),
                              "kernel_ms_max": round(float(t.max()), 4), "algorithmic_GBps": round(nbytes / med / 1e6, 1),
                              "vs_out": round(med / float(np.median(times["out"])), 3), "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
