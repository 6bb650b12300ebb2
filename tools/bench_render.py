"""Kernel time of wf_render (the display stage on caller-held dB rows) next to wf_peak_normalize alone.

Two config-5 shapes, device-resident buffers, dB rows made once by a spectrum call of the same engine:
    n16384   1024 streams x 16 ticks, N=16384, 800-point Lanczos curve
    n2048    4096 streams x 16 ticks, N=2048, 26 Catmull-Rom bars (bar_width 24, gap 6)
Variants, timed in alternation on one engine per shape (CUDA events around the launch, wf_last_kernel_ms):
    normalize        wf_peak_normalize on the dB rows (read + write every bin)
    render           wf_render, points + pixels + min, no peak
    render+peak      the same with the peak gain applied in registers
    render+peak+wb   ... and the normalised rows written back (write_db)
It prints one JSON line per (shape, variant): median / min / max kernel time and the bytes the variant has to move (dB rows
read, rows written back, outputs written) over the median time, also as a share of the H100 SXM's 3.35 TB/s.  The card's
name and power limit are read in the same process.

    python tools/bench_render.py [--repeats 30] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from helpers import device_pcm  # noqa: E402
from waveform_b200 import Engine  # noqa: E402

HBM_BPS = 3.35e12

SHAPES = {
    "n16384": ({"fft_size": 16384, "interp_mode": "lanczos", "width": 800}, 1024, 16),
    "n2048": ({"fft_size": 2048, "display_mode": "bars", "interp_mode": "catmull_rom", "bar_width": 24, "bar_gap": 6,
               "width": 800}, 4096, 16),
}


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
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="n16384,n2048")
    a = ap.parse_args()
    name, power = card()
    for shape in a.shapes.split(","):
        settings, S, T = SHAPES[shape]
        N = settings["fft_size"]
        eng = Engine(settings, channels=1, max_streams=S)
        pcm = device_pcm(S, 1, (T - 1) * N + N, zero_every=7, frame_len=N)
        out = eng.process(pcm, T, N, want_peak=True)
        del pcm
        db, peak = out["db"], out["peak"]
        work = db.clone()
        torch.cuda.synchronize()
        dch, B, P = eng.display_channels, eng.bins, eng.num_points
        rows = S * T
        row_bytes = rows * dch * B * 4
        out_bytes = rows * dch * P * 4 * 2 + rows * 8      # points + pixels + (miny, minpos)
        variants = {
            "normalize": (lambda: eng.peak_normalize(work, peak, -3.0, 30.0), 2 * row_bytes),
            "render": (lambda: eng.render(db, want_points=True, want_pixels=True), row_bytes + out_bytes),
            "render+peak": (lambda: eng.render(db, peak, -3.0, 30.0, want_points=True, want_pixels=True),
                            row_bytes + out_bytes),
            "render+peak+wb": (lambda: eng.render(work, peak, -3.0, 30.0, write_db=True, want_points=True,
                                                  want_pixels=True), 2 * row_bytes + out_bytes),
        }
        times = {k: [] for k in variants}
        kernels = {}
        for r in range(a.warmup + a.repeats):
            for k, (fn, _) in variants.items():
                fn()
                ms = eng.last_kernel_ms()
                kernels[k] = eng.last_kernel_name() if k != "normalize" else "peak_normalize_kernel"
                if r >= a.warmup:
                    times[k].append(ms)
        torch.cuda.synchronize()
        for k, (_, nbytes) in variants.items():
            t = np.array(times[k])
            med = float(np.median(t))
            print(json.dumps({"shape": shape, "variant": k, "streams": S, "ticks": T, "fft_size": N, "points": P,
                              "kernel": kernels[k], "kernel_ms_median": round(med, 4), "kernel_ms_min": round(float(t.min()), 4),
                              "kernel_ms_max": round(float(t.max()), 4), "bytes": nbytes,
                              "GBps": round(nbytes / med / 1e6, 1), "share_of_3.35TBps": round(nbytes / med / 1e-3 / HBM_BPS, 3),
                              "gpu": name, "power_limit": power}), flush=True)
        del out, db, peak, work, eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
