"""float32 vs int16 PCM input (wf_batch.pcm_format) on the same spectrum calls, timed in alternation in one process.

Shapes (mono unless noted, hop = N, 16 ticks):
    n2048      4096 streams, N=2048, device-resident (the headline: stft2048_fast_kernel)
    n800       4096 streams, N=800, device-resident (stft_warp2_kernel)
    n4096st    1024 streams, N=4096 stereo, device-resident (stft_v3_kernel)
    n2048pin   4096 streams, N=2048, pinned host buffers end to end (H2D of the PCM, kernel, D2H of the dB rows)
For each shape and format: median / min / max over the rounds of the kernel time (wf_last_kernel_ms: CUDA events around
the kernel section; for the pinned shape, the whole staged pipeline), spectra/s, and the algorithmic bytes (PCM read once +
dB rows written once) over the median time.  The two formats' outputs are compared bit for bit at the timed size.  The
card's name, power limit and maximum SM clock are read in the same process.

    python tools/bench_pcm_s16.py [--rounds 7] [--warmup 2]
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
from waveform_b200 import Engine  # noqa: E402

SHAPES = {
    "n2048": (2048, 1, False, 4096, False),
    "n800": (800, 1, False, 4096, False),
    "n4096st": (4096, 2, True, 1024, False),
    "n2048pin": (2048, 1, False, 4096, True),
}
T = 16


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [v.strip() for v in q.split(",")]
    except Exception:  # no nvidia-smi: the name from torch, the rest unknown
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    name, power, sm_clock = card()
    print(json.dumps({"gpu": name, "power_limit": power, "max_sm_clock": sm_clock}), flush=True)
    for key in a.shapes.split(","):
        N, cc, stereo, S, pinned = SHAPES[key]
        settings = {"fft_size": N, **({"channel_mode": "stereo"} if stereo else {})}
        ns = T * N
        g = torch.Generator().manual_seed(N)
        x16 = torch.randint(-32768, 32768, (S, cc, ns), dtype=torch.int16, generator=g)
        x32 = x16.to(torch.float32) * 2.0 ** -15
        engines = {f: Engine(settings, channels=cc, max_streams=S, device=0) for f in ("f32", "s16")}
        dch, B = engines["f32"].display_channels, engines["f32"].bins
        if pinned:
            pcm = {"f32": x32.pin_memory(), "s16": x16.pin_memory()}
            outs = {f: torch.empty((S, T, dch, B), dtype=torch.float32).pin_memory() for f in pcm}
        else:
            pcm = {"f32": x32.cuda(), "s16": x16.cuda()}
            outs = {f: torch.empty((S, T, dch, B), dtype=torch.float32, device="cuda") for f in pcm}
        times = {f: [] for f in pcm}
        for r in range(a.warmup + a.rounds):
            for f in ("f32", "s16"):
                e = engines[f]
                e.reset_state()
                e.process_raw(pcm[f].data_ptr(), S, T, N, cc * ns, ns, out_db=outs[f].data_ptr(), pcm_format=f)
                e.synchronize()
                if r >= a.warmup:
                    times[f].append(e.last_kernel_ms())
        same = bool(torch.equal(outs["f32"].view(torch.int32), outs["s16"].view(torch.int32)))
        for f in ("f32", "s16"):
            t = np.array(times[f])
            med = float(np.median(t))
            spectra = S * T * (2 if stereo else 1)
            nbytes = S * cc * ns * (2 if f == "s16" else 4) + S * T * dch * B * 4
            print(json.dumps({"shape": key, "format": f, "kernel": engines[f].last_kernel_name(), "N": N, "streams": S,
                              "ticks": T, "channels": cc, "pinned_host": pinned, "median_ms": round(med, 4),
                              "min_ms": round(float(t.min()), 4), "max_ms": round(float(t.max()), 4),
                              "spectra_per_s": round(S * T / (med * 1e-3)),
                              "channel_spectra_per_s": round(spectra / (med * 1e-3)),
                              "algorithmic_GB_per_s": round(nbytes / (med * 1e-3) / 1e9, 1),
                              "bit_equal_outputs": same}), flush=True)


if __name__ == "__main__":
    main()
