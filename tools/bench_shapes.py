#!/usr/bin/env python
"""Device-resident throughput of the BASELINE.json configs other than the headline and of the other kernel families.
Prints frames/s and the fraction of the measured HBM roofline using SURVEY §8(d) nominal bytes
(hop*4 per channel in + written floats out per frame).  bench.py imports run_shapes() for its config.extra.other_shapes."""
import json, os, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = [
    ("c2 stereo N=4096 BH, hop 800 (60 fps)", {"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2, 2048, 16, 800, "db"),
    ("c4 N=8192 hop 2048, 800-pt Lanczos curve", {"fft_size": 8192, "window": "hann", "interp_mode": "lanczos"}, 1, 256, 256, 2048, "points"),
    ("c4' N=8192 hop 2048, bins out", {"fft_size": 8192, "window": "hann"}, 1, 256, 256, 2048, "db"),
    ("c5 N=16384 hop N, peak", {"fft_size": 16384, "window": "hann"}, 1, 128, 64, 16384, "db+peak"),
    ("c5 full N=16384 128x256", {"fft_size": 16384, "window": "hann"}, 1, 128, 256, 16384, "db+peak"),
    ("N=4096 mono 4096x16 hop N", {"fft_size": 4096, "window": "hann"}, 1, 4096, 16, 4096, "db"),
    ("N=8192 mono 2048x16 hop N", {"fft_size": 8192, "window": "hann"}, 1, 2048, 16, 8192, "db"),
    ("c1 N=1024 bars catrom", {"fft_size": 1024, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 1, 4096, 16, 1024, "points"),
    ("N=2048 generic (WF_FORCE_GENERIC)", {"fft_size": 2048, "window": "hann"}, 1, 4096, 16, 2048, "db"),
    ("N=800 (auto size 48k/60fps) 4096x16", {"fft_size": 800, "window": "hann"}, 1, 4096, 16, 800, "db"),
    ("N=1920 4096x16", {"fft_size": 1920, "window": "hann"}, 1, 4096, 16, 1920, "db"),
    ("N=1600 4096x16", {"fft_size": 1600, "window": "hann"}, 1, 4096, 16, 1600, "db"),
    # display outputs of one-channel sources (render-time stages fused; WF_WARP2_DISPLAY=0 puts them back on the CTA-per-tick /
    # any-N kernels)
    ("disp N=800 Catmull-Rom curve, points out", {"fft_size": 800, "window": "hann", "interp_mode": "catmull_rom"}, 1, 4096, 16, 800, "points"),
    ("disp N=2048 Lanczos curve, points out", {"fft_size": 2048, "window": "hann", "interp_mode": "lanczos"}, 1, 4096, 16, 2048, "points"),
    ("disp N=2048 Lanczos curve, bins + points", {"fft_size": 2048, "window": "hann", "interp_mode": "lanczos"}, 1, 4096, 16, 2048, "db+points"),
]


def run_shapes(torch, only=None, iters=10, peak_gbs=None):
    from waveform_b200 import Engine

    if peak_gbs is None:
        pk = ROOT / "MEASURED_PEAKS.json"
        peak_gbs = json.loads(pk.read_text())["hbm_gbs"] if pk.exists() else 3350.0
    res = []
    for name, settings, ch, S, T, hop, mode in SHAPES:
        if only and not any(o in name for o in only):
            continue
        if "FORCE_GENERIC" in name:
            os.environ["WF_FORCE_GENERIC"] = "1"
        eng = Engine(settings, channels=ch, max_streams=S)
        os.environ.pop("WF_FORCE_GENERIC", None)
        N, cc, dch, B, P = eng.fft_size, eng.capture_channels, eng.display_channels, eng.bins, eng.num_points
        ns = (T - 1) * hop + N
        pcm = (torch.rand((S, cc, ns), device="cuda") - 0.5) * 0.5
        out_db = torch.empty((S, T, dch, B), device="cuda") if "db" in mode else None
        out_pts = torch.empty((S, T, dch, P), device="cuda") if "points" in mode else None
        peak = torch.empty((T,), device="cuda") if "peak" in mode else None
        st = torch.cuda.Stream()

        def step():
            eng.process_raw(pcm.data_ptr(), S, T, hop, cc * ns, ns, out_db=None if out_db is None else out_db.data_ptr(),
                            out_points=None if out_pts is None else out_pts.data_ptr(),
                            out_peak=None if peak is None else peak.data_ptr(), stream=st.cuda_stream, sync=False)
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(iters):
            step()
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        frames = S * T
        out_floats = (dch * B if out_db is not None else 0) + (dch * P if out_pts is not None else 0)
        bytes_per_frame = min(hop, N) * 4 * cc + out_floats * 4
        gbs = frames * bytes_per_frame / (ms * 1e-3) / 1e9
        res.append({"shape": name, "streams": S, "frames": T, "hop": hop, "value": frames / (ms * 1e-3), "unit": "frames/s",
                    "us_per_launch": ms * 1e3, "bytes_per_frame": bytes_per_frame, "gbs": gbs, "frac": gbs / peak_gbs,
                    "kernel": eng.last_kernel_name()})
        del eng, pcm, out_db, out_pts
    return res


if __name__ == "__main__":
    import torch
    ONLY = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--only=")]
    ITERS = int(([a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--iters=")] or ["10"])[0])
    print("env:", {k: v for k, v in os.environ.items() if k.startswith("WF_")})
    for r in run_shapes(torch, ONLY or None, ITERS):
        print(f"{r['shape']:45s} {r['value']/1e6:9.2f} M frames/s  {r['us_per_launch']:9.1f} us/launch  {r['bytes_per_frame']:6d} B/frame  "
              f"{r['gbs']:7.1f} GB/s  frac {r['frac']:.3f}  {r['kernel']}")
