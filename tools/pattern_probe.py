#!/usr/bin/env python
"""Bandwidth ceiling of the headline workload's access pattern (4096 streams x 16 frames of N=2048: 512 MiB read,
256 MiB written per step), measured without the FFT.  One JSON line per variant; see tools/pattern_probe.cu.

    python tools/pattern_probe.py [--iters 50] [--spin 0,8000] [--warps 16,12,10]

GB/s counts the algorithmic 12 288 B/frame (8 KiB in, 4 KiB out), as bench.py's roofline does; gbs_incl_state adds the
4 KiB read + 4 KiB written of EMA state per stream that the stream variants move as well.  The library is compiled
into a temporary directory with the flags of waveform_b200/csrc/Makefile."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
NVCC = "/usr/local/cuda/bin/nvcc"
S, T, N, B = 4096, 16, 2048, 1024


def card():
    """Name, power limit and maximum SM clock of GPU 0, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, pl, clk = [x.strip() for x in r.stdout.strip().split(",")]
        return {"gpu": name, "power_limit_w": float(pl), "sm_clock_max_mhz": int(clk)}
    except Exception as ex:  # the numbers stay usable; the card is then named by torch alone
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_max_mhz": None, "query_error": str(ex)}


def build(tmp):
    so = Path(tmp) / "libpattern_probe.so"
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++20", "-O3", "-Xcompiler", "-fPIC,-ffp-contract=off",
                    "-shared", "-o", str(so), str(HERE / "pattern_probe.cu")], check=True)
    lib = C.CDLL(str(so))
    lib.probe_copy.restype = C.c_float
    lib.probe_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.probe_stream.restype = C.c_float
    lib.probe_stream.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 7
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--spin", default="0", help="comma-separated busy-wait cycles per frame standing in for the arithmetic")
    ap.add_argument("--warps", default="16,12,10", help="warps per CTA of variant (c); (b) runs at the first")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("pattern_probe.py needs a CUDA device")
    info = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pcm = torch.rand((S * T * N,), device="cuda")
    out = torch.empty((S * T * B,), device="cuda")
    state = torch.zeros((S * B,), device="cuda")
    frame_bytes = S * T * (N + B) * 4
    state_bytes = S * 2 * B * 4
    warps = [int(w) for w in args.warps.split(",")]
    with tempfile.TemporaryDirectory() as tmp:
        lib = build(tmp)

        def emit(variant, ms, **kw):
            if ms <= 0:
                raise SystemExit(f"{variant}: CUDA error")
            line = {"probe": variant, "shape": f"{S}x{T} N={N}", "ms": ms, "gbs": frame_bytes / (ms * 1e-3) / 1e9, **kw, **info}
            if variant != "a_copy":
                line["gbs_incl_state"] = (frame_bytes + state_bytes) / (ms * 1e-3) / 1e9
            print(json.dumps(line), flush=True)

        ms = lib.probe_copy(pcm.data_ptr(), out.data_ptr(), out.numel(), sms * 4, 512, args.warmup, args.iters)
        emit("a_copy", ms, blocks=sms * 4, threads=512)
        for spin in [int(x) for x in args.spin.split(",")]:
            ms = lib.probe_stream(0, pcm.data_ptr(), out.data_ptr(), state.data_ptr(), S, T, sms, warps[0], spin, args.warmup, args.iters)
            emit("b_half_lead_scalar_stores", ms, warps=warps[0], spin_cycles=spin)
            for w in warps:
                ms = lib.probe_stream(1, pcm.data_ptr(), out.data_ptr(), state.data_ptr(), S, T, sms, w, spin, args.warmup, args.iters)
                emit("c_full_lead_bulk_stores", ms, warps=w, spin_cycles=spin)
    torch.cuda.synchronize()
    return 0


if __name__ == "__main__":
    sys.exit(main())
