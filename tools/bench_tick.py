"""Host-side cost of one live tick: two builds of libwfstft.so, alternating in one process.

A live source ticks one stream x one frame.  Here that is N=2048 mono with the spectrum output, in page-locked,
device-mapped buffers from wf_host_alloc, so the call runs zero-copy: one launch and one synchronisation, and its time
is mostly host work and launch latency rather than kernel time.  Each tick is timed with a host clock around the blocking
wf_process.  The two builds take turns in blocks of `--ticks` ticks, the order flipping every block, so that drift on a
shared host lands on both.  Both builds are driven through the same C entry points, each with its own engine and its own
wf_host_alloc buffers, on the same input; their dB rows must stay bit-identical.  Printed: the card's name and power
limit, then one JSON line with each build's median per-tick time over all ticks and the range of its per-block medians
(the spread to compare a difference against).

    python tools/bench_tick.py --old-lib PATH [--new-lib PATH] [--blocks 40] [--ticks 1000] [--warmup 500]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import waveform_b200.engine as wfe  # noqa: E402

N = 2048


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return [v.strip() for v in q.split(",")]


class Tick:
    """One engine of one build, with its live-tick buffers in wf_host_alloc memory."""

    def __init__(self, path, frame):
        L = self.L = C.CDLL(str(path))
        vp = C.c_void_p
        L.wf_create.argtypes = [C.POINTER(wfe.WfConfig), C.POINTER(vp)]
        L.wf_destroy.argtypes = [vp]
        L.wf_process.argtypes = [vp, C.POINTER(wfe.WfBatch)]
        L.wf_last_kernel_name.restype = C.c_char_p
        L.wf_last_kernel_name.argtypes = [vp]
        L.wf_host_alloc.restype = vp
        L.wf_host_alloc.argtypes = [C.c_size_t]
        L.wf_host_free.argtypes = [vp]
        self.h = vp()
        cfg = wfe.make_config({"fft_size": N}, 48000, 1, 1, 0)
        rc = L.wf_create(C.byref(cfg), C.byref(self.h))
        if rc != 0:
            raise RuntimeError(f"wf_create of {path} failed with status {rc} (this measurement needs a GPU)")
        self.pcm = L.wf_host_alloc(N * 4)
        self.out = L.wf_host_alloc(N // 2 * 4)
        if not self.pcm or not self.out:
            raise RuntimeError("wf_host_alloc failed")
        C.memmove(self.pcm, frame.ctypes.data, N * 4)
        b = self.b = wfe.WfBatch()
        b.struct_size = C.sizeof(wfe.WfBatch)
        b.n_streams, b.n_frames, b.hop, b.seconds = 1, 1, N, 1.0 / 60.0
        b.pcm, b.stream_stride, b.channel_stride, b.out_db = self.pcm, N, N, self.out

    def run(self, n, times=None):
        L, h, b = self.L, self.h, C.byref(self.b)
        for _ in range(n):
            t0 = time.perf_counter()
            rc = L.wf_process(h, b)
            t1 = time.perf_counter()
            if rc != 0:
                raise RuntimeError(f"wf_process failed with status {rc}")
            if times is not None:
                times.append((t1 - t0) * 1e6)

    def row(self):
        return np.ctypeslib.as_array((C.c_float * (N // 2)).from_address(self.out)).copy()

    def close(self):
        self.L.wf_host_free(self.pcm)
        self.L.wf_host_free(self.out)
        self.L.wf_destroy(self.h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old-lib", required=True)
    ap.add_argument("--new-lib", default=str(wfe.LIB_PATH))
    ap.add_argument("--blocks", type=int, default=40)
    ap.add_argument("--ticks", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=500)
    a = ap.parse_args()
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)

    t = np.arange(N) / 48000.0
    frame = (0.25 * np.sin(2 * np.pi * 997.0 * t) + 0.01 * np.random.default_rng(7).standard_normal(N)).astype(np.float32)
    libs = {"old": Tick(a.old_lib, frame), "new": Tick(a.new_lib, frame)}
    for lib in libs.values():
        lib.run(a.warmup)
    times = {c: [] for c in libs}
    block_medians = {c: [] for c in libs}
    for k in range(a.blocks):
        for c in ("old", "new") if k % 2 == 0 else ("new", "old"):
            block = []
            libs[c].run(a.ticks, block)
            times[c] += block
            block_medians[c].append(float(np.median(block)))
    same = np.array_equal(libs["old"].row().view(np.int32), libs["new"].row().view(np.int32))
    res = {"shape": "live_tick_N2048_1x1_host_alloc", "ticks_per_build": len(times["new"]),
           "kernel": libs["new"].L.wf_last_kernel_name(libs["new"].h).decode(), "bit_equal_outputs": bool(same)}
    for c in libs:
        res[f"{c}_median_us"] = round(float(np.median(times[c])), 2)
        res[f"{c}_block_median_range_us"] = [round(min(block_medians[c]), 2), round(max(block_medians[c]), 2)]
    print(json.dumps(res), flush=True)
    for lib in libs.values():
        lib.close()


if __name__ == "__main__":
    main()
