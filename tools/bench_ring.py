"""Capture-ring calls (wf_batch.capture_ring) against the two ways a caller streams overlapped frames without them.

Cases, per shape (16 ticks per call, mono), timed with CUDA events around each call after warm-up, alternating:
    ring    the call hands over only the new samples (n_frames*hop per stream); splice + spectrum kernel
    copy    plain calls, the caller building the overlapped buffer (last N - hop samples ++ new) by device copies first
    floor   plain calls on a buffer that already holds the overlap (what the spectrum kernel alone costs)
Shapes: config 4 as a stream (256 streams, N=8192, hop 2048) and N=2048 hop 800 with 4096 streams, in float32 and
int16.  A torch.profiler pass splits the ring call into splice and spectrum kernel time.  `--pinned` adds config 4 end to
end from pinned host buffers (ring: n_frames*hop samples cross PCIe per stream; plain: (n_frames-1)*hop + N), timed with
a host clock around the blocking call.  `--old-lib PATH` adds the plain headline call (4096 x 16, N=2048, hop = N, device
buffers) on another build of libwfstft.so and this one, alternating in one process.  The splice's bytes per call are
computed from the shapes.  The card's name and power limit are read in the same process.

    python tools/bench_ring.py [--rounds 20] [--warmup 3] [--pinned] [--old-lib PATH]
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
import waveform_b200.engine as wfe  # noqa: E402
from waveform_b200 import Engine  # noqa: E402

T = 16
SHAPES = {"c4": (8192, 2048, 256), "n2048h800": (2048, 800, 4096)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [v.strip() for v in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown"]


def splice_bytes(N, hop, S, es):
    """Bytes the splice moves per call: with hop < N the ring (float) read N - hop and written N, the window written
    (T-1)*hop + N and its last N read back, the new samples read T*hop; with hop >= N the ring written N from the last N
    new samples."""
    if hop >= N:
        return S * (N * es + N * 4)
    per = (N - hop) * 4 + N * 4 + ((T - 1) * hop + N) * es + N * es + T * hop * es
    return S * per


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def run_shape(key, fmt, rounds, warmup):
    N, hop, S = SHAPES[key]
    dt = torch.int16 if fmt == "s16" else torch.float32
    es = 2 if fmt == "s16" else 4
    g = torch.Generator(device="cuda").manual_seed(N + hop)
    total = (rounds + warmup) * T * hop
    src = torch.randint(-32768, 32768, (S, 1, N + total), dtype=torch.int16, generator=g, device="cuda")
    if fmt == "f32":
        src = src.to(torch.float32) * 2.0 ** -15
    src[:, :, :N] = 0
    st = torch.cuda.current_stream().cuda_stream
    settings = {"fft_size": N}
    eng = {c: Engine(settings, channels=1, max_streams=S, device=0) for c in ("ring", "copy", "floor")}
    B = eng["ring"].bins
    out = {c: torch.empty((S, T, 1, B), device="cuda") for c in eng}
    span = (T - 1) * hop + N
    hist = torch.zeros((S, 1, span), dtype=dt, device="cuda")
    new = torch.empty((S, 1, T * hop), dtype=dt, device="cuda")
    times = {c: [] for c in eng}
    pos = 0
    for r in range(warmup + rounds):
        new.copy_(src[:, :, N + pos: N + pos + T * hop])
        floor = src[:, :, pos + hop: pos + hop + span].contiguous()
        torch.cuda.synchronize()

        def ring():
            eng["ring"].process_raw(new.data_ptr(), S, T, hop, T * hop, T * hop, out_db=out["ring"].data_ptr(),
                                    pcm_format=fmt, capture_ring=True, stream=st, sync=False)

        def copy():  # the caller's own overlap: keep the last N - hop samples, append the new ones
            hist[:, :, : N - hop].copy_(hist[:, :, span - (N - hop):])  # disjoint: T * hop >= N
            hist[:, :, N - hop:].copy_(new)
            eng["copy"].process_raw(hist.data_ptr(), S, T, hop, span, span, out_db=out["copy"].data_ptr(), pcm_format=fmt,
                                    stream=st, sync=False)

        def floor_call():
            eng["floor"].process_raw(floor.data_ptr(), S, T, hop, span, span, out_db=out["floor"].data_ptr(),
                                     pcm_format=fmt, stream=st, sync=False)

        for c, fn in (("ring", ring), ("copy", copy), ("floor", floor_call)):
            ms = timed(fn)
            if r >= warmup:
                times[c].append(ms)
        pos += T * hop
    same = all(torch.equal(out[c].view(torch.int32), out["floor"].view(torch.int32)) for c in ("ring", "copy"))

    # kernel split of the ring call (a separate, profiled pass)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            eng["ring"].process_raw(new.data_ptr(), S, T, hop, T * hop, T * hop, out_db=out["ring"].data_ptr(),
                                    pcm_format=fmt, capture_ring=True, stream=st, sync=False)
        torch.cuda.synchronize()
    splice_us = kern_us = 0.0
    for ev in prof.key_averages():
        t_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if "ring_splice_kernel" in ev.key:
            splice_us += t_us / 5
        elif "stft" in ev.key:
            kern_us += t_us / 5
    sb = splice_bytes(N, hop, S, es)
    res = {"shape": key, "format": fmt, "N": N, "hop": hop, "streams": S, "ticks": T,
           "kernel": eng["ring"].last_kernel_name(), "bit_equal_outputs": same,
           "splice_bytes_per_call": sb, "new_bytes_per_call": S * T * hop * es,
           "profiled_splice_ms": round(splice_us / 1e3, 4), "profiled_spectrum_kernel_ms": round(kern_us / 1e3, 4)}
    for c in times:
        t = np.array(times[c])
        res[f"{c}_median_ms"] = round(float(np.median(t)), 4)
        res[f"{c}_min_ms"] = round(float(t.min()), 4)
    print(json.dumps(res), flush=True)


def run_pinned(rounds, warmup):
    N, hop, S = SHAPES["c4"]
    span = (T - 1) * hop + N
    g = torch.Generator().manual_seed(1)
    x = torch.randn((S, 1, span), generator=g) * 0.1
    plain_in = x.pin_memory()
    ring_in = x[:, :, : T * hop].contiguous().pin_memory()
    outs = {c: torch.empty((S, T, 1, N // 2)).pin_memory() for c in ("ring", "plain")}
    eng = {c: Engine({"fft_size": N}, channels=1, max_streams=S, device=0) for c in outs}
    times = {c: [] for c in outs}
    for r in range(warmup + rounds):
        for c in ("ring", "plain"):
            t0 = time.perf_counter()
            if c == "ring":
                eng[c].process_raw(ring_in.data_ptr(), S, T, hop, T * hop, T * hop, out_db=outs[c].data_ptr(),
                                   capture_ring=True)
            else:
                eng[c].process_raw(plain_in.data_ptr(), S, T, hop, span, span, out_db=outs[c].data_ptr())
            if r >= warmup:
                times[c].append((time.perf_counter() - t0) * 1e3)
    res = {"shape": "c4_pinned_host", "N": N, "hop": hop, "streams": S, "ticks": T,
           "ring_pcm_bytes": S * T * hop * 4, "plain_pcm_bytes": S * span * 4}
    for c in times:
        res[f"{c}_median_ms"] = round(float(np.median(times[c])), 4)
        res[f"{c}_min_ms"] = round(float(np.min(times[c])), 4)
    print(json.dumps(res), flush=True)


def run_headline(old_lib, rounds, warmup):
    """The plain headline call on another build of libwfstft.so and on this one, alternating in one process.  The other
    build is driven through its own C entry points (wf_create / wf_process / wf_last_kernel_ms), which every build has."""
    import ctypes as C

    N, S = 2048, 4096
    cfg = wfe.make_config({"fft_size": N}, 48000, 1, S, 0)
    old = C.CDLL(str(old_lib))
    old.wf_create.argtypes = [C.POINTER(wfe.WfConfig), C.POINTER(C.c_void_p)]
    old.wf_process.argtypes = [C.c_void_p, C.POINTER(wfe.WfBatch)]
    old.wf_last_kernel_ms.argtypes = [C.c_void_p]
    old.wf_last_kernel_ms.restype = C.c_float
    old.wf_destroy.argtypes = [C.c_void_p]
    h = C.c_void_p()
    assert old.wf_create(C.byref(cfg), C.byref(h)) == 0, "wf_create of the other build failed"
    new = Engine(config=cfg)
    x = (torch.randn((S, 1, T * N), generator=torch.Generator().manual_seed(2)) * 0.1).cuda()
    outs = {c: torch.empty((S, T, 1, N // 2), device="cuda") for c in ("old", "new")}
    b = wfe.WfBatch()
    b.struct_size = C.sizeof(wfe.WfBatch)
    b.n_streams, b.n_frames, b.hop, b.seconds = S, T, N, 1.0 / 60.0
    b.pcm, b.stream_stride, b.channel_stride, b.out_db = x.data_ptr(), T * N, T * N, outs["old"].data_ptr()

    def call(c):
        if c == "old":
            assert old.wf_process(h, C.byref(b)) == 0
            return float(old.wf_last_kernel_ms(h))
        new.process_raw(x.data_ptr(), S, T, N, T * N, T * N, out_db=outs["new"].data_ptr())
        return new.last_kernel_ms()

    times = {c: [] for c in outs}
    for r in range(warmup + rounds):
        for c in ("old", "new") if r % 2 == 0 else ("new", "old"):
            ms = call(c)
            if r >= warmup:
                times[c].append(ms)
    old.wf_destroy(h)
    res = {"shape": "headline_old_vs_new", "N": N, "streams": S, "ticks": T, "kernel": new.last_kernel_name(),
           "bit_equal_outputs": bool(torch.equal(outs["old"].view(torch.int32), outs["new"].view(torch.int32)))}
    for c in times:
        res[f"{c}_median_ms"] = round(float(np.median(times[c])), 4)
        res[f"{c}_min_ms"] = round(float(np.min(times[c])), 4)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pinned", action="store_true")
    ap.add_argument("--old-lib", default=None)
    a = ap.parse_args()
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    for key in SHAPES:
        for fmt in ("f32", "s16"):
            run_shape(key, fmt, a.rounds, a.warmup)
    if a.pinned:
        run_pinned(max(5, a.rounds // 2), a.warmup)
    if a.old_lib:
        run_headline(a.old_lib, 4 * a.rounds, a.warmup)


if __name__ == "__main__":
    main()
