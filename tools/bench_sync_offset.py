"""The audio sync offset's cost: each engine with D = 0 against offsets of 200 ms and 1000 ms, timed in alternation.

Shapes (device buffers, float32, steady state: every start-up tick is behind, so no mask work):
    c4          spectrum ring calls, config 4 as a stream: 256 streams x 16 ticks, N=8192, hop 2048, mono
    n2048h800   spectrum ring calls, 4096 streams x 16 ticks, N=2048, hop 800, mono
    meter_rms   RMS meter, 150 ms window, stereo, 4096 streams x 64 ticks of 800 (tools/bench_meter_wave_s16.py)
    feed        the RMS feed (1 s window), stereo, 4096 streams x 64 ticks of 800
    wave_mix    waveform, width 800, 150 ms, two channels mixed, 4096 streams x 64 ticks of 800
For each shape and offset: median / min over the rounds of the engine's kernel time (CUDA events around the call's kernel
section, splice included).  The splice's bytes per call are computed from the shapes (splice_bytes): without an offset the
meter and the waveform run no splice at all.  `--old-lib PATH` adds the plain headline call (4096 x
16, N=2048, hop = N) on another build of libwfstft.so and this one, alternating in one process, with its outputs compared
bit for bit.  The card's name and power limit are read in the same process.

    python tools/bench_sync_offset.py [--rounds 30] [--warmup 3] [--old-lib PATH]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import waveform_b200.engine as wfe  # noqa: E402
from waveform_b200 import Engine, MeterEngine, WaveEngine  # noqa: E402
from waveform_b200.engine import METER_INPUT_RMS  # noqa: E402

OFFSETS = (0, 200, 1000)
SR = 48000
# name: (kind, settings, channels, streams, ticks, hop, meter mode)
SHAPES = {
    "c4": ("ring", {"fft_size": 8192}, 1, 256, 16, 2048, None),
    "n2048h800": ("ring", {"fft_size": 2048}, 1, 4096, 16, 800, None),
    "meter_rms": ("meter", {"meter_buf": 150, "rms_mode": True}, 2, 4096, 64, 800, None),
    "feed": ("meter", {}, 2, 4096, 64, 800, METER_INPUT_RMS),
    "wave_mix": ("wave", {"width": 800, "meter_buf": 150}, 2, 4096, 64, 800, None),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [v.strip() for v in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def splice_bytes(kind, N, D, hop, T, S, cc, es=4):
    """Bytes the history splice (wf_splice.hpp) moves per call: the window written and its history and new parts read,
    the history rewritten from the window (or the new samples past it)."""
    L = T * hop
    if kind == "ring":
        R, ws = N + D, hop
        wl = 0 if hop >= R else max((T - 1) * hop + N, R - hop)
    else:
        if D == 0:
            return 0
        R, ws = D, 0
        wl = max(L, D) if kind == "meter" else D + L
    hw = max(0, min(wl, R - ws)) if wl else 0
    win = wl * es + (wl - hw) * es + hw * 4
    hist = R * 4 + R * es
    return S * cc * (win + hist)


def make(kind, settings, cc, S, mode, ms):
    s = {**settings, "audio_sync_offset": ms}
    if kind == "ring":
        return Engine(s, channels=cc, max_streams=S, device=0)
    if kind == "meter":
        return MeterEngine(s, channels=cc, max_streams=S, device=0, mode=mode)
    return WaveEngine(s, channels=cc, max_streams=S, device=0)


def run_shape(name, rounds, warmup):
    kind, settings, cc, S, T, hop, mode = SHAPES[name]
    gen = torch.Generator().manual_seed(7)
    engines = {ms: make(kind, settings, cc, S, mode, ms) for ms in OFFSETS}
    x = (torch.randn((S, cc, T * hop), generator=gen) * 0.1).cuda()

    def call(ms):
        e = engines[ms]
        if kind == "ring":
            e.process(x, T, hop, capture_ring=True, want_silent=False)
        elif kind == "meter":
            e.process(x, T, hop)
        else:
            e.process(x, T, hop)
        torch.cuda.synchronize()
        return e.last_kernel_ms()

    for ms in OFFSETS:  # past every start-up tick (1000 ms = 48000 samples) before timing
        for _ in range(max(warmup, -(-_delay(1000) // (T * hop)) + 1)):
            call(ms)
    times = {ms: [] for ms in OFFSETS}
    for r in range(rounds):
        order = OFFSETS if r % 2 == 0 else OFFSETS[::-1]
        for ms in order:
            times[ms].append(call(ms))
    res = {"shape": name, "kind": kind, "streams": S, "ticks": T, "hop": hop, "channels": cc}
    for ms in OFFSETS:
        D = _delay(ms)
        res[f"D{D}_median_ms"] = round(float(np.median(times[ms])), 4)
        res[f"D{D}_min_ms"] = round(float(np.min(times[ms])), 4)
        res[f"D{D}_splice_MB"] = round(splice_bytes(kind, settings.get("fft_size", 0), D, hop, T, S, cc) / 1e6, 1)
    print(json.dumps(res), flush=True)


def _delay(ms):
    return SR * ms // 1000


def run_headline(old_lib, rounds, warmup):
    """The plain headline call on another build and on this one, alternating; the other build takes the config of its own
    (previous) size."""
    N, S, T = 2048, 4096, 16
    cfg = wfe.make_config({"fft_size": N}, 48000, 1, S, 0)
    old_cfg = wfe.WfConfig.from_buffer_copy(cfg)
    old_cfg.struct_size = wfe.WfConfig.sync_offset_ms.offset
    old = C.CDLL(str(old_lib))
    old.wf_create.argtypes = [C.POINTER(wfe.WfConfig), C.POINTER(C.c_void_p)]
    old.wf_process.argtypes = [C.c_void_p, C.POINTER(wfe.WfBatch)]
    old.wf_last_kernel_ms.argtypes = [C.c_void_p]
    old.wf_last_kernel_ms.restype = C.c_float
    old.wf_destroy.argtypes = [C.c_void_p]
    h = C.c_void_p()
    assert old.wf_create(C.byref(old_cfg), C.byref(h)) == 0, "wf_create of the other build failed"
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
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--old-lib", type=Path, default=None)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sync_offset.py needs a CUDA device: nothing is measured on the CPU")
    name, power, clock = card()
    print(json.dumps({"gpu": name, "power_limit": power, "max_sm_clock": clock}), flush=True)
    for s in a.shapes.split(","):
        run_shape(s, a.rounds, a.warmup)
    if a.old_lib:
        run_headline(a.old_lib, a.rounds, a.warmup)


if __name__ == "__main__":
    main()
