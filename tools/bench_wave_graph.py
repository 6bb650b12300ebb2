"""Waveform calls on the host clock, on the device clock, and replayed from a CUDA graph, alternating in one process.

Three engines are fed the same samples: a host-clock engine (wf_wave_create) and a device-clock engine
(wf_wave_create_with_clock, device_clock = 1) driven by eager wf_wave_process_async calls, and a second device-clock
engine driven by replays of one call captured once (torch.cuda.graph, default capture mode, no warm-up call).  Shapes:
  * live:  1 stream x 1 tick, stereo capture and display, width 800, 150 ms, hop 800, out_pixels + out_min, every buffer
           in wf_host_alloc (device-mapped) memory; once without a sync offset and once with 40 ms;
  * chain: the live shape with 40 ms as a waveform-mode tick: an RMS feed (WF_METER_INPUT_RMS) of the same samples
           feeding the waveform's input_rms, with normalize_volume (the host variant's waveform is on the host clock);
  * batch: 1024 streams x 64 ticks, hop 800, dB rows and silent flags in device buffers;
  * long:  1 stream x 4096 ticks, hop 800, the same outputs: the device planner's longest walk (runs of 1024 ticks).
The variants take turns in blocks, the order rotating every block, so that drift on a shared host lands on all of them.  A
call is timed by a host clock around the call and a stream synchronise (wall), and by CUDA events recorded on the stream
around it (device).  For the batch and long shapes the plan kernel's own time is then taken from torch.profiler over
device-clock calls.  Printed: the card's name and power limit, then one JSON line per shape with each variant's median
per-call times, the range of its per-block wall medians, and whether the three variants' outputs stayed bit-identical.

    python tools/bench_wave_graph.py [--blocks 12] [--calls 200] [--big-blocks 6] [--big-calls 10]
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
from waveform_b200 import MeterEngine, WaveEngine  # noqa: E402

VARIANTS = ("host", "device", "graph")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return [v.strip() for v in q.split(",")]


class Calls:
    """One waveform engine over its own buffers (mapped host memory or device tensors) and one wf_wave_batch.  With `feed`
    (mapped buffers only), an RMS feed (WF_METER_INPUT_RMS) of the same samples goes first and its output is the waveform's
    input_rms: the waveform-mode tick of a plugin source."""

    def __init__(self, settings, S, cc, T, hop, mapped, device_clock, feed=None):
        import torch

        self.eng = WaveEngine(settings, channels=cc, max_streams=S, device_clock=device_clock)
        L = self.L = self.eng.L
        W, dch = self.eng.cfg.width, self.eng.display_channels
        n_pcm, n_row = S * cc * T * hop, S * T * dch * W
        b = self.b = wfe.WfWaveBatch()
        b.struct_size = C.sizeof(wfe.WfWaveBatch)
        b.n_streams, b.n_ticks, b.hop = S, T, hop
        b.stream_stride, b.channel_stride = cc * T * hop, T * hop
        self.mapped = mapped
        if mapped:  # display outputs: pixels and (miny, minpos)
            nbytes = (4 * n_pcm, 4 * n_row, 4 * S * T * 2, S * T)
            self.ptrs = [L.wf_host_alloc(n) for n in nbytes]
            if not all(self.ptrs):
                raise RuntimeError("wf_host_alloc failed")
            self.pcm = np.ctypeslib.as_array((C.c_float * n_pcm).from_address(self.ptrs[0]))
            self.outs = [np.ctypeslib.as_array((C.c_uint8 * n).from_address(p)) for n, p in zip(nbytes[1:], self.ptrs[1:])]
            b.pcm, b.out_pixels, b.out_min, b.out_silent = self.ptrs
            self.feed = None
            if feed is not None:
                self.feed = MeterEngine(feed, channels=cc, max_streams=S, mode=wfe.METER_INPUT_RMS)
                self.ptrs.append(L.wf_host_alloc(4 * S * T))
                if not self.ptrs[-1]:
                    raise RuntimeError("wf_host_alloc failed")
                self.outs.append(np.ctypeslib.as_array((C.c_uint8 * (4 * S * T)).from_address(self.ptrs[-1])))
                mb = self.mb = wfe.WfMeterBatch()
                mb.struct_size = C.sizeof(wfe.WfMeterBatch)
                mb.n_streams, mb.n_ticks, mb.hop, mb.seconds = S, T, hop, 1.0 / 60.0
                mb.pcm, mb.stream_stride, mb.channel_stride = self.ptrs[0], cc * T * hop, T * hop
                mb.out_lin = b.input_rms = self.ptrs[-1]
        else:  # dB rows and silent flags
            self.pcm = torch.zeros(n_pcm, device="cuda")
            self.outs = [torch.zeros(n_row, device="cuda"), torch.zeros(S * T, dtype=torch.uint8, device="cuda")]
            b.pcm, b.out, b.out_silent = self.pcm.data_ptr(), self.outs[0].data_ptr(), self.outs[1].data_ptr()

    def set_pcm(self, x):
        if self.mapped:
            self.pcm[:] = x
        else:
            import torch
            self.pcm.copy_(torch.from_numpy(x))

    def call(self, stream):
        if getattr(self, "feed", None) is not None and self.L.wf_meter_process_async(self.feed.h, C.byref(self.mb), stream):
            raise RuntimeError(f"feed call failed: {self.L.wf_meter_last_error(self.feed.h)}")
        if self.L.wf_wave_process_async(self.eng.h, C.byref(self.b), stream) != 0:
            raise RuntimeError(f"call failed: {self.L.wf_wave_last_error(self.eng.h)}")

    def out(self):
        return [o.copy() if self.mapped else o.cpu().numpy() for o in self.outs]

    def close(self):
        if self.mapped:
            for p in self.ptrs:
                self.L.wf_host_free(p)


def plan_kernel_us(calls, stream, n):
    """Mean device time of wave_plan_kernel over n eager calls of a device-clock engine, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            calls.call(stream.cuda_stream)
        stream.synchronize()
    ev = [e for e in prof.key_averages() if "wave_plan_kernel" in e.key]
    if not ev:
        return None
    total = sum(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0) for e in ev)
    torch.cuda.synchronize()
    return round(total / sum(e.count for e in ev), 2)


def bench(shape, settings, S, cc, T, hop, mapped, blocks, calls, warmup, plan_calls=0, feed=None):
    import torch

    stream = torch.cuda.Stream()
    rng = np.random.default_rng(11)
    frames = []
    for _ in range(4):
        x = (0.3 * rng.standard_normal(S * cc * T * hop)).astype(np.float32)
        x[: x.size // 8] = 0.0  # a stretch of digital silence
        frames.append(x)
    eng = {c: Calls(settings, S, cc, T, hop, mapped, c != "host", feed) for c in VARIANTS}
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        eng["graph"].call(torch.cuda.current_stream().cuda_stream)
    runs = {"host": lambda: eng["host"].call(stream.cuda_stream), "device": lambda: eng["device"].call(stream.cuda_stream),
            "graph": g.replay}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    wall = {c: [] for c in VARIANTS}
    dev = {c: [] for c in VARIANTS}
    block_medians = {c: [] for c in VARIANTS}
    count = {c: 0 for c in VARIANTS}

    def run(c, n, record):
        block = []
        with torch.cuda.stream(stream):
            for _ in range(n):
                eng[c].set_pcm(frames[count[c] % len(frames)])
                count[c] += 1
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record(stream)
                runs[c]()
                e1.record(stream)
                stream.synchronize()
                t1 = time.perf_counter()
                if record:
                    block.append((t1 - t0) * 1e6)
                    dev[c].append(e0.elapsed_time(e1) * 1e3)
        if record:
            wall[c] += block
            block_medians[c].append(float(np.median(block)))

    for c in VARIANTS:
        run(c, warmup, False)
    for k in range(blocks):
        for c in VARIANTS[k % 3:] + VARIANTS[: k % 3]:
            run(c, calls, True)
    torch.cuda.synchronize()
    outs = {c: eng[c].out() for c in VARIANTS}
    same = all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
               for c in ("device", "graph") for a, b in zip(outs[c], outs["host"]))
    res = {"shape": shape, "calls_per_variant": len(wall["host"]), "bit_equal_outputs": bool(same)}
    for c in VARIANTS:
        res[f"{c}_wall_median_us"] = round(float(np.median(wall[c])), 2)
        res[f"{c}_device_median_us"] = round(float(np.median(dev[c])), 2)
        res[f"{c}_block_wall_median_range_us"] = [round(min(block_medians[c]), 2), round(max(block_medians[c]), 2)]
    if plan_calls:
        res["plan_kernel_us"] = plan_kernel_us(eng["device"], stream, plan_calls)
    print(json.dumps(res), flush=True)
    for e in eng.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=12)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--big-blocks", type=int, default=6)
    ap.add_argument("--big-calls", type=int, default=10)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("this measurement needs a GPU")
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    live = {"width": 800, "meter_buf": 150, "channel_mode": "stereo"}
    bench("live_1x1_w800_stereo_pixels+min_host_alloc", live, 1, 2, 1, 800, True, a.blocks, a.calls, 100)
    bench("live_1x1_w800_stereo_pixels+min_host_alloc_offset40ms", {**live, "audio_sync_offset": 40}, 1, 2, 1, 800, True,
          a.blocks, a.calls, 100)
    bench("live_1x1_feed+wave_w800_stereo_normalized_pixels+min_host_alloc_offset40ms",
          {**live, "normalize_volume": True, "audio_sync_offset": 40}, 1, 2, 1, 800, True, a.blocks, a.calls, 100,
          feed={"audio_sync_offset": 40})
    wide = {"width": 800, "meter_buf": 150}
    bench("batch_1024x64_w800_mono_db_device", wide, 1024, 2, 64, 800, False, a.big_blocks, a.big_calls, 3, plan_calls=20)
    bench("long_1x4096_w800_mono_db_device", wide, 1, 2, 4096, 800, False, a.big_blocks, a.big_calls, 3, plan_calls=20)


if __name__ == "__main__":
    main()
