"""Eager calls against a replayed CUDA graph of the same calls, alternating in one process.

One spectrum-mode tick is an RMS-feed call (wf_meter_process_async, WF_METER_INPUT_RMS) followed by a capture-ring
spectrum call (wf_process_async) that normalises the volume with the feed's output.  Two shapes:
  * live:  1 stream x 1 frame, N=800, stereo capture, hop 800, every buffer in wf_host_alloc (device-mapped) memory;
  * batch: 4096 streams x 16 ticks, N=2048 mono, hop 800, device buffers.
Each shape has two engine pairs fed the same samples: one driven by eager calls, one by replays of a graph captured once
(torch.cuda.graph, default capture mode, no warm-up call).  They take turns in blocks, the order flipping every block, so
that drift on a shared host lands on both.  A tick is timed by a host clock around the tick and a stream synchronise
(wall), and by CUDA events recorded on the stream around it (device).  Printed: the card's name and power limit, then one
JSON line per shape with each variant's median per-tick times, the range of its per-block wall medians, and whether the
two pairs' outputs stayed bit-identical.

    python tools/bench_graph.py [--live-blocks 20] [--live-ticks 500] [--batch-blocks 6] [--batch-ticks 10]
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
from waveform_b200 import Engine, MeterEngine  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return [v.strip() for v in q.split(",")]


class Pair:
    """RMS feed + ring spectrum engines over one set of buffers (mapped host memory or device tensors)."""

    def __init__(self, S, cc, N, T, hop, mapped):
        import torch

        self.S, self.cc, self.T, self.hop = S, cc, T, hop
        settings = {"fft_size": N, "normalize_volume": True}
        self.spec = Engine(settings, channels=cc, max_streams=S)
        self.feed = MeterEngine({}, channels=cc, max_streams=S, mode=wfe.METER_INPUT_RMS)
        L = self.L = self.spec.L
        n_pcm, n_rms = S * cc * T * hop, S * T
        n_db, n_sil = S * T * self.spec.display_channels * self.spec.bins, S * T
        self.mapped = mapped
        if mapped:
            self.ptrs = [L.wf_host_alloc(n * es) for n, es in ((n_pcm, 4), (n_rms, 4), (n_db, 4), (n_sil, 1))]
            if not all(self.ptrs):
                raise RuntimeError("wf_host_alloc failed")
            self.pcm = np.ctypeslib.as_array((C.c_float * n_pcm).from_address(self.ptrs[0]))
            self.db = np.ctypeslib.as_array((C.c_float * n_db).from_address(self.ptrs[2]))
        else:
            self.pcm = torch.zeros(n_pcm, device="cuda")
            self.bufs = [self.pcm, torch.zeros(n_rms, device="cuda"), torch.zeros(n_db, device="cuda"),
                         torch.zeros(n_sil, dtype=torch.uint8, device="cuda")]
            self.ptrs = [t.data_ptr() for t in self.bufs]
            self.db = self.bufs[2]
        mb = self.mb = wfe.WfMeterBatch()
        mb.struct_size = C.sizeof(wfe.WfMeterBatch)
        mb.n_streams, mb.n_ticks, mb.hop, mb.seconds = S, T, hop, 1.0 / 60.0
        mb.pcm, mb.stream_stride, mb.channel_stride, mb.out_lin = self.ptrs[0], cc * T * hop, T * hop, self.ptrs[1]
        sb = self.sb = wfe.WfBatch()
        sb.struct_size = C.sizeof(wfe.WfBatch)
        sb.n_streams, sb.n_frames, sb.hop, sb.seconds = S, T, hop, 1.0 / 60.0
        sb.pcm, sb.stream_stride, sb.channel_stride = self.ptrs[0], cc * T * hop, T * hop
        sb.input_rms, sb.out_db, sb.out_silent = self.ptrs[1], self.ptrs[2], self.ptrs[3]
        sb.capture_ring = wfe.CAPTURE_RING

    def set_pcm(self, x):
        if self.mapped:
            self.pcm[:] = x
        else:
            import torch
            self.pcm.copy_(torch.from_numpy(x))

    def tick(self, stream):
        rc = self.L.wf_meter_process_async(self.feed.h, C.byref(self.mb), stream)
        rc = rc or self.L.wf_process_async(self.spec.h, C.byref(self.sb), stream)
        if rc != 0:
            raise RuntimeError(f"tick failed: {self.spec.L.wf_last_error(self.spec.h)}")

    def out(self):
        return self.db.copy() if self.mapped else self.db.cpu().numpy()

    def close(self):
        if self.mapped:
            for p in self.ptrs:
                self.L.wf_host_free(p)


def bench(shape, S, cc, N, T, hop, mapped, blocks, ticks, warmup):
    import torch

    stream = torch.cuda.Stream()
    rng = np.random.default_rng(11)
    frames = [(0.3 * rng.standard_normal(S * cc * T * hop)).astype(np.float32) for _ in range(4)]
    pairs = {"eager": Pair(S, cc, N, T, hop, mapped), "graph": Pair(S, cc, N, T, hop, mapped)}
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        pairs["graph"].tick(torch.cuda.current_stream().cuda_stream)
    runs = {"eager": lambda: pairs["eager"].tick(stream.cuda_stream), "graph": g.replay}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    wall = {c: [] for c in runs}
    dev = {c: [] for c in runs}
    block_medians = {c: [] for c in runs}
    count = {c: 0 for c in runs}

    def run(c, n, record):
        block = []
        with torch.cuda.stream(stream):
            for _ in range(n):
                pairs[c].set_pcm(frames[count[c] % len(frames)])
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

    for c in runs:
        run(c, warmup, False)
    for k in range(blocks):
        for c in ("eager", "graph") if k % 2 == 0 else ("graph", "eager"):
            run(c, ticks, True)
    torch.cuda.synchronize()
    res = {"shape": shape, "ticks_per_variant": len(wall["eager"]),
           "bit_equal_outputs": bool(np.array_equal(pairs["eager"].out().view(np.int32),
                                                    pairs["graph"].out().view(np.int32)))}
    for c in runs:
        res[f"{c}_wall_median_us"] = round(float(np.median(wall[c])), 2)
        res[f"{c}_device_median_us"] = round(float(np.median(dev[c])), 2)
        res[f"{c}_block_wall_median_range_us"] = [round(min(block_medians[c]), 2), round(max(block_medians[c]), 2)]
    print(json.dumps(res), flush=True)
    for p in pairs.values():
        p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--live-blocks", type=int, default=20)
    ap.add_argument("--live-ticks", type=int, default=500)
    ap.add_argument("--batch-blocks", type=int, default=6)
    ap.add_argument("--batch-ticks", type=int, default=10)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("this measurement needs a GPU")
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    bench("live_1x1_N800_stereo_feed+ring_host_alloc", 1, 2, 800, 1, 800, True, a.live_blocks, a.live_ticks, 200)
    bench("batch_4096x16_N2048_mono_feed+ring_device", 4096, 1, 2048, 16, 800, False, a.batch_blocks, a.batch_ticks, 3)


if __name__ == "__main__":
    main()
