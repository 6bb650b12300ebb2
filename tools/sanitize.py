"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / synccheck) covering the three kernels.
Run:  PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool memcheck python tools/sanitize.py"""
import sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np, torch
from waveform_b200 import Engine
from helpers import synth_pcm
CASES = [({"fft_size": 2048}, 1, 20, 3, 1, False),
         ({"fft_size": 2048, "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "normalize_volume": True}, 1, 5, 3, 1, False),
         ({"fft_size": 1024, "channel_mode": "stereo", "interp_mode": "lanczos", "filter_mode": "gauss"}, 2, 3, 3, 2, True),
         ({"fft_size": 4096, "display_mode": "bars"}, 2, 2, 3, 4, True),
         ({"fft_size": 800}, 1, 3, 3, 1, True),
         ({"fft_size": 256}, 1, 9, 3, 1, True),
         ({"fft_size": 128, "channel_mode": "stereo"}, 2, 17, 2, 1, True),
         ({"fft_size": 16384}, 1, 2, 2, 2, False),
         # round 2: team kernel (few streams x many ticks, gate traffic), warp2 plans with radix 5 / 3 / 7 / 13 butterflies
         ({"fft_size": 2048, "gravity": 0.3, "floor": -40}, 1, 3, 37, 1, False),
         ({"fft_size": 800}, 1, 40, 5, 1, False),
         ({"fft_size": 1920, "slope": 0.5, "fast_peaks": True}, 1, 9, 4, 2, False),
         ({"fft_size": 1456}, 1, 5, 3, 1, False),
         # display variant of the warp-per-stream kernel (tables + dB row in shared memory), split runs of the headline kernel
         ({"fft_size": 1024, "display_mode": "bars", "interp_mode": "catmull_rom"}, 1, 5, 4, 1, True),
         ({"fft_size": 2048, "interp_mode": "lanczos", "filter_mode": "gauss"}, 1, 3, 3, 2, True),
         ({"fft_size": 2048}, 1, 2400, 3, 1, False)]
ONLY_NEXT = "--next-rows" in sys.argv   # meter / feed / waveform only (short enough for racecheck)
for s, ch, S, T, hopdiv, pts in ([] if ONLY_NEXT else CASES):
    e = Engine(s, channels=ch, max_streams=S); N = e.fft_size; hop = N // hopdiv
    x = synth_pcm(S, e.capture_channels, (T - 1) * hop + N); x[0, :, :] = 0
    if T > 20:
        x[1, :, 4 * hop:] = 0   # decay -> freeze: the team kernel's lazy team-wide gate reduction
    rms = np.full((S, T), 0.1, np.float32) if s.get("normalize_volume") else None
    o = e.process(torch.from_numpy(x).cuda(), T, hop, want_points=pts, want_peak=True,
                  input_rms=None if rms is None else torch.from_numpy(rms))
    torch.cuda.synchronize()
    o2 = Engine(s, channels=ch, max_streams=S).process(x, T, hop, want_points=pts, input_rms=rms)  # host-pointer path
    assert np.array_equal(o["db"].cpu().numpy(), o2["db"])
    print(s.get("fft_size"), "ok", float(o["db"].float().mean()), flush=True)

# level meter, RMS feed and waveform mode (host-pointer path, history shorter and longer than the window)
from waveform_b200 import MeterEngine, WaveEngine
from waveform_b200.engine import METER_INPUT_RMS
for mode, st in ((None, {"meter_buf": 20, "rms_mode": True}), (None, {"meter_buf": 50, "rms_mode": False}), (METER_INPUT_RMS, {})):
    for hop in (441, 480):   # 441: three-kernel path; 480 divides the windows (960 / 2400 / 48000): one-pass path, partials carried
        m = MeterEngine(st, channels=2, max_streams=3, mode=mode)
        x = synth_pcm(3, 2, 9 * hop)
        a = m.process(x[:, :, : 4 * hop], 4, hop); b = m.process(torch.from_numpy(x[:, :, 4 * hop:]).cuda(), 5, hop)
        torch.cuda.synchronize()
        print("meter", mode, hop, "ok", flush=True)
# waveform mode: the four channel layouts of the chunked kernel, many ticks per chunk (hop 97), a tick that replaces the whole
# buffer (hop 2000 at 64 points / 5 ms), and input that trips the silent rule (|x| = 1 for a full buffer, then zeros)
for st, ch, hop in (({"width": 300, "meter_buf": 50, "channel_mode": "stereo"}, 2, 800), ({"width": 200, "meter_buf": 10}, 1, 800),
                    ({"width": 301, "meter_buf": 40}, 2, 97), ({"width": 301, "meter_buf": 40, "channel_mode": "stereo"}, 1, 97),
                    ({"width": 64, "meter_buf": 5, "channel_mode": "stereo"}, 2, 2000)):
    w = WaveEngine(st, channels=ch, max_streams=3)
    T = 40
    x = synth_pcm(3, ch, T * hop)
    x[1, :, : 25 * hop] = 1.0
    x[1, :, 25 * hop:] = 0.0
    a = w.process(x[:, :, : 4 * hop], 4, hop); b = w.process(torch.from_numpy(x[:, :, 4 * hop:]).cuda(), T - 4, hop)
    torch.cuda.synchronize()
    print("wave", st["width"], ch, hop, "ok silent ticks:", int(b["silent"].sum()), flush=True)
# display stages: the waveform's render_curve in both kernels (with the Gaussian's scratch row, display-only calls) and the
# meter's render_bars on its fused and three-kernel paths
import os
for chunk in ("1", "0"):
    os.environ["WF_WAVE_CHUNK"] = chunk
    for st, ch, hop in (({"width": 301, "meter_buf": 40, "channel_mode": "stereo", "filter_mode": "gauss"}, 1, 97),
                        ({"width": 200, "meter_buf": 10, "interp_mode": "lanczos"}, 2, 800)):
        w = WaveEngine(st, channels=ch, max_streams=3)
        x = synth_pcm(3, ch, 12 * hop)
        a = w.process(x[:, :, : 4 * hop], 4, hop, want_points=True, want_pixels=True)
        b = w.process(torch.from_numpy(x[:, :, 4 * hop:]).cuda(), 8, hop, want_db=False, want_pixels=True)
        torch.cuda.synchronize()
        print("wave display", chunk, st["width"], ch, hop, "ok", float(b["min"][..., 0].mean()), flush=True)
os.environ.pop("WF_WAVE_CHUNK")
# device-clock waveform engine: the plan kernel, a call captured into a graph (sync offset: start-up ticks, then points) and
# replayed between eager calls
w = WaveEngine({"width": 301, "meter_buf": 40, "channel_mode": "stereo", "audio_sync_offset": 20}, channels=2, max_streams=2,
               device_clock=True)
xin = torch.zeros((2, 2, 3 * 441), device="cuda")
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    o = w.process(xin, 3, 441, want_pixels=True)
for i in range(4):
    xin.copy_(torch.from_numpy(synth_pcm(2, 2, 3 * 441, seed=i)))
    g.replay()
    w.process(torch.from_numpy(synth_pcm(2, 2, 5 * 97, seed=10 + i)).cuda(), 5, 97)
torch.cuda.synchronize()
print("wave device clock graph ok", float(o["min"][..., 0].mean()), flush=True)
for hop in (441, 480):
    m = MeterEngine({"meter_buf": 20, "rounded_caps": True}, channels=2, max_streams=3)
    x = synth_pcm(3, 2, 9 * hop)
    a = m.process(x, 9, hop, want_pixels=True)
    print("meter display", hop, "ok", float(a["pixels"].mean()), flush=True)
# checkpoints: meter and waveform state (ring halves picked on the device, delay lines, holdbacks) and the waveform clock,
# moved from one engine into slots of a larger one and run on; the device-clock engine's graph replays after a restore
for mode in (None, METER_INPUT_RMS):
    src, dst = (MeterEngine({"meter_buf": 20, "audio_sync_offset": 15}, channels=2, max_streams=n, mode=mode) for n in (2, 5))
    src.process(synth_pcm(2, 2, 7 * 480), 7, 480)
    dst.set_state(src.get_state(), first_stream=3)
    dst.process(synth_pcm(2, 2, 3 * 441), 3, 441, first_stream=3)
    print("meter state", mode, "ok", float(dst.get_state(3, 2)["ring"].mean()), flush=True)
src = WaveEngine({"width": 301, "meter_buf": 40, "channel_mode": "stereo", "audio_sync_offset": 20}, channels=2, max_streams=3)
src.process(synth_pcm(3, 2, 4 * 441), 4, 441)
w.set_state(src.get_state(1, 2))
w.set_clock(src.get_clock())
xin.copy_(torch.from_numpy(synth_pcm(2, 2, 3 * 441, seed=20)))
g.replay()
torch.cuda.synchronize()
print("wave state", "ok", float(w.get_state()["db"].mean()), w.get_clock(), flush=True)
