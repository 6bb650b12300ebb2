"""CPU-only checks of the audio sync offset (wf_config / wf_meter_config / wf_wave_config .sync_offset_ms): the configs'
layout against the header, the previous struct sizes, the range check, and the numpy model of each engine against the
compiled plugin (oracle/_ref) fed packet by packet with its `audio_sync_offset` setting."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
OFFSETS_MS = [10, 170, 1000]
SR = 48000


def _delay(ms):
    return SR * ms // 1000 if ms > 0 else 0


def _need_reference():
    from oracle import refbind

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return refbind


def test_config_layouts_match_header(tmp_path):
    from waveform_b200.engine import WfConfig, WfMeterConfig, WfWaveConfig, load_library

    src = tmp_path / "c.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(wf_config), offsetof(wf_config, sync_offset_ms),'
                   ' sizeof(wf_meter_config), offsetof(wf_meter_config, sync_offset_ms),'
                   ' sizeof(wf_wave_config), offsetof(wf_wave_config, sync_offset_ms));return 0;}\n')
    exe = tmp_path / "c"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(WfConfig), WfConfig.sync_offset_ms.offset, C.sizeof(WfMeterConfig),
                   WfMeterConfig.sync_offset_ms.offset, C.sizeof(WfWaveConfig), WfWaveConfig.sync_offset_ms.offset]
    for cls in (WfConfig, WfMeterConfig, WfWaveConfig):
        assert cls.sync_offset_ms.offset + 4 == C.sizeof(cls)  # appended last
    L = load_library()
    for cls, init in ((WfConfig, L.wf_config_init), (WfMeterConfig, L.wf_meter_config_init),
                      (WfWaveConfig, L.wf_wave_config_init)):
        c = cls()
        c.sync_offset_ms = 123
        init(C.byref(c))
        assert c.sync_offset_ms == 0 and c.struct_size == C.sizeof(cls)


def test_settings_map_onto_the_field():
    from waveform_b200.engine import make_config, make_meter_config, make_wave_config

    assert make_config({"audio_sync_offset": 170}).sync_offset_ms == 170
    assert make_meter_config({"audio_sync_offset": -30}).sync_offset_ms == -30
    assert make_wave_config({"audio_sync_offset": 1000}).sync_offset_ms == 1000
    assert make_config().sync_offset_ms == 0


def test_previous_sizes_and_range():
    from waveform_b200.engine import (TABLE_WINDOW, WF_ERR_INVALID_ARG, WfConfig, WfInfo, WfWaveConfig, load_library,
                                      make_config, make_wave_config)

    L = load_library()
    cfg = make_config({"fft_size": 1024})
    want = np.zeros(1024, np.float32)
    assert L.wf_preview_table(C.byref(cfg), TABLE_WINDOW, want.ctypes.data, 1024, None) == 1024
    old = make_config({"fft_size": 1024})
    old.sync_offset_ms = 999  # past the previous struct's end: never read
    old.struct_size = WfConfig.sync_offset_ms.offset
    got = np.zeros(1024, np.float32)
    info = WfInfo()
    assert L.wf_preview_table(C.byref(old), TABLE_WINDOW, got.ctypes.data, 1024, C.byref(info)) == 1024
    assert np.array_equal(got, want) and info.fft_size == 1024
    for ms in (-1000, 0, 10, 1000):
        cfg.sync_offset_ms = ms
        assert L.wf_preview_table(C.byref(cfg), TABLE_WINDOW, None, 0, None) == 1024
    for ms in (-1010, 1001, 2**31 - 1):
        cfg.sync_offset_ms = ms
        assert L.wf_preview_table(C.byref(cfg), TABLE_WINDOW, None, 0, None) == WF_ERR_INVALID_ARG

    wc = make_wave_config({"width": 300, "meter_buf": 50}, channels=1)
    counts = np.zeros(8, np.int32)
    n0 = L.wf_wave_preview_plan(C.byref(wc), 8, 441, counts.ctypes.data, None, 0)
    assert n0 > 0
    wc.sync_offset_ms = 999
    wc.struct_size = WfWaveConfig.sync_offset_ms.offset  # previous size: no offset
    c2 = np.zeros(8, np.int32)
    assert L.wf_wave_preview_plan(C.byref(wc), 8, 441, c2.ctypes.data, None, 0) == n0
    assert np.array_equal(c2, counts)
    wc.struct_size = C.sizeof(WfWaveConfig)
    for ms in (-1001, 1010):
        wc.sync_offset_ms = ms
        assert L.wf_wave_preview_plan(C.byref(wc), 8, 441, None, None, 0) == WF_ERR_INVALID_ARG
    wc.sync_offset_ms = -1000  # a negative offset holds nothing back
    assert L.wf_wave_preview_plan(C.byref(wc), 8, 441, c2.ctypes.data, None, 0) == n0


# ---- spectrum: ring calls with an offset ----------------------------------------------------------------------------

# (ticks, hop) per call: hops below, at and above N, changing between calls
def _calls(N):
    return [(3, 800), (1, 800), (2, N), (1, N + 400), (4, 512), (6, 1600), (2, 300)]


def spectrum_model(N, D, x, calls):
    """The ring model of a capture-ring call with sync delay D: per call, (frames [T, cc, N], skipped [T]).  Frame t is the
    oldest N of the newest N + D samples of zeros(N + D) ++ stream (the ring's start-up zeros) once the packet of tick t has
    arrived; a tick is short of audio ("skipped") while fewer than D samples have arrived in all."""
    cc = x.shape[0]
    C_ = np.concatenate([np.zeros((cc, N + D), np.float32), x], axis=1)
    pos, out = 0, []
    for T_, hop in calls:
        frames, skip = [], []
        for t in range(T_):
            p = pos + (t + 1) * hop  # samples arrived in all
            frames.append(C_[:, p: p + N])
            skip.append(p < D)
        out.append((np.stack(frames), np.array(skip)))
        pos += T_ * hop
    return out


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("N,cc,stereo,window", [(800, 1, False, "hann"), (2048, 1, False, "hann"),
                                                 (4096, 2, True, "blackman_harris")])
def test_spectrum_ring_model_is_the_plugins(N, cc, stereo, window, ms):
    """The plugin fed packet by packet with its audio sync offset: every tick the model calls short of audio leaves
    m_decibels and m_last_silent as they were, and the other ticks equal a plain run (no offset) over the model's frames."""
    from helpers import synth_pcm

    refbind = _need_reference()
    D = _delay(ms)
    calls = _calls(N)
    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=0x5C + N + ms)[0]
    x[:, total // 3: total // 3 + N] = 0.0  # digital silence inside
    settings = {"fft_size": N, "window": window, "silence_gate": True}
    if stereo:
        settings["channel_mode"] = "stereo"
    pk = refbind.RefSource({**settings, "audio_sync_offset": ms}, channels=cc)
    plain = refbind.RefSource(settings, channels=cc)
    dch = pk.display_channels
    prev_db = np.stack([pk.decibels(c) for c in range(dch)])
    prev_sil = pk.last_silent
    timeline = np.concatenate([np.zeros((cc, N + D), np.float32), x], axis=1)
    pos = 0
    n_skipped = 0
    for (T_, hop), (frames, skip) in zip(calls, spectrum_model(N, D, x, calls)):
        got_db, got_sil = [], []
        for t in range(T_):
            seg = x[:, pos + t * hop: pos + (t + 1) * hop]
            pk.advance(hop / pk.sample_rate)
            pk.push(seg[0], seg[1] if cc == 2 else None)
            pk.tick(1.0 / 60.0)
            got_db.append(np.stack([pk.decibels(c) for c in range(dch)]))
            got_sil.append(pk.last_silent)
            if skip[t]:
                assert np.array_equal(got_db[-1], prev_db) and got_sil[-1] == prev_sil, (N, ms, t)
            prev_db, prev_sil = got_db[-1], got_sil[-1]
        n_skipped += int(skip.sum())
        run = ~skip
        assert not (skip[1:] & ~skip[:-1]).any()  # the start-up ticks come first
        k = int(run.sum())
        if k:  # the frames of the real ticks, `hop` apart: one plain run over their span
            p0 = pos + (T_ - k + 1) * hop
            want = plain.run_stft(timeline[:, p0: p0 + (k - 1) * hop + N], k, hop)
            assert want["frames"] == k
            assert np.array_equal(np.stack(got_db)[run], want["db"]), (N, ms, T_, hop)
            assert np.array_equal(np.array(got_sil, np.uint8)[run], want["silent"]), (N, ms, T_, hop)
            assert np.array_equal(frames[run][0], timeline[:, p0: p0 + N])
        pos += T_ * hop
    assert n_skipped == sum(1 for _, s in spectrum_model(N, D, x, calls) for v in s if v)
    if D > 800:
        assert n_skipped > 0


# ---- level meter and RMS feed: zeros(D) ++ stream --------------------------------------------------------------------

METER_CASES = [({"display_mode": "level_meter", "rms_mode": False, "meter_buf": 100}, 2),
               ({"display_mode": "level_meter", "rms_mode": True, "meter_buf": 150}, 2),
               ({"display_mode": "level_meter", "rms_mode": True, "meter_buf": 20}, 1),
               ({"fft_size": 1024, "normalize_volume": True, "channel_mode": "stereo"}, 2)]  # the RMS feed


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("settings,cc", METER_CASES)
def test_meter_offset_is_a_zero_prefixed_stream(settings, cc, ms):
    """tick_meter / sync_rms_buffer with the offset consume all but the newest D samples: the plugin with the offset equals
    the plugin without it fed zeros(D) ++ stream (peaks exactly; RMS sums in another ring order, to a few 1e-6)."""
    from helpers import synth_pcm

    refbind = _need_reference()
    D = _delay(ms)
    feed = bool(settings.get("normalize_volume"))
    # capture_audio squares the first AUDIO_OUTPUT_FRAMES (1024) samples of a packet again for each further 1024-sample part
    # (src/source.cpp:1846-1864 never advances `data`), so the feed depends on where packets start unless they are that short
    calls = [(5, 480), (3, 800), (9, 1024), (2, 97), (7, 333), (4, 1000)] if feed else \
        [(5, 480), (3, 800), (2, 4800), (1, 9000), (7, 333), (4, 2048)]
    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=0x3E + ms)[0]
    x[:, total // 4: total // 4 + 6000] = 0.0
    xd = np.concatenate([np.zeros((cc, D), np.float32), x], axis=1)
    off = refbind.RefSource({**settings, "audio_sync_offset": ms}, channels=cc)
    zero = refbind.RefSource(settings, channels=cc)
    peak = settings.get("rms_mode") is False
    pos = 0
    for T_, hop in calls:
        a = off.run_meter(x[:, pos: pos + T_ * hop], T_, hop)
        b = zero.run_meter(xd[:, pos: pos + T_ * hop], T_, hop)
        for k in (("rms",) if feed else ("db", "lin", "silent")):
            if peak or k == "silent":
                assert np.array_equal(a[k], b[k]), (k, ms, hop)
            else:
                np.testing.assert_allclose(a[k], b[k], rtol=1e-5, atol=1e-9 if k != "db" else 1e-4, err_msg=f"{k} {ms} {hop}")
        pos += T_ * hop


# ---- waveform: the plan with the reserve -----------------------------------------------------------------------------

def wave_plan(width, meter_ms, D, hops, sr=SR):
    """tick_waveform's timestamp walk with the reserve of D samples (src/source_generic.cpp:290-339,358) for packets of the
    given sizes stamped "now": per tick, the stream index of every new point's sample (negative: a start-up or delay zero)."""
    ws = int(float(sr) * (meter_ms / 1000.0))
    step = meter_ms * 1000000 // width
    clock, wts, buffered, pos = 10 * 10**9, 0, width, 0
    out = []
    for hop in hops:
        clock += hop * 10**9 // sr
        ats = clock
        pos += hop
        total = min(buffered + hop, ws + D)
        buffered = total
        pts = []
        if total > D:
            start, stop = ats - total * 10**9 // sr, ats - D * 10**9 // sr
            if wts < start:
                wts = start
            if wts > stop and wts - stop > step:
                wts = start
            for i in range(width):
                ts = wts + i * step
                if ts >= stop:
                    break
                index = min(max((ats - ts) * sr // 10**9, D + 1), total)
                pts.append(pos - index)
            wts += len(pts) * step
            buffered = D
        out.append(np.array(pts, np.int64))
    return out


@pytest.mark.parametrize("ms", OFFSETS_MS)
@pytest.mark.parametrize("width,meter_ms", [(800, 150), (300, 50), (200, 10), (640, 500)])
def test_wave_plan_model_is_the_plugins(width, meter_ms, ms):
    """A mono capture shown as two channels leaves the raw new samples in the second channel, so a ramp reveals which
    sample the plugin took for every point of every tick; the model (and wf_wave_preview_plan on a first call) agree."""
    from waveform_b200.engine import make_wave_config, preview_wave_plan

    refbind = _need_reference()
    D = _delay(ms)
    settings = {"display_mode": "waveform", "width": width, "meter_buf": meter_ms, "channel_mode": "stereo"}
    hops = [480] * 6 + [800] * 5 + [4800, 300, 300] + [2000] * 8 + [97] * 30 + [1600] * 10 + [30000, 441, 441]
    total = sum(hops)
    ramp = ((np.arange(total, dtype=np.float64) + 1.0) * 2.0 ** -20).astype(np.float32)[None, :]  # exact, never 0
    r = refbind.RefSource({**settings, "audio_sync_offset": ms}, channels=1)
    plan = wave_plan(width, meter_ms, D, hops)
    pos, emitted = 0, 0
    for t, hop in enumerate(hops):
        out = r.run_wave(ramp[:, pos: pos + hop], 1, hop)["out"][0, 1]
        pts = plan[t]
        c = len(pts)
        emitted += c
        want = np.where(pts >= 0, ramp[0, np.maximum(pts, 0)], np.float32(0.0))
        assert np.array_equal(out[width - c:], want), (t, hop, c)
        pos += hop
    assert emitted > 0
    # the engine's own plan of a first call (one hop throughout)
    for hop in (480, 97, 4800):
        cfg = make_wave_config({k: v for k, v in settings.items() if k != "display_mode"} | {"audio_sync_offset": ms},
                               channels=1)
        counts, src = preview_wave_plan(cfg, 40, hop)
        model = wave_plan(width, meter_ms, D, [hop] * 40)
        assert np.array_equal(counts, [len(p) for p in model]), hop
        assert np.array_equal(src, np.concatenate(model).clip(min=-1)), hop
