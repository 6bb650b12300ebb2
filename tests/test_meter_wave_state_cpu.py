"""CPU-only checks of the level-meter and waveform checkpoint calls (wf_meter_get_state / wf_meter_set_state,
wf_wave_get_state / wf_wave_set_state, wf_wave_get_clock / wf_wave_set_clock): the exports, the clock struct against the
header, the NULL-handle refusals that come before CUDA, and the binding's shape checks, which come before any library call."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
NEW = ["wf_meter_get_state", "wf_meter_set_state", "wf_wave_get_state", "wf_wave_set_state", "wf_wave_get_clock",
       "wf_wave_set_clock"]


def test_new_symbols_are_exported():
    from waveform_b200.engine import EXPORTS, load_library

    L = load_library()
    for name in NEW:
        assert name in EXPORTS and hasattr(L, name), name


def test_clock_struct_matches_the_header(tmp_path):
    from waveform_b200.engine import WfWaveClock

    src = tmp_path / "k.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(wf_wave_clock), offsetof(wf_wave_clock, clock_ns),'
                   ' offsetof(wf_wave_clock, audio_ts), offsetof(wf_wave_clock, waveform_ts),'
                   ' offsetof(wf_wave_clock, buffered));return 0;}\n')
    exe = tmp_path / "k"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(WfWaveClock), WfWaveClock.clock_ns.offset, WfWaveClock.audio_ts.offset,
                   WfWaveClock.waveform_ts.offset, WfWaveClock.buffered.offset]
    assert got == [32, 0, 8, 16, 24]


def test_null_handles_are_refused_before_cuda():
    from waveform_b200.engine import WF_ERR_INVALID_ARG, WfWaveClock, load_library

    L = load_library()
    buf, fl, clk = np.zeros(64, np.float32), np.zeros(4, np.uint8), WfWaveClock()
    p, q = buf.ctypes.data, fl.ctypes.data
    assert L.wf_meter_get_state(None, 0, 1, p, p, p, q) == WF_ERR_INVALID_ARG
    assert L.wf_meter_set_state(None, 0, 1, p, p, p, q) == WF_ERR_INVALID_ARG
    assert L.wf_wave_get_state(None, 0, 1, p, p, q) == WF_ERR_INVALID_ARG
    assert L.wf_wave_set_state(None, 0, 1, p, p, q) == WF_ERR_INVALID_ARG
    assert L.wf_wave_get_clock(None, C.byref(clk)) == WF_ERR_INVALID_ARG
    assert L.wf_wave_set_clock(None, C.byref(clk)) == WF_ERR_INVALID_ARG


class _NoCalls:
    """Stands for the library: any call is a failure of the test (the shape checks must come first)."""

    def __getattr__(self, name):
        raise AssertionError(f"library call {name} before the shape check")


def _meter(settings, cc, mode=None):
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import WfMeterConfig

    m = object.__new__(MeterEngine)
    m.L, m.h = _NoCalls(), None
    m.cfg = WfMeterConfig(max_streams=4, sample_rate=48000, capture_channels=cc, mode=1 if mode is None else mode,
                          sync_offset_ms=settings.get("audio_sync_offset", 0))
    m.window = 7200
    return m


def _wave(cc, stereo, offset=0):
    from waveform_b200 import WaveEngine
    from waveform_b200.engine import WfWaveConfig

    w = object.__new__(WaveEngine)
    w.L, w.h = _NoCalls(), None
    w.cfg = WfWaveConfig(max_streams=4, sample_rate=48000, capture_channels=cc, stereo=int(stereo), width=300,
                         sync_offset_ms=offset)
    return w


def test_meter_shape_checks_raise_before_the_library():
    m = _meter({"audio_sync_offset": 40}, 2)  # D = 1920
    good = {"ring": np.zeros((2, 2, 7200), np.float32), "line": np.zeros((2, 2, 1920), np.float32),
            "ema": np.zeros((2, 2), np.float32), "flags": np.zeros(2, np.uint8)}
    for key, bad in (("ring", np.zeros((2, 1, 7200))), ("ring", np.zeros((2, 2, 7199))), ("line", np.zeros((2, 2, 0))),
                     ("ema", np.zeros((2, 3))), ("flags", np.zeros((2, 1))), ("ring", np.zeros((2 * 2 * 7200,))),
                     ("ema", np.zeros((3, 2)))):
        with pytest.raises(ValueError):
            m.set_state({**good, key: bad})
    # without an offset the delay line is [count, cc, 0]
    m0 = _meter({}, 1)
    with pytest.raises(ValueError):
        m0.set_state({"line": np.zeros((1, 1, 1920), np.float32)})


def test_wave_shape_checks_raise_before_the_library():
    for cc, stereo, rows in ((1, False, 1), (2, False, 2), (1, True, 2), (2, True, 2)):
        w = _wave(cc, stereo, offset=10)  # D = 480
        good = {"db": np.zeros((3, rows, 300), np.float32), "hold": np.zeros((3, cc, 480), np.float32),
                "flags": np.zeros(3, np.uint8)}
        for key, bad in (("db", np.zeros((3, 3 - rows, 300))), ("db", np.zeros((3, rows, 301))),
                         ("hold", np.zeros((3, cc, 479))), ("flags", np.zeros(2)), ("hold", np.zeros((2, cc, 480)))):
            with pytest.raises(ValueError):
                w.set_state({**good, key: bad})
    with pytest.raises(ValueError):
        _wave(2, False).set_clock((1, 2, 3))
    with pytest.raises(KeyError):
        _wave(2, False).set_clock({"clock_ns": 1, "audio_ts": 1, "waveform_ts": 0})
