"""CPU-only checks of the waveform engine's device clock (wf_wave_create_with_clock): the ABI, the argument checks that come
before the device, the Python keyword, and the host plan it is held to on the GPU, which must not depend on the config's
struct size."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_create_with_clock_is_declared_and_leaves_the_config_alone(tmp_path):
    """The choice is an argument of the create call: wf_wave_config keeps its layout, sync_offset_ms last."""
    from waveform_b200.engine import EXPORTS, WfWaveConfig, load_library

    src = tmp_path / "c.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){int (*f)(const wf_wave_config *, int32_t, wf_wave **) = wf_wave_create_with_clock; (void)f;'
                   'printf("%zu %zu\\n", sizeof(wf_wave_config), offsetof(wf_wave_config, sync_offset_ms));return 0;}\n')
    exe = tmp_path / "c"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe), "-Wl,--unresolved-symbols=ignore-all"],
                   check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(WfWaveConfig), WfWaveConfig.sync_offset_ms.offset]
    assert "wf_wave_create_with_clock" in EXPORTS and hasattr(load_library(), "wf_wave_create_with_clock")


def test_argument_errors_come_before_the_device():
    """device_clock other than 0 / 1 is WF_ERR_INVALID_ARG, as is a bad config, with or without a GPU; without one, a valid
    call is WF_ERR_NO_DEVICE (no CPU fallback) for both clocks."""
    import torch
    from waveform_b200.engine import WF_ERR_INVALID_ARG, make_wave_config, load_library

    L = load_library()
    h = C.c_void_p()
    cfg = make_wave_config({}, channels=2)
    for bad in (2, -1, 1 << 30):
        assert L.wf_wave_create_with_clock(C.byref(cfg), bad, C.byref(h)) == WF_ERR_INVALID_ARG and not h.value
        assert b"device_clock" in L.wf_wave_last_error(None)
    cfg.width = 0
    assert L.wf_wave_create_with_clock(C.byref(cfg), 1, C.byref(h)) == WF_ERR_INVALID_ARG and not h.value
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device branch cannot be exercised")
    cfg.width = 800
    for clock in (0, 1):
        assert L.wf_wave_create_with_clock(C.byref(cfg), clock, C.byref(h)) == -4 and not h.value


def test_python_keyword_selects_the_clock(monkeypatch):
    """WaveEngine(device_clock=...) passes 0 / 1 to wf_wave_create_with_clock; it is not a settings key."""
    from waveform_b200 import WaveEngine
    from waveform_b200.engine import WfError, load_library, make_wave_config

    L = load_library()
    seen = []

    class Spy:
        def __getattr__(self, name):
            if name == "wf_wave_create_with_clock":
                def create(cfg, clock, h):
                    seen.append(clock)
                    return -4
                return create
            return getattr(L, name)

    monkeypatch.setattr("waveform_b200.engine.load_library", lambda: Spy())
    for kw, want in (({}, 0), ({"device_clock": False}, 0), ({"device_clock": True}, 1)):
        with pytest.raises(WfError):
            WaveEngine({}, channels=2, **kw)
        assert seen[-1] == want
    with pytest.raises(KeyError):
        make_wave_config({"device_clock": True})


@pytest.mark.parametrize("settings,ch,hop,T", [({"width": 800, "meter_buf": 150}, 2, 800, 24),
                                               ({"width": 300, "meter_buf": 50, "audio_sync_offset": 40}, 1, 441, 30),
                                               ({"width": 8192, "meter_buf": 150, "channel_mode": "stereo"}, 2, 7, 50),
                                               ({"width": 1, "meter_buf": 20, "audio_sync_offset": 170}, 1, 9000, 12)])
def test_preview_plan_is_the_same_for_every_struct_size(settings, ch, hop, T):
    """wf_wave_preview_plan (the host walk) gives the same counts and sources for the current config and for the sizes
    before it (without the offset the previous sizes plan with D = 0, as a zero offset does)."""
    from waveform_b200.engine import WfWaveConfig, make_wave_config, preview_wave_plan

    cfg = make_wave_config(settings, channels=ch)
    counts, src = preview_wave_plan(cfg, T, hop)
    assert counts.sum() == len(src) and counts.max() <= cfg.width
    plain = make_wave_config({**settings, "audio_sync_offset": 0}, channels=ch)
    c0, s0 = preview_wave_plan(plain, T, hop)
    for size in (WfWaveConfig.sync_offset_ms.offset, WfWaveConfig.interp_mode.offset):
        old = make_wave_config(settings, channels=ch)
        old.struct_size = size
        c1, s1 = preview_wave_plan(old, T, hop)
        assert np.array_equal(c1, c0) and np.array_equal(s1, s0)
