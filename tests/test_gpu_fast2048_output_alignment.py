"""The N=2048 warp-per-stream kernel writes each dB row with one bulk copy, which needs a 16-byte aligned destination.
An output buffer that is only 4-byte aligned is still served, by the generic kernel, with the same spectra."""
from __future__ import annotations

import pytest

from gpu_common import clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import device_pcm, parity_report

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]


def test_fast2048_unaligned_output_takes_generic_kernel(monkeypatch):
    import torch
    from waveform_b200 import Engine

    set_knobs(monkeypatch, {"WF_TEAM_W": "1"})  # keep the aligned run on the warp-per-stream kernel at this stream count
    S, T, N, B = 300, 4, 2048, 1024
    settings = {"fft_size": N, "window": "hann", "gravity": 0.65}
    pcm = device_pcm(S, 1, T * N, seed=2048)
    res = {}
    for off in (0, 1):  # 0: 256-byte aligned (torch allocation); 1: 4 bytes past it
        eng = Engine(settings, channels=1, max_streams=S)
        buf = torch.full((S * T * B + 4,), float("nan"), device="cuda")
        out = buf[off:off + S * T * B]
        eng.process_raw(pcm.data_ptr(), S, T, N, T * N, T * N, out_db=out.data_ptr())
        torch.cuda.synchronize()
        res[off] = (out.view(S, T, B).cpu().numpy(), eng.last_kernel_name())
    assert res[0][1].startswith("stft2048_fast_kernel"), res[0][1]
    assert not res[1][1].startswith("stft2048_fast_kernel"), res[1][1]
    rep = parity_report(res[1][0], res[0][0])
    assert rep["ok"], rep
