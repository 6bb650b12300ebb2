"""Host-buffer spectrum calls that carry every buffer of wf_batch, staged through device memory in several chunks.

A host batch is copied to the engine's staging buffers and back one chunk of streams at a time, each buffer at its own
per-stream offset, and the per-call peak once after the last chunk.  Such a call must give, bit for bit, what the same
call gives with device buffers on a fresh engine: every output, the carried state and the capture ring.  wf_peak_normalize
stages host rows and a host peak the same way.

Run on an H100:  python -m pytest tests/test_gpu_batch_buffers.py -m gpu -q
"""
from __future__ import annotations

import numpy as np
import pytest

from gpu_common import clean_knobs  # noqa: F401 (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

N, HOP, T, S = 2048, 1024, 48, 1100
SETTINGS = {"fft_size": N, "normalize_volume": True, "volume_target": -12.0, "max_gain": 20.0,
            "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5, "silence_gate": True, "width": 96}


def _chunks(n_streams, pcm_bytes):
    """(streams per chunk, chunks) of a staged call: one chunk per 32 MiB of PCM, at most 16, as wf_process_async splits it."""
    n = min(16, n_streams, max(1, pcm_bytes >> 25))
    per = -(-n_streams // n)
    return per, -(-n_streams // per)


def _inputs(ns, fmt):
    """PCM [S, 1, ns] (int16, or float32 holding the same values * 2^-15), input_rms, skip_mask and frame_seconds."""
    rng = np.random.default_rng(0xB0F + ns)
    x = rng.integers(-12000, 12001, size=(S, 1, ns), dtype=np.int16)
    x[7] = 0                    # a silent stream
    x[S - 1, :, : ns // 2] = 0  # silent, then loud, in the last (short) chunk
    pcm = x if fmt == "s16" else x.astype(np.float32) * np.float32(2.0 ** -15)
    rms = rng.uniform(0.01, 0.5, (S, T)).astype(np.float32)
    skip = (rng.random((S, T)) < 0.1).astype(np.uint8)
    secs = rng.uniform(0.01, 0.03, T).astype(np.float32)
    return pcm, rms, skip, secs


@pytest.mark.parametrize("ring", [False, True], ids=["plain", "ring"])
@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("memory", ["pinned", "pageable"])
def test_host_batch_every_buffer_chunked(memory, fmt, ring):
    """input_rms, skip_mask, frame_seconds and all six outputs at once, in at least three staging chunks with a short last
    one: host buffers equal device buffers bit for bit."""
    import torch
    from waveform_b200 import Engine

    ns = T * HOP if ring else (T - 1) * HOP + N
    pcm, rms, skip, secs = _inputs(ns, fmt)
    per, n = _chunks(S, pcm.nbytes)
    assert n >= 3 and S % per != 0, (per, n)

    dev = Engine(SETTINGS, channels=1, max_streams=S)
    want = dev.process(torch.from_numpy(pcm).cuda(), T, HOP, input_rms=torch.from_numpy(rms).cuda(),
                       skip_mask=torch.from_numpy(skip).cuda(), want_points=True, want_peak=True, want_pixels=True,
                       frame_seconds=secs, pcm_format=fmt, capture_ring=ring)
    torch.cuda.synchronize()

    host = Engine(SETTINGS, channels=1, max_streams=S)
    dch, B, P = host.display_channels, host.bins, host.num_points
    mk = (lambda a: torch.from_numpy(a).pin_memory()) if memory == "pinned" else torch.from_numpy
    x, r, k = mk(pcm), mk(rms), mk(skip)
    got = {"db": mk(np.full((S, T, dch, B), np.nan, np.float32)),
           "points": mk(np.full((S, T, dch, P), np.nan, np.float32)),
           "silent": mk(np.full((S, T), 7, np.uint8)),
           "peak": mk(np.full(T, np.nan, np.float32)),
           "pixels": mk(np.full((S, T, dch, P), np.nan, np.float32)),
           "min": mk(np.full((S, T, 2), np.nan, np.float32))}
    assert x.is_pinned() == (memory == "pinned") and all(v.is_pinned() == x.is_pinned() for v in got.values())
    host.process_raw(x.data_ptr(), S, T, HOP, ns, ns, input_rms=r.data_ptr(), skip_mask=k.data_ptr(),
                     out_db=got["db"].data_ptr(), out_points=got["points"].data_ptr(),
                     out_silent=got["silent"].data_ptr(), out_peak=got["peak"].data_ptr(),
                     out_pixels=got["pixels"].data_ptr(), out_min=got["min"].data_ptr(),
                     frame_seconds=secs.ctypes.data, pcm_format=fmt, capture_ring=ring)

    assert got.keys() == want.keys()
    for key in want:
        a, b = got[key].numpy(), want[key].cpu().numpy()
        assert a.dtype == b.dtype and a.shape == b.shape, key
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), key
    sh, sd = host.get_state(), dev.get_state()
    for key in sd:
        assert np.array_equal(sh[key].view(np.uint8), sd[key].view(np.uint8)), key
    if ring:
        assert np.array_equal(host.get_ring().view(np.uint32), dev.get_ring().view(np.uint32))


def test_peak_normalize_host_buffers():
    """Host rows with a host peak, and device rows with a host peak, equal device rows with a device peak bit for bit."""
    import torch
    from waveform_b200 import Engine

    S_, T_ = 37, 24
    eng = Engine({"fft_size": N}, channels=1, max_streams=1)
    rng = np.random.default_rng(0x9EA)
    db = rng.uniform(-120.0, 0.0, (S_, T_, eng.display_channels, eng.bins)).astype(np.float32)
    peak = rng.uniform(-40.0, 0.0, T_).astype(np.float32)  # some gains clamp at max_gain
    want = torch.from_numpy(db).cuda()
    eng.peak_normalize(want, torch.from_numpy(peak).cuda(), -3.0, 20.0)
    torch.cuda.synchronize()
    want = want.cpu().numpy()
    assert not np.array_equal(want, db)

    rows = db.copy()
    eng.peak_normalize(rows, peak, -3.0, 20.0)  # host rows: staged, and home when the call returns
    assert np.array_equal(rows.view(np.uint32), want.view(np.uint32))

    rows = torch.from_numpy(db).cuda()
    eng.peak_normalize(rows, peak, -3.0, 20.0)
    torch.cuda.synchronize()
    assert np.array_equal(rows.cpu().numpy().view(np.uint32), want.view(np.uint32))
