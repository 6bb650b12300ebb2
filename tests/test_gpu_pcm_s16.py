"""int16 PCM (wf_batch.pcm_format = WF_PCM_S16) in every spectrum kernel family.

A sample v of an int16 batch stands for v * 2^-15, which float32 holds exactly.  So an int16 call has an exact reference:
the float32 call on pcm * 2^-15.  When both take the same kernel (the int16 name is the float32 name + " s16"), every output
and the carried state must match it bit for bit; every int16 case is also held to the float64 restatement of tick_spectrum
(fp64_spectrum.compare), including the calls whose alignment sends them to another family than float32 would take.

Run on an H100:  python -m pytest tests/test_gpu_pcm_s16.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from fp64_spectrum import Fp64Spectrum, compare
from gpu_common import CATALOGUE, assert_bits_equal, clean_knobs, route_id, set_knobs  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

T = 8  # ticks per run, in two calls of 4

ROUTES = [CATALOGUE[k] for k in (
    "fast-2048", "team-2048", "warp2-800", "warp2-1456", "warp2-800-display", "warp2-1024-display", "v3-1024",
    "v3-4096-stereo-display", "v3-4096-mix", "v3-16384", "parity-16384", "wide-4096-display", "wide-32768",
    "fused-256-display", "fused-2048-mix", "smem-800-display", "l2-40000")]


def _signals(N, cc, hop, pad=16):
    """[5, cc, ns] int16, ns rounded up to `pad` samples (so that the stream stride keeps frames 16-byte aligned):
    noise + sines; the same with an all-zero frame (tick 2) and a zero tail; the extremes -32768 / +32767 / -32767;
    digital silence (the gate); a quiet stream (|v| <= 3)."""
    need = (T - 1) * hop + N
    ns = -(-need // pad) * pad
    base = synth_pcm(1, cc, ns, seed=0x516 + N)[0]
    x = np.zeros((5, cc, ns), np.int16)
    x[0] = np.round(base * 32767.0).astype(np.int16)
    x[1] = x[0]
    x[1, :, 2 * hop: 2 * hop + N] = 0
    x[1, :, 6 * hop:] = 0
    rng = np.random.default_rng(N + hop)
    x[2] = rng.choice(np.array([-32768, 32767, -32767, 0], np.int16), size=(cc, ns))
    x[4] = rng.integers(-3, 4, size=(cc, ns), dtype=np.int16)
    return x


def _options(N, all_options, stereo):
    s = {"fft_size": N, "window": "hann", "silence_gate": True}
    if all_options:
        s = {"fft_size": N, "window": "blackman_harris", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0,
             "fast_peaks": True, "normalize_volume": True, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5,
             "silence_gate": True}
    if stereo:
        s["channel_mode"] = "stereo"
    return s


def _run(eng, x, hop, fmt, disp, extras):
    """Two calls of T/2 ticks on device tensors; returns the concatenated outputs (numpy) and the engine's state."""
    import torch

    outs = []
    for a, b in ((0, T // 2), (T // 2, T)):
        kw = {}
        if extras is not None:
            secs, rms, skip = extras
            kw = dict(frame_seconds=secs[a:b], input_rms=torch.from_numpy(rms[:, a:b].copy()).cuda(),
                      skip_mask=torch.from_numpy(skip[:, a:b].copy()).cuda(), want_peak=True)
        xs = torch.from_numpy(np.ascontiguousarray(x[:, :, a * hop:])).cuda()
        outs.append(eng.process(xs, b - a, hop, want_points=disp, want_pixels=disp, pcm_format=fmt, **kw))
    torch.cuda.synchronize()
    got = {k: torch.cat([o[k] for o in outs], dim=0 if k == "peak" else 1).cpu().numpy() for k in outs[0]}
    return got, eng.get_state(), eng.last_kernel_name()


def _check_fp64(settings, cc, x, hop, got, eng, extras, ctx):
    db_min = float(eng.db_min)
    xf = x.astype(np.float32) * np.float32(2.0 ** -15)
    if extras is not None:
        secs, rms, skip = extras
        gvals = np.array([eng.gravity(float(s)) for s in secs], np.float32)
    else:
        rms = skip = None
        gvals = np.float32(eng.gravity(1.0 / 60.0))
    f = Fp64Spectrum(settings, channels=cc)
    for s in range(x.shape[0]):
        f.reset()
        tr = f.run(xf[s], T, hop, gvals, input_rms=None if rms is None else rms[s],
                   skip_mask=None if skip is None else skip[s])
        err, bad_floor = compare(got["db"][s], tr, db_min)
        assert not bad_floor, ("DB_MIN above the flush level", ctx, s)
        assert np.array_equal(got["silent"][s].astype(bool), tr["silent"]), (ctx, s)
        assert err.max() < 1e-6, (err.max(), ctx, s)


def _extras(S, seed):
    rng = np.random.default_rng(seed)
    secs = (1.0 / 60.0 * (0.5 + rng.uniform(size=T))).astype(np.float32)
    rms = (0.02 + 0.3 * rng.uniform(size=(S, T))).astype(np.float32)
    skip = np.zeros((S, T), np.uint8)
    skip[1::2, 5] = 1
    skip[2::3, 2] = 1
    return secs, rms, skip


@pytest.mark.parametrize("all_opt", [False, True], ids=["plain", "all-options"])
@pytest.mark.parametrize("route", ROUTES, ids=[route_id(r) for r in ROUTES])
def test_s16_matches_f32_bit_for_bit(route, all_opt, monkeypatch):
    from waveform_b200 import Engine

    fam, N, cc, stereo, env, disp = route
    set_knobs(monkeypatch, env)
    for hop in sorted({N, (N // 4) & ~7}, reverse=True):     # multiples of 8 samples: both formats' frames 16-byte aligned
        x = _signals(N, cc, hop)
        S = x.shape[0]
        settings = _options(N, all_opt, stereo)
        extras = _extras(S, N + hop) if all_opt else None
        e16 = Engine(settings, channels=cc, max_streams=S)
        e32 = Engine(settings, channels=cc, max_streams=S)
        g16, st16, n16 = _run(e16, x, hop, "s16", disp, extras)
        g32, st32, n32 = _run(e32, x.astype(np.float32) * np.float32(2.0 ** -15), hop, "f32", disp, extras)
        ctx = (fam, N, hop, all_opt, n16)
        assert n32.startswith(fam.split("/")[0] + "<") and (("display" in n32) == fam.endswith("/display")), (ctx, n32)
        assert n16 == n32 + " s16", (n16, n32)
        assert_bits_equal(g16, g32, ctx)
        assert_bits_equal(st16, st32, ctx)
        _check_fp64(settings, cc, x, hop, g16, e16, extras, ctx)


def test_s16_alignment_routes(monkeypatch):
    """hop % 8 == 4 keeps float32 frames 16-byte aligned but not int16 ones: at N=2048 float32 takes the TMA kernel,
    int16 the CTA-per-tick kernel (the next family in routing order), and is still right against float64."""
    from waveform_b200 import Engine

    set_knobs(monkeypatch, {"WF_TEAM_W": "1"})
    N, hop = 2048, 2044
    x = _signals(N, 1, hop)
    settings = _options(N, False, False)
    e16 = Engine(settings, channels=1, max_streams=x.shape[0])
    e32 = Engine(settings, channels=1, max_streams=x.shape[0])
    g16, _, n16 = _run(e16, x, hop, "s16", False, None)
    _, _, n32 = _run(e32, x.astype(np.float32) * np.float32(2.0 ** -15), hop, "f32", False, None)
    assert n32.startswith("stft2048_fast_kernel<"), n32
    assert n16.startswith("stft_v3_kernel<2048,1,") and n16.endswith(" s16"), n16
    _check_fp64(settings, 1, x, hop, g16, e16, None, (N, hop, n16))


def _raw_call(eng, pcm_ptr, S, n_frames, hop, ss, cs, out_db, out_silent, fmt):
    eng.process_raw(pcm_ptr, S, n_frames, hop, ss, cs, out_db=out_db, out_silent=out_silent, pcm_format=fmt)


@pytest.mark.parametrize("N,cc,stereo", [(800, 1, False), (2048, 1, False), (800, 2, True), (2048, 2, False)])
def test_s16_buffer_kinds(N, cc, stereo):
    """Device, pageable host and wf_host_alloc (zero-copy) buffers give the same bits, for live ticks (1 stream x 1
    frame) and a few calls in a row."""
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import load_library

    settings = _options(N, False, stereo)
    L = load_library()
    rng = np.random.default_rng(N * cc)
    frames = [rng.integers(-32768, 32768, size=(1, cc, N), dtype=np.int16) for _ in range(3)]
    frames[1][:] = 0  # a silent tick between two loud ones
    ref_eng = Engine(settings, channels=cc, max_streams=1)
    ref = [ref_eng.process(torch.from_numpy(f).cuda(), 1, N, pcm_format="s16") for f in frames]
    torch.cuda.synchronize()
    ref = [{k: v.cpu().numpy() for k, v in r.items()} for r in ref]
    f32 = Engine(settings, channels=cc, max_streams=1)
    want = [f32.process(f.astype(np.float32) * np.float32(2.0 ** -15), 1, N) for f in frames]
    for r, w in zip(ref, want):
        assert_bits_equal(r, w, ("device vs float32", N, cc))

    host = Engine(settings, channels=cc, max_streams=1)
    for f, r in zip(frames, ref):
        assert_bits_equal(host.process(f, 1, N, pcm_format="s16"), r, ("pageable", N, cc))

    mapped = Engine(settings, channels=cc, max_streams=1)
    dch, B = mapped.display_channels, mapped.bins
    pin, pout, psil = L.wf_host_alloc(cc * N * 2), L.wf_host_alloc(dch * B * 4), L.wf_host_alloc(16)
    assert pin and pout and psil
    try:
        for f, r in zip(frames, ref):
            C.memmove(pin, f.ctypes.data, f.nbytes)
            _raw_call(mapped, pin, 1, 1, N, cc * N, N, pout, psil, "s16")
            db = np.frombuffer((C.c_float * (dch * B)).from_address(pout), np.float32).reshape(r["db"].shape).copy()
            sil = np.frombuffer((C.c_uint8 * 1).from_address(psil), np.uint8).reshape(r["silent"].shape).copy()
            assert_bits_equal({"db": db, "silent": sil}, r, ("wf_host_alloc", N, cc))
        assert mapped.last_kernel_name().endswith(" s16")
    finally:
        for q in (pin, pout, psil):
            L.wf_host_free(q)


def test_s16_pinned_host_chunked():
    """A pinned host batch big enough to be staged in several chunks (64 MiB of int16 PCM) equals the device call."""
    import torch
    from waveform_b200 import Engine

    N, S, T_ = 2048, 1024, 16
    ns = T_ * N
    x = torch.randint(-32768, 32768, (S, 1, ns), dtype=torch.int16)
    x[5, :, 3 * N: 4 * N] = 0
    xp = x.pin_memory()
    assert xp.numel() * 2 >= 2 << 25  # at least two staging chunks
    settings = {"fft_size": N, "silence_gate": True}
    dev = Engine(settings, channels=1, max_streams=S)
    want = dev.process(xp.cuda(), T_, N, pcm_format="s16")
    torch.cuda.synchronize()
    host = Engine(settings, channels=1, max_streams=S)
    out_db = torch.empty((S, T_, 1, N // 2), dtype=torch.float32).pin_memory()
    out_sil = torch.empty((S, T_), dtype=torch.uint8).pin_memory()
    host.process_raw(xp.data_ptr(), S, T_, N, ns, ns, out_db=out_db.data_ptr(), out_silent=out_sil.data_ptr(),
                     pcm_format="s16")
    assert host.last_kernel_name() == dev.last_kernel_name()
    assert torch.equal(out_db.view(torch.int32), want["db"].cpu().view(torch.int32))
    assert torch.equal(out_sil, want["silent"].cpu())
    assert_bits_equal(host.get_state(), dev.get_state(), "pinned vs device state")


def test_s16_side_stream_after_busy_producer():
    """A device int16 call on the caller's side stream runs after the kernel that wrote its PCM on that stream."""
    import torch
    from waveform_b200 import Engine

    N, S = 2048, 264
    src = torch.randint(-32768, 32768, (S, 1, 4 * N), dtype=torch.int16)
    ref_eng = Engine({"fft_size": N}, channels=1, max_streams=S)
    want = ref_eng.process(src.cuda(), 4, N, pcm_format="s16")
    torch.cuda.synchronize()
    eng = Engine({"fft_size": N}, channels=1, max_streams=S)
    side = torch.cuda.Stream()
    src_dev = src.cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        a = torch.randn(4096, 4096, device="cuda")
        dst = torch.zeros((S, 1, 4 * N), dtype=torch.int16, device="cuda")
        for _ in range(16):
            b = a @ a                 # keeps the side stream busy before the PCM exists
        dst.copy_(src_dev)
        got = eng.process(dst, 4, N, pcm_format="s16")
    side.synchronize()
    assert torch.equal(got["db"].view(torch.int32), want["db"].view(torch.int32))


def _batch(eng_pcm, S, n_frames, hop, ns, out_db, fmt, struct_size=None):
    from waveform_b200.engine import WfBatch

    b = WfBatch()
    b.struct_size = C.sizeof(WfBatch) if struct_size is None else struct_size
    b.n_streams, b.n_frames, b.hop, b.seconds = S, n_frames, hop, 1.0 / 60.0
    b.pcm, b.stream_stride, b.channel_stride = eng_pcm, ns, ns
    b.out_db = out_db
    b.pcm_format = fmt
    return b


def test_s16_abi_and_errors():
    """The previous struct_size reads as float32 and gives the current-size float32 result; any other size is
    WF_ERR_ABI; an unknown pcm_format and an odd int16 address are WF_ERR_INVALID_ARG."""
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import WF_ERR_ABI, WF_ERR_INVALID_ARG, WfBatch

    N, S = 1024, 3
    ns = 2 * N
    eng = Engine({"fft_size": N}, channels=1, max_streams=S)
    L = eng.L
    xf = torch.from_numpy(synth_pcm(S, 1, ns)).cuda()
    out = torch.empty((S, 2, 1, N // 2), device="cuda")
    prev = WfBatch.pcm_format.offset
    assert prev == C.sizeof(WfBatch) - 8
    b_old = _batch(xf.data_ptr(), S, 2, N, ns, out.data_ptr(), 0, struct_size=prev)
    b_old.pcm_format = 1          # beyond the previous struct: must not be read
    assert L.wf_process(eng.h, C.byref(b_old)) == 0
    old = out.clone()
    cur = Engine({"fft_size": N}, channels=1, max_streams=S)
    assert L.wf_process(cur.h, C.byref(_batch(xf.data_ptr(), S, 2, N, ns, out.data_ptr(), 0))) == 0
    assert torch.equal(old.view(torch.int32), out.view(torch.int32))
    assert not eng.last_kernel_name().endswith(" s16")
    for size in (prev - 8, prev + 4, C.sizeof(WfBatch) + 8, 0):
        assert L.wf_process(eng.h, C.byref(_batch(xf.data_ptr(), S, 2, N, ns, out.data_ptr(), 0, struct_size=size))) == \
            WF_ERR_ABI, size
    x16 = torch.zeros(S * ns + 8, dtype=torch.int16, device="cuda")
    assert L.wf_process(eng.h, C.byref(_batch(x16.data_ptr(), S, 2, N, ns, out.data_ptr(), 2))) == WF_ERR_INVALID_ARG
    assert b"pcm_format" in L.wf_last_error(eng.h)
    assert L.wf_process(eng.h, C.byref(_batch(x16.data_ptr(), S, 2, N, ns, out.data_ptr(), -1))) == WF_ERR_INVALID_ARG
    assert L.wf_process(eng.h, C.byref(_batch(x16.data_ptr() + 1, S, 2, N, ns, out.data_ptr(), 1))) == WF_ERR_INVALID_ARG
    assert b"aligned" in L.wf_last_error(eng.h)
    assert L.wf_process(eng.h, C.byref(_batch(x16.data_ptr() + 2, S, 2, N, ns, out.data_ptr(), 1))) == 0


def test_numpy_int16_without_keyword_stays_unscaled():
    """The default keeps today's behaviour: an int16 numpy array is converted to float32 as it is, without 2^-15."""
    from waveform_b200 import Engine

    N = 1024
    x = np.random.default_rng(1).integers(-200, 200, size=(2, 1, 2 * N), dtype=np.int16)
    a = Engine({"fft_size": N}, channels=1, max_streams=2).process(x, 2, N)
    b = Engine({"fft_size": N}, channels=1, max_streams=2).process(x.astype(np.float32), 2, N)
    assert_bits_equal(a, b, "int16 numpy without pcm_format")
    s = Engine({"fft_size": N}, channels=1, max_streams=2).process(x, 2, N, pcm_format="s16")
    assert not np.array_equal(a["db"], s["db"])
    with pytest.raises(ValueError):
        Engine({"fft_size": N}, channels=1, max_streams=2).process(x.astype(np.float32), 2, N, pcm_format="s16")
