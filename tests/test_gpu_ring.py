"""Capture-ring calls (wf_batch.capture_ring = 1) in every spectrum kernel family.

A ring call hands the engine only the samples captured since the previous call; frame t of stream s is the newest fft_size
samples of ring[s] ++ new[0 .. (t+1)*hop), and the ring starts as fft_size zeros.  So a run of ring calls has an exact
reference: plain calls on the contiguous zeros(N) ++ samples, each starting where the matching ring call's first frame
does.  Every output, the carried state and the ring itself must match bit for bit, and the kernel is the plain call's with
" ring" appended.

Run on an H100:  python -m pytest tests/test_gpu_ring.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from gpu_common import CATALOGUE, assert_bits_equal, clean_knobs, route_id, set_knobs  # noqa: F401 (fixture)
from helpers import synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

# (route, streams, start of the last call's kernel name)
ROUTES = [(*CATALOGUE[k], S, name) for k, S, name in [
    ("fast-2048", 5, "stft2048_fast_kernel<12,1,1,1> grid 5 x 8 warps"),
    ("fast-2048-split", 300, "stft2048_fast_kernel<12,1,1,1> grid 132 x 8 warps"),
    ("team-2048", 5, "stft2048_team_kernel<4,1> grid 5 x 4 teams"),
    ("warp2-800", 5, "stft_warp2_kernel<20,20> N=800"),
    ("warp2-1024-display", 5, "stft_warp2_kernel<16,32,display> N=1024"),
    ("v3-1024", 5, "stft_v3_kernel<1024,1,"),
    ("v3-4096-mix", 5, "stft_v3_kernel<4096,2,"),
    ("v3-4096-stereo-display", 5, "stft_v3_kernel<4096,2,"),
    ("parity-16384", 3, "stft16384_parity_kernel<1> 3 clusters of 2"),
    ("wide-32768", 2, "stft_wide_kernel<32768,1,2>"),
    ("fused-256-display", 5, "stft_fused_kernel<256,1>"),
    ("smem-800-display", 5, "stft_anyn_kernel<1> N=800"),
    ("l2-40000", 2, "stft_anyn_kernel<1> N=40000"),
]]


def _calls(N):
    """(n_frames, hop) of successive calls: head frames beyond the call (k > T), k < T, hop = N, hop > N, a smaller hop.
    Every hop is a multiple of 8 samples, so that the plain calls' slices keep the ring calls' alignment facts."""
    a = max(16, (N * 2 // 5) // 16 * 16)
    b = max(8, (a // 2) // 8 * 8)
    return [(1, a), (4, a), (2, N), (1, N + a), (6, b)]


def _signal(S, cc, n, seed, s16):
    """[S, cc, n] noise + sines with a digital-silence stretch (the gate) on stream 1."""
    x = synth_pcm(S, cc, n, seed=seed)
    if S > 1:
        x[1, :, n // 3: n // 3 + n // 4] = 0.0
    if s16:
        return np.round(x * 32767.0).astype(np.int16)
    return x.astype(np.float32)


def _run_pair(settings, cc, S, calls, x, fmt, disp, feed):
    """Ring calls on one engine, plain calls over zeros(N) ++ x on another; `feed(eng, pcm, T, hop, ring)` makes one call
    and returns its outputs as numpy.  Asserts per call that outputs, names, state and ring agree."""
    from waveform_b200 import Engine

    ring_eng = Engine(settings, channels=cc, max_streams=S)
    plain_eng = Engine(settings, channels=cc, max_streams=S)
    N = ring_eng.fft_size
    full = np.concatenate([np.zeros((S, cc, N), x.dtype), x], axis=2)
    pos = 0
    for T_, hop in calls:
        new = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
        plain = np.ascontiguousarray(full[:, :, pos + hop: pos + hop + (T_ - 1) * hop + N])
        got = feed(ring_eng, new, T_, hop, True)
        want = feed(plain_eng, plain, T_, hop, False)
        ctx = (settings, fmt, T_, hop)
        assert_bits_equal(got, want, ctx)
        assert ring_eng.last_kernel_name() == plain_eng.last_kernel_name() + " ring", ctx
        assert_bits_equal(ring_eng.get_state(), plain_eng.get_state(), ctx)
        pos += T_ * hop
        want_ring = full[:, :, pos: pos + N].astype(np.float32)
        if x.dtype == np.int16:
            want_ring *= np.float32(2.0 ** -15)
        assert np.array_equal(ring_eng.get_ring(), want_ring), ctx
    return ring_eng


def _device_feed(disp, fmt):
    def feed(eng, pcm, T_, hop, ring):
        import torch

        o = eng.process(torch.from_numpy(pcm).cuda(), T_, hop, want_points=disp, want_pixels=disp, want_peak=True,
                        pcm_format=fmt, capture_ring=ring)
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in o.items()}
    return feed


def _options(N, stereo):
    s = {"fft_size": N, "window": "hann", "silence_gate": True}
    if stereo:
        s["channel_mode"] = "stereo"
    return s


def _host_feed(disp, fmt):
    def feed(eng, pcm, T_, hop, ring):
        return dict(eng.process(pcm, T_, hop, want_points=disp, want_pixels=disp, want_peak=True, pcm_format=fmt,
                                capture_ring=ring))
    return feed


@pytest.mark.parametrize("buf", ["device", "host"])
@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("route", ROUTES, ids=[route_id(r) for r in ROUTES])
def test_ring_matches_plain_bit_for_bit(route, fmt, buf, monkeypatch):
    fam, N, cc, stereo, env, disp, S, name = route
    set_knobs(monkeypatch, env)
    calls = _calls(N)
    x = _signal(S, cc, sum(t * h for t, h in calls), 0x5150 + N, fmt == "s16")
    feed = (_device_feed if buf == "device" else _host_feed)(disp, fmt)
    eng = _run_pair(_options(N, stereo), cc, S, calls, x, fmt, disp, feed)
    got = eng.last_kernel_name()
    assert got.startswith(name), (got, fam)
    assert got.endswith(" s16 ring" if fmt == "s16" else " ring"), got


@pytest.mark.parametrize("fmt", ["f32", "s16"])
@pytest.mark.parametrize("N,cc,stereo", [(2048, 1, False), (4096, 2, True)])
def test_ring_host_buffers(N, cc, stereo, fmt):
    """Pageable host buffers and wf_host_alloc (zero-copy) live ticks give the device path's bits."""
    from waveform_b200 import Engine
    from waveform_b200.engine import load_library

    settings = _options(N, stereo)
    calls = [(1, 800), (1, 800), (2, N), (1, N + 800), (3, 400)]
    x = _signal(1, cc, sum(t * h for t, h in calls), 7 + N, fmt == "s16")

    def host_feed(eng, pcm, T_, hop, ring):
        o = eng.process(pcm, T_, hop, want_peak=True, pcm_format=fmt, capture_ring=ring)
        return dict(o)
    _run_pair(settings, cc, 1, calls, x, fmt, False, host_feed)

    # zero-copy: the live adapter's buffers, reused every tick
    L = load_library()
    dev = Engine(settings, channels=cc, max_streams=1)
    mapped = Engine(settings, channels=cc, max_streams=1)
    dch, B, es = dev.display_channels, dev.bins, x.dtype.itemsize
    cap = max(t * h for t, h in calls)
    pin, pout, psil = L.wf_host_alloc(cc * cap * es), L.wf_host_alloc(3 * dch * B * 4), L.wf_host_alloc(16)
    assert pin and pout and psil
    try:
        pos = 0
        for T_, hop in calls:
            new = np.ascontiguousarray(x[:, :, pos: pos + T_ * hop])
            pos += T_ * hop
            import torch
            o = dev.process(torch.from_numpy(new).cuda(), T_, hop, pcm_format=fmt, capture_ring=True)
            torch.cuda.synchronize()
            want = {k: v.cpu().numpy() for k, v in o.items()}
            C.memmove(pin, new.ctypes.data, new.nbytes)
            mapped.process_raw(pin, 1, T_, hop, cc * T_ * hop, T_ * hop, out_db=pout, out_silent=psil, pcm_format=fmt,
                               capture_ring=True)
            db = np.frombuffer((C.c_float * (T_ * dch * B)).from_address(pout), np.float32).reshape(want["db"].shape)
            sil = np.frombuffer((C.c_uint8 * T_).from_address(psil), np.uint8).reshape(want["silent"].shape)
            assert np.array_equal(db.view(np.uint32), want["db"].view(np.uint32)), (N, fmt, T_, hop)
            assert np.array_equal(sil, want["silent"]), (N, fmt, T_, hop)
            assert mapped.last_kernel_name() == dev.last_kernel_name()
        assert np.array_equal(mapped.get_ring(), dev.get_ring())
    finally:
        for q in (pin, pout, psil):
            L.wf_host_free(q)


@pytest.mark.parametrize("fmt", ["f32", "s16"])
def test_ring_pinned_chunks(fmt):
    """A pinned host batch large enough for several staging chunks: each chunk's splice runs after its own copy."""
    import torch
    from waveform_b200 import Engine

    S, N, hop = 512, 2048, 1024
    T_ = 32 if fmt == "f32" else 64
    es = 4 if fmt == "f32" else 2
    assert S * T_ * hop * es >= 2 << 25  # at least two staging chunks
    settings = {"fft_size": N, "silence_gate": True}
    x = torch.from_numpy(_signal(S, 1, 2 * T_ * hop, 11, fmt == "s16"))
    dev = Engine(settings, channels=1, max_streams=S)
    host = Engine(settings, channels=1, max_streams=S)
    for i in range(2):
        new = x[:, :, i * T_ * hop: (i + 1) * T_ * hop].contiguous()
        want = dev.process(new.cuda(), T_, hop, pcm_format=fmt, capture_ring=True)
        torch.cuda.synchronize()
        xp = new.pin_memory()
        out_db = torch.empty((S, T_, 1, N // 2), dtype=torch.float32).pin_memory()
        out_sil = torch.empty((S, T_), dtype=torch.uint8).pin_memory()
        host.process_raw(xp.data_ptr(), S, T_, hop, T_ * hop, T_ * hop, out_db=out_db.data_ptr(),
                         out_silent=out_sil.data_ptr(), pcm_format=fmt, capture_ring=True)
        assert host.last_kernel_name().endswith(" ring")  # per chunk: fewer streams, possibly another team size
        assert torch.equal(out_db.view(torch.int32), want["db"].cpu().view(torch.int32))
        assert torch.equal(out_sil, want["silent"].cpu())
    assert np.array_equal(host.get_ring(), dev.get_ring())


def test_ring_slot_ranges_and_reset():
    """A call on slots [a, a+b) leaves the other slots' rings and states alone; wf_reset_state keeps the rings."""
    import torch
    from waveform_b200 import Engine

    N, S = 2048, 8
    eng = Engine({"fft_size": N}, channels=1, max_streams=S)
    x = _signal(S, 1, 4 * 800, 3, False)
    eng.process(torch.from_numpy(x).cuda(), 4, 800, capture_ring=True)
    torch.cuda.synchronize()
    ring0, state0 = eng.get_ring(), eng.get_state()
    y = _signal(3, 1, 2 * 512, 4, False)
    eng.process(torch.from_numpy(y).cuda(), 2, 512, first_stream=2, capture_ring=True)
    torch.cuda.synchronize()
    ring1, state1 = eng.get_ring(), eng.get_state()
    others = [0, 1, 5, 6, 7]
    assert np.array_equal(ring1[others], ring0[others])
    for k in state0:
        assert np.array_equal(state1[k][others], state0[k][others]), k
    want = np.concatenate([ring0[2:5], y], axis=2)[:, :, -N:]
    assert np.array_equal(ring1[2:5], want)
    eng.reset_state()
    assert np.array_equal(eng.get_ring(), ring1)
    assert eng.get_ring(3, 2).shape == (2, 1, N)


def test_ring_priming():
    """set_ring with the N samples before a cut, then ring calls, equals one plain call over the uncut signal; a float
    ring followed by an int16 call equals the int16 plain call on the rounded ring."""
    import torch
    from waveform_b200 import Engine

    N, hop, T_ = 2048, 512, 12
    settings = {"fft_size": N, "silence_gate": True}
    x = _signal(2, 1, N + T_ * hop, 21, False)
    plain = Engine(settings, channels=1, max_streams=2)
    want = plain.process(torch.from_numpy(x[:, :, hop:]).contiguous().cuda(), T_, hop)
    ring = Engine(settings, channels=1, max_streams=2)
    ring.set_ring(x[:, :, :N])
    got = [ring.process(torch.from_numpy(x[:, :, N + i * hop: N + (i + 4) * hop]).contiguous().cuda(), 4, hop,
                        capture_ring=True) for i in range(0, T_, 4)]
    torch.cuda.synchronize()
    db = torch.cat([g["db"] for g in got], dim=1)
    assert torch.equal(db.view(torch.int32), want["db"].view(torch.int32))
    assert np.array_equal(ring.get_ring(), x[:, :, -N:])

    # a float ring (not representable in int16) under an int16 call: the call sees lrintf(x * 32768), saturated
    prime = (1.2 * _signal(2, 1, N, 22, False)).astype(np.float32)
    y = np.round(_signal(2, 1, 3 * hop, 23, False) * 32767).astype(np.int16)
    rounded = np.clip(np.rint(prime.astype(np.float64) * 32768.0), -32768, 32767).astype(np.int16)
    s16 = Engine(settings, channels=1, max_streams=2)
    s16.set_ring(prime)
    got = s16.process(torch.from_numpy(y).cuda(), 3, hop, pcm_format="s16", capture_ring=True)
    ref = Engine(settings, channels=1, max_streams=2)
    full = np.concatenate([rounded, y], axis=2)
    want = ref.process(torch.from_numpy(full[:, :, hop:]).contiguous().cuda(), 3, hop, pcm_format="s16")
    torch.cuda.synchronize()
    assert torch.equal(got["db"].view(torch.int32), want["db"].view(torch.int32))
    assert np.array_equal(s16.get_ring(), full[:, :, -N:].astype(np.float32) * np.float32(2.0 ** -15))


def test_ring_launches_and_errors():
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import WfError

    eng = Engine({"fft_size": 2048}, channels=1, max_streams=2)
    x = torch.zeros((2, 1, 2048), device="cuda")
    eng.process(x, 1, 800)
    n0 = eng.launch_count
    eng.process(x[:, :, :1600].contiguous(), 2, 800, capture_ring=True)
    torch.cuda.synchronize()
    assert eng.launch_count - n0 == 2  # the splice and the spectrum kernel
    with pytest.raises(WfError):
        eng.get_ring(1, 2)
    with pytest.raises(WfError):
        eng.set_ring(np.zeros((3, 1, 2048), np.float32))
    with pytest.raises(ValueError):
        eng.set_ring(np.zeros((1, 1, 1024), np.float32))
    with pytest.raises(ValueError):  # fewer than n_frames * hop samples
        eng.process(x[:, :, :1000].contiguous(), 2, 800, capture_ring=True)
    L = eng.L
    assert L.wf_get_ring(eng.h, 0, 1, None) != 0
    assert L.wf_set_ring(eng.h, -1, 1, None) != 0


def test_ring_abi_sizes():
    """capture_ring fills the previous struct's tail padding, so the previous header's size is the current one: only the
    WF_CAPTURE_RING pattern makes a ring call, and any other value there (what an older caller's padding may hold) is a
    plain call.  The size ending before pcm_format is a plain float call whatever lies beyond it; other sizes are
    WF_ERR_ABI."""
    import torch
    from waveform_b200 import Engine
    from waveform_b200.engine import CAPTURE_RING, WF_ERR_ABI, WfBatch

    N, S, T_ = 1024, 2, 2
    x = torch.from_numpy(_signal(S, 1, (T_ - 1) * N + N, 5, False)).cuda()
    out = torch.empty((S, T_, 1, N // 2), device="cuda")

    def call(eng, size, ring_value, fmt=0):
        b = WfBatch()
        b.struct_size = size
        b.n_streams, b.n_frames, b.hop, b.seconds = S, T_, N, 1.0 / 60.0
        b.pcm, b.stream_stride, b.channel_stride = x.data_ptr(), T_ * N, T_ * N
        b.out_db = out.data_ptr()
        b.pcm_format = fmt
        b.capture_ring = ring_value
        rc = eng.L.wf_process(eng.h, C.byref(b))
        return rc, out.clone()

    ref = Engine({"fft_size": N}, channels=1, max_streams=S)
    rc, want = call(ref, C.sizeof(WfBatch), 0)
    assert rc == 0 and not ref.last_kernel_name().endswith(" ring")
    for value in (1, 0xFFFFFFFF, 0x12345678, CAPTURE_RING ^ 1):  # older callers' padding: plain calls
        e = Engine({"fft_size": N}, channels=1, max_streams=S)
        rc, got = call(e, C.sizeof(WfBatch), value)
        assert rc == 0 and torch.equal(got.view(torch.int32), want.view(torch.int32)), hex(value)
        assert not e.last_kernel_name().endswith(" ring")
    e = Engine({"fft_size": N}, channels=1, max_streams=S)
    rc, got = call(e, WfBatch.pcm_format.offset, CAPTURE_RING, fmt=1)  # beyond the struct: neither is read
    assert rc == 0 and torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert e.last_kernel_name() == ref.last_kernel_name()
    e = Engine({"fft_size": N}, channels=1, max_streams=S)
    rc, _ = call(e, C.sizeof(WfBatch), CAPTURE_RING)
    assert rc == 0 and e.last_kernel_name() == ref.last_kernel_name() + " ring"
    for size in (WfBatch.pcm_format.offset + 4, C.sizeof(WfBatch) + 8):
        assert call(e, size, CAPTURE_RING)[0] == WF_ERR_ABI, size


REF_CASES = [  # (id, settings, channels, packets of (n_frames, hop) per call)
    ("plugin-default-800", {"fft_size": 800, "window": "blackman", "temporal_smoothing": "tv_exp_moving_avg"}, 1,
     [(1, 800)] * 24),
    ("2048-hop800-gate", {"fft_size": 2048, "window": "hann", "silence_gate": True}, 1, [(1, 800)] * 12 + [(4, 800)] * 3),
    ("4096-stereo-bh", {"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2,
     [(1, 800)] * 8 + [(3, 800)] * 3),
]


@pytest.mark.parametrize("case", REF_CASES, ids=[c[0] for c in REF_CASES])
def test_ring_against_the_plugin(case):
    """Ring calls, packet by packet from the first tick, against the compiled plugin fed the same packets: the spectra
    meet parity_report's criterion and the silent flags are identical."""
    import torch
    from helpers import parity_report
    from oracle import refbind
    from waveform_b200 import Engine

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    _, settings, cc, calls = case
    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=0x2E6 + cc)[0]
    x[:, total // 4: total // 4 + 3 * 800] = 0.0   # a silence stretch: the gate and m_last_silent
    x[:, total // 2: total // 2 + 800] *= 1e-4
    eng = Engine(settings, channels=cc, max_streams=1)
    ref = refbind.RefSource(settings, channels=cc)
    dch = ref.display_channels
    got_db, got_sil, want_db, want_sil = [], [], [], []
    pos = 0
    for T_, hop in calls:
        new = torch.from_numpy(np.ascontiguousarray(x[None, :, pos: pos + T_ * hop])).cuda()
        o = eng.process(new, T_, hop, seconds=1.0 / 60.0, capture_ring=True)
        torch.cuda.synchronize()
        got_db.append(o["db"][0].cpu().numpy())
        got_sil.append(o["silent"][0].cpu().numpy())
        for t in range(T_):
            seg = x[:, pos + t * hop: pos + (t + 1) * hop]
            ref.advance(hop / ref.sample_rate)
            ref.push(seg[0], seg[1] if cc == 2 else None)
            ref.tick(1.0 / 60.0)
            want_db.append(np.stack([ref.decibels(c) for c in range(dch)]))
            want_sil.append(1 if ref.last_silent else 0)
        pos += T_ * hop
    got_db, want_db = np.concatenate(got_db), np.stack(want_db)
    rep = parity_report(got_db, want_db, db_min=float(eng.db_min))
    assert rep["ok"], rep
    assert np.array_equal(np.concatenate(got_sil), np.array(want_sil, np.uint8))
    assert eng.last_kernel_name().endswith(" ring")
