"""int16 PCM (pcm_format = WF_PCM_S16) in the level meter, the RMS feed and the waveform.

A sample v of an int16 batch stands for v * 2^-15, which float32 holds exactly.  So every int16 call has an exact reference:
the float32 call on pcm * 2^-15, made on a second engine with the same config.  Both take the same path (the alignment
facts are stated in samples), so every output must match it bit for bit, and so must the carried state: the ring, the
one-pass partials, m_meter_buf and the flags of the meter, the scrolling buffers and flags of the waveform.  A third call
with the same float32 input on both engines shows the state: it reads the ring and partials, continues the EMA, and (after a
reset) depends on the flags.  The float paths are tied to the compiled reference by test_meter.py, test_wave.py and
test_display_modes.py, so bit identity ties the int16 paths to it too.

Run on an H100:  python -m pytest tests/test_gpu_meter_wave_s16.py -m gpu -q
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from gpu_common import assert_bits_equal, clean_knobs, set_knobs, to_host  # noqa: F401 (fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

SCALE = np.float32(2.0 ** -15)


def _signals(S, cc, ns, seed, zero_ticks=None):
    """[S, cc, ns] int16, cycling over: noise; the same with an all-zero stretch; the extremes -32768 / +32767 / -32767;
    digital silence; a quiet stream (|v| <= 3)."""
    rng = np.random.default_rng(seed)
    x = np.zeros((S, cc, ns), np.int16)
    for s in range(S):
        k = s % 5
        if k in (0, 1):
            x[s] = rng.integers(-20000, 20001, size=(cc, ns), dtype=np.int16)
            if k == 1:
                a, b = zero_ticks if zero_ticks else (ns // 4, ns // 2)
                x[s, :, a:b] = 0
        elif k == 2:
            x[s] = rng.choice(np.array([-32768, 32767, -32767, 0], np.int16), size=(cc, ns))
        elif k == 4:
            x[s] = rng.integers(-3, 4, size=(cc, ns), dtype=np.int16)
    return x


def _f32(x):
    return x.astype(np.float32) * SCALE


def _dev(x, offset=0):
    """x as a contiguous CUDA tensor whose data starts `offset` samples past an aligned allocation."""
    import torch

    flat = torch.zeros(x.size + offset + 8, dtype=torch.from_numpy(x[:0]).dtype, device="cuda")
    view = flat[offset: offset + x.size].view(x.shape)
    view.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    return view


# ---- level meter ----------------------------------------------------------------------------------------------------
METER_MODES = {"peak": {"rms_mode": False}, "rms": {"rms_mode": True}, "feed": None}
# path: (hop, WF_METER_FUSED, extra samples per row (stride % 4 != 0), pcm offset in samples, launches per call)
METER_PATHS = {
    "one-pass": (800, "1", 0, 0, 1),
    "three-kernel-hop441": (441, "1", 0, 0, 3),
    "three-kernel-unfused": (800, "0", 0, 0, 3),
    "scalar-stride": (800, "1", 2, 0, 3),
    "scalar-offset1": (800, "1", 0, 1, 3),
    "scalar-offset3": (441, "1", 0, 3, 3),
}


def _meter_pair(mode, cc, S, settings_extra=None):
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    base = METER_MODES[mode]
    settings = {} if base is None else {"meter_buf": 150, **base}
    settings.update(settings_extra or {})
    kw = dict(channels=cc, max_streams=S, mode=METER_INPUT_RMS if base is None else None)
    return MeterEngine(settings, **kw), MeterEngine(settings, **kw)


def _meter_call(eng, x, T, hop, fmt, offset, seconds, want_pixels):
    before = eng.launch_count
    out = eng.process(_dev(x, offset), T, hop, pcm_format=fmt, seconds=seconds, want_pixels=want_pixels)
    import torch

    torch.cuda.synchronize()
    return to_host(out), eng.launch_count - before


@pytest.mark.parametrize("opts", ["plain", "fastpeaks-tvexp", "reset"])
@pytest.mark.parametrize("path", list(METER_PATHS))
@pytest.mark.parametrize("cc", [1, 2])
@pytest.mark.parametrize("mode", list(METER_MODES))
def test_meter_s16_matches_f32_bit_for_bit(mode, cc, path, opts, monkeypatch):
    hop, fused, extra, offset, launches = METER_PATHS[path]
    set_knobs(monkeypatch, {"WF_METER_FUSED": fused})
    S, T = 5, 12 if mode != "feed" else 16
    settings = {"fast_peaks": True, "temporal_smoothing": "tv_exp_moving_avg"} if opts == "fastpeaks-tvexp" else None
    e16, e32 = _meter_pair(mode, cc, S, settings)
    want_pixels = mode != "feed"
    ns = 2 * T * hop + extra
    x = _signals(S, cc, ns, seed=hop * 10 + cc, zero_ticks=(T * hop // 2, T * hop + hop))
    secs = (1.0 / 60.0, 1.0 / 45.0)
    for k in range(2):
        xs = np.ascontiguousarray(x[:, :, k * T * hop: k * T * hop + T * hop + extra])
        g16, n16 = _meter_call(e16, xs, T, hop, "s16", offset, secs[k], want_pixels)
        g32, n32 = _meter_call(e32, _f32(xs), T, hop, "f32", offset, secs[k], want_pixels)
        ctx = (mode, cc, path, opts, k)
        assert_bits_equal(g16, g32, ctx)
        assert n16 == n32 == launches, (n16, n32, ctx)
        if opts == "reset" and k == 0:
            for e in (e16, e32):
                # PEAK / RMS: stream 3 is digital silence, already silent, and its flag keeps the reset from touching it
                e.reset(1, 3)
    # the carried state: one more call with the same float32 input on both engines
    x3 = _f32(_signals(S, cc, T * hop + extra, seed=7))
    g16, _ = _meter_call(e16, x3, T, hop, "f32", offset, secs[0], want_pixels)
    g32, _ = _meter_call(e32, x3, T, hop, "f32", offset, secs[0], want_pixels)
    assert_bits_equal(g16, g32, (mode, cc, path, opts, "state"))


def test_meter_formats_alternated_on_one_engine():
    """S16, F32, S16 on one engine give what three F32 calls give (ring and partials hold float either way)."""
    for mode in ("rms", "feed"):
        mixed, ref = _meter_pair(mode, 2, 5)
        hop, T = 800, 16
        x = _signals(5, 2, 3 * T * hop, seed=3)
        for k, fmt in enumerate(("s16", "f32", "s16")):
            xs = np.ascontiguousarray(x[:, :, k * T * hop: (k + 1) * T * hop])
            a, _ = _meter_call(mixed, xs if fmt == "s16" else _f32(xs), T, hop, fmt, 0, 1 / 60, mode != "feed")
            b, _ = _meter_call(ref, _f32(xs), T, hop, "f32", 0, 1 / 60, mode != "feed")
            assert_bits_equal(a, b, (mode, k, fmt))


def test_meter_buffer_kinds():
    """Device tensors, pinned host and pageable numpy int16 buffers give the same bits (host buffers are staged)."""
    import torch

    for mode, cc in (("rms", 2), ("peak", 1), ("feed", 2)):
        S, T, hop = 5, 12, 800
        x = _signals(S, cc, 2 * T * hop, seed=11)
        engines = [_meter_pair(mode, cc, S)[0] for _ in range(3)]
        for k in range(2):
            xs = np.ascontiguousarray(x[:, :, k * T * hop: (k + 1) * T * hop])
            dev, _ = _meter_call(engines[0], xs, T, hop, "s16", 0, 1 / 60, mode != "feed")
            pinned = torch.from_numpy(xs).pin_memory()
            pin = engines[1].process(pinned.numpy(), T, hop, pcm_format="s16", want_pixels=mode != "feed")
            page = engines[2].process(xs, T, hop, pcm_format="s16", want_pixels=mode != "feed")
            assert_bits_equal(pin, dev, (mode, "pinned", k))
            assert_bits_equal(page, dev, (mode, "pageable", k))


# ---- waveform -------------------------------------------------------------------------------------------------------
# (channels, channel_mode): one capture channel; two mixed to one; stereo; one capture channel shown as two
WAVE_LAYOUTS = {"mono": (1, "mono"), "mix": (2, "mono"), "stereo": (2, "stereo"), "mono-as-two": (1, "stereo")}
WAVE_DISPLAYS = {
    "none": None,
    "point": {"interp_mode": "point"},
    "catmull-rom-gauss": {"interp_mode": "catmull_rom", "filter_mode": "gauss", "filter_radius": 2.0},
    "lanczos": {"interp_mode": "lanczos"},
    "lanczos-gauss": {"interp_mode": "lanczos", "filter_mode": "gauss"},
}


def _wave_pair(layout, display, normalize, S):
    from waveform_b200 import WaveEngine

    cc, cm = WAVE_LAYOUTS[layout]
    settings = {"width": 800, "meter_buf": 150, "channel_mode": cm, **(WAVE_DISPLAYS[display] or {})}
    if normalize:
        settings.update(normalize_volume=True, volume_target=-12.0, max_gain=20.0)
    return WaveEngine(settings, channels=cc, max_streams=S), WaveEngine(settings, channels=cc, max_streams=S), cc


def _wave_call(eng, x, T, hop, fmt, rms, display, device=True):
    import torch

    pcm = _dev(x) if device else x
    r = None if rms is None else (torch.from_numpy(rms).cuda() if device else rms)
    disp = display != "none"
    before = eng.launch_count
    out = eng.process(pcm, T, hop, input_rms=r, want_points=disp, want_pixels=disp, pcm_format=fmt)
    torch.cuda.synchronize()
    assert eng.launch_count - before == 1
    return to_host(out)


@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalized"])
@pytest.mark.parametrize("display", list(WAVE_DISPLAYS))
@pytest.mark.parametrize("chunk", ["1", "0"], ids=["chunked", "per-tick"])
@pytest.mark.parametrize("layout", list(WAVE_LAYOUTS))
def test_wave_s16_matches_f32_bit_for_bit(layout, chunk, display, normalize, monkeypatch):
    set_knobs(monkeypatch, {"WF_WAVE_CHUNK": chunk})
    S, T, hop = 5, 24, 800
    e16, e32, cc = _wave_pair(layout, display, normalize, S)
    x = _signals(S, cc, 2 * T * hop, seed=cc * 100 + len(display))
    # stream 1: ten packets of -32768 (= -1.0, 0 dB: they fill the 150 ms buffer with 0.0f) and then all-zero packets trip
    # the silent rule (the reference's test is "every entry exactly 0.0f"; the mixed layout's raw second row never passes it)
    x[1, :, 2 * hop: 12 * hop] = -32768
    x[1, :, 12 * hop: 16 * hop] = 0
    rng = np.random.default_rng(5)
    rms = (0.01 + 0.3 * rng.uniform(size=(S, 2 * T))).astype(np.float32) if normalize else None
    for k in range(2):
        xs = np.ascontiguousarray(x[:, :, k * T * hop: (k + 1) * T * hop])
        r = None if rms is None else np.ascontiguousarray(rms[:, k * T: (k + 1) * T])
        g16 = _wave_call(e16, xs, T, hop, "s16", r, display)
        g32 = _wave_call(e32, _f32(xs), T, hop, "f32", r, display)
        assert_bits_equal(g16, g32, (layout, chunk, display, normalize, k))
        if k == 0:
            # (volume normalisation adds its gain to the 0 dB entries, so they are no longer 0.0f)
            assert g16["silent"][1].any() == (layout != "mix" and not normalize) and not g16["silent"][0].any()
    x3 = _f32(_signals(S, cc, T * hop, seed=9))
    r3 = None if rms is None else np.ascontiguousarray(rms[:, :T])
    assert_bits_equal(_wave_call(e16, x3, T, hop, "f32", r3, display), _wave_call(e32, x3, T, hop, "f32", r3, display),
                      (layout, chunk, display, normalize, "state"))


def test_wave_formats_alternated_and_buffer_kinds():
    """S16, F32, S16 on one engine equal three F32 calls; pinned and pageable host int16 equal the device call."""
    import torch

    S, T, hop = 5, 24, 800
    for layout in ("mix", "mono-as-two"):
        mixed, ref, cc = _wave_pair(layout, "catmull-rom-gauss", False, S)
        pin_e, page_e, _ = _wave_pair(layout, "catmull-rom-gauss", False, S)
        x = _signals(S, cc, 3 * T * hop, seed=21)
        x[1, :, 2 * hop: 12 * hop] = -32768
        x[1, :, 12 * hop: 16 * hop] = 0
        for k, fmt in enumerate(("s16", "f32", "s16")):
            xs = np.ascontiguousarray(x[:, :, k * T * hop: (k + 1) * T * hop])
            a = _wave_call(mixed, xs if fmt == "s16" else _f32(xs), T, hop, fmt, None, "catmull-rom-gauss")
            b = _wave_call(ref, _f32(xs), T, hop, "f32", None, "catmull-rom-gauss")
            assert_bits_equal(a, b, (layout, k, fmt))
            if fmt == "s16":
                pinned = torch.from_numpy(xs).pin_memory()
                p = _wave_call(pin_e, pinned.numpy(), T, hop, "s16", None, "catmull-rom-gauss", device=False)
                q = _wave_call(page_e, xs, T, hop, "s16", None, "catmull-rom-gauss", device=False)
            else:
                p = _wave_call(pin_e, _f32(xs), T, hop, "f32", None, "catmull-rom-gauss", device=False)
                q = _wave_call(page_e, _f32(xs), T, hop, "f32", None, "catmull-rom-gauss", device=False)
            assert_bits_equal(p, a, (layout, k, "pinned"))
            assert_bits_equal(q, a, (layout, k, "pageable"))


# ---- the volume-normalisation chain, fully in int16 -------------------------------------------------------------------
def test_normalization_chain_all_int16():
    """An INPUT_RMS meter feeds wf_process (normalize_volume) and a waveform engine (normalize_volume); with every call
    in S16 the results equal the all-float32 chain bit for bit."""
    import torch
    from waveform_b200 import Engine

    S, T, hop, N = 5, 16, 800, 1024
    x = _signals(S, 2, 2 * T * hop + N, seed=31)
    spec = {"fft_size": N, "normalize_volume": True, "volume_target": -10.0, "silence_gate": True}
    chains = {}
    for fmt in ("s16", "f32"):
        feed = _meter_pair("feed", 2, S)[0]
        eng = Engine(spec, channels=2, max_streams=S)
        wave = _wave_pair("mix", "lanczos", True, S)[0]
        outs = []
        for k in range(2):
            xs = np.ascontiguousarray(x[:, :, k * T * hop: k * T * hop + T * hop + N])
            pcm = _dev(xs if fmt == "s16" else _f32(xs))
            rms = feed.process(pcm, T, hop, pcm_format=fmt)["rms"]
            sp = eng.process(pcm, T, hop, input_rms=rms, want_points=True, pcm_format=fmt)
            wv = wave.process(pcm, T, hop, input_rms=rms, want_points=True, want_pixels=True, pcm_format=fmt)
            torch.cuda.synchronize()
            outs.append({"rms": rms, **{f"spec_{a}": b for a, b in sp.items()}, **{f"wave_{a}": b for a, b in wv.items()}})
        chains[fmt] = outs
    for k in range(2):
        assert_bits_equal(chains["s16"][k], chains["f32"][k], ("chain", k))
    assert np.isfinite(to_host(chains["s16"][1])["spec_db"]).all()


# ---- ABI ------------------------------------------------------------------------------------------------------------
def test_meter_wave_abi_sizes_and_errors():
    """The current size, the size that ends before pcm_format and the size that ends before the display outputs are
    accepted; the two older ones read as float32 whatever pcm_format holds.  Any other size is WF_ERR_ABI; an unknown
    pcm_format and an odd int16 address are WF_ERR_INVALID_ARG."""
    import torch
    from waveform_b200.engine import WF_ERR_ABI, WF_ERR_INVALID_ARG, WF_OK, WfMeterBatch, WfWaveBatch

    S, T, hop = 2, 4, 800
    x = _signals(S, 2, T * hop, seed=41)
    xf = _dev(_f32(x))
    x16 = torch.zeros(S * 2 * T * hop + 8, dtype=torch.int16, device="cuda")
    for kind in ("meter", "wave"):
        if kind == "meter":
            Batch, prev_sizes = WfMeterBatch, (WfMeterBatch.pcm_format.offset, WfMeterBatch.out_pixels.offset)
            mk = lambda: _meter_pair("rms", 2, S)[0]  # noqa: E731
            fn = "wf_meter_process"
        else:
            Batch, prev_sizes = WfWaveBatch, (WfWaveBatch.pcm_format.offset, WfWaveBatch.out_points.offset)
            mk = lambda: _wave_pair("mix", "none", False, S)[0]  # noqa: E731
            fn = "wf_wave_process"
        ref_eng = mk()
        L = ref_eng.L
        out_shape = (S, T, 2) if kind == "meter" else (S, T, 1, 800)

        def batch(pcm, fmt, size=None):
            out = torch.empty(out_shape, device="cuda")
            b = Batch(struct_size=C.sizeof(Batch) if size is None else size, n_streams=S, n_ticks=T, hop=hop, pcm=pcm,
                      stream_stride=2 * T * hop, channel_stride=T * hop, pcm_format=fmt)
            if kind == "meter":
                b.out_db = out.data_ptr()
            else:
                b.out = out.data_ptr()
            return b, out

        b, want = batch(xf.data_ptr(), 0)
        assert getattr(L, fn)(ref_eng.h, C.byref(b)) == WF_OK
        for size in prev_sizes:
            e = mk()
            b, got = batch(xf.data_ptr(), 1, size)  # pcm_format lies beyond the struct: must not be read
            assert getattr(L, fn)(e.h, C.byref(b)) == WF_OK, (kind, size)
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (kind, size)
        e = mk()
        for size in (prev_sizes[1] - 8, prev_sizes[0] + 4, C.sizeof(Batch) + 8, 0):
            assert getattr(L, fn)(e.h, C.byref(batch(xf.data_ptr(), 0, size)[0])) == WF_ERR_ABI, (kind, size)
        for fmt in (2, -1):
            assert getattr(L, fn)(e.h, C.byref(batch(x16.data_ptr(), fmt)[0])) == WF_ERR_INVALID_ARG, (kind, fmt)
            assert b"pcm_format" in getattr(L, fn.replace("process", "last_error"))(e.h)
        assert getattr(L, fn)(e.h, C.byref(batch(x16.data_ptr() + 1, 1)[0])) == WF_ERR_INVALID_ARG
        assert b"aligned" in getattr(L, fn.replace("process", "last_error"))(e.h)
        assert getattr(L, fn)(e.h, C.byref(batch(x16.data_ptr() + 2, 1)[0])) == WF_OK


def test_meter_wave_numpy_int16_without_keyword_stays_unscaled():
    """Without pcm_format an int16 numpy array is converted to float32 as it is (unscaled), as before."""
    x = np.random.default_rng(2).integers(-200, 200, size=(2, 2, 8 * 800), dtype=np.int16)
    for mk in (lambda: _meter_pair("rms", 2, 2)[0], lambda: _wave_pair("mix", "none", False, 2)[0]):
        a = mk().process(x, 8, 800)
        b = mk().process(x.astype(np.float32), 8, 800)
        assert_bits_equal(a, b, "int16 numpy without pcm_format")
