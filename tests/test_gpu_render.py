"""wf_render / Engine.render: the display stage on dB rows the caller passes in (csrc/wf_render.cu).

Rendering a spectrum call's own out_db must give that call's display outputs bit for bit, whichever kernel family made
them: all of them run the same display_stage_tab (wf_kernels.cuh).  With a peak, the rows are normalised with
wf_peak_normalize's arithmetic before they are rendered, and the result is checked against the oracle's render_curve /
render_bars restatement of the normalised rows."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from gpu_common import CATALOGUE, assert_bits_equal, clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import check_points, synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]


def _case(route, **display):
    """(kernel family of the spectrum call, knobs, settings, capture channels): a route with these display settings."""
    r = CATALOGUE[route]
    settings = {"fft_size": r.N, **({"channel_mode": "stereo"} if r.stereo else {}), **display}
    return r.family.split("/")[0], r.env, settings, r.cc


FAMILY_CASES = [
    _case("warp2-1024-display", interp_mode="lanczos", height=300),
    _case("warp2-2048-display", display_mode="bars", interp_mode="catmull_rom", rounded_caps=True, min_bar_height=5,
          bar_width=10, bar_gap=2),
    _case("warp2-800-display", interp_mode="point", filter_mode="gauss", mirror_freq_axis=True),
    _case("v3-1024-stereo-display", channel_spacing=20, mirror_freq_axis=True, filter_mode="gauss", height=400),
    _case("v3-4096-stereo-display", display_mode="bars", channel_spacing=10, rounded_caps=True, mirror_freq_axis=True,
          interp_mode="point"),
    _case("v3-4096-mix-display", display_mode="bars", interp_mode="lanczos", min_bar_height=4),
    _case("wide-8192-display", interp_mode="lanczos", filter_mode="gauss"),
    _case("wide-4096-stereo-display", display_mode="bars", interp_mode="catmull_rom", mirror_freq_axis=True),
    _case("fused-2048-stereo-display", display_mode="bars", interp_mode="lanczos", min_bar_height=3, channel_spacing=6),
    _case("fused-512-display", interp_mode="catmull_rom", filter_mode="gauss"),
    _case("smem-800-stereo-display", display_mode="bars", interp_mode="catmull_rom", rounded_caps=True, bar_width=8,
          bar_gap=3),
    _case("smem-1456-display", interp_mode="lanczos", mirror_freq_axis=True),
    # a stereo row of 65536 floats does not fit in shared memory: the render kernel keeps it in its L2 scratch
    _case("l2-65536-stereo-display", interp_mode="lanczos", width=640),
]


def _case_id(c):
    fam, env, s, cc = c
    return f"{fam}-{s['fft_size']}-{s.get('display_mode', 'curve')}-{'stereo' if s.get('channel_mode') == 'stereo' else cc}"


def _spectrum(eng, settings, T=6, S=4, silent=True, **kw):
    """A device spectrum call with silent stretches: stream 1 is digital silence throughout (DB_MIN rows), stream 2 from
    tick 3 on (the silence gate holds and then clears its rows)."""
    import torch
    N = eng.fft_size
    hop = N // 2
    zf = [(1, 0, T + 1), (2, 3, T + 1)] if silent and S > 2 else []
    pcm = synth_pcm(S, eng.capture_channels, (T - 1) * hop + N, zero_frames=zf, frame_len=N, hop=hop)
    out = eng.process(torch.from_numpy(pcm).cuda(), T, hop, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", FAMILY_CASES, ids=[_case_id(c) for c in FAMILY_CASES])
def test_render_of_own_db_is_bit_identical(case, monkeypatch):
    import torch
    from waveform_b200 import Engine

    fam, env, settings, cc = case
    set_knobs(monkeypatch, env)
    S, T = (2, 2) if settings["fft_size"] > 32768 else (4, 6)
    eng = Engine(settings, channels=cc, max_streams=S)
    out = _spectrum(eng, settings, T=T, S=S, want_points=True, want_pixels=True)
    name = eng.last_kernel_name()
    assert name.startswith(fam + "<"), (fam, name)
    if fam == "stft_warp2_kernel":
        assert "display" in name, name
    db = out["db"]
    if S > 2:
        assert (db[1].cpu().numpy() <= eng.db_min).any(), "stream 1 should carry DB_MIN rows"
    db0 = db.clone()
    r = eng.render(db, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert eng.last_kernel_name().startswith("render_kernel<")
    for key in ("points", "pixels", "min"):
        assert_bits_equal(r[key], out[key], (key, name))
    # points only (the display stage stores them without its shared-memory rows), pixels only
    rp = eng.render(db, want_points=True)
    rx = eng.render(db, want_pixels=True)
    torch.cuda.synchronize()
    assert_bits_equal(rp["points"], out["points"], ("points only", name))
    assert_bits_equal(rx["pixels"], out["pixels"], ("pixels only", name))
    assert_bits_equal(rx["min"], out["min"], ("min only", name))
    assert_bits_equal(db, db0, "db untouched")


PEAK_CASES = [FAMILY_CASES[1], FAMILY_CASES[3], FAMILY_CASES[4], FAMILY_CASES[6]]


@pytest.mark.parametrize("case", PEAK_CASES, ids=[_case_id(c) for c in PEAK_CASES])
def test_render_with_peak(case, monkeypatch):
    import torch
    from oracle.oraclebind import OracleSource
    from waveform_b200 import Engine

    fam, env, settings, cc = case
    set_knobs(monkeypatch, env)
    eng = Engine(settings, channels=cc, max_streams=4)
    out = _spectrum(eng, settings, want_peak=True)
    db, peak = out["db"], out["peak"]
    db0 = db.clone()
    ref = db.clone()
    eng.peak_normalize(ref, peak, -3.0, 20.0)
    got = db.clone()
    r = eng.render(got, peak, -3.0, 20.0, write_db=True, want_points=True, want_pixels=True)
    r_keep = eng.render(db, peak, -3.0, 20.0, want_points=True, want_pixels=True)
    r0 = eng.render(ref, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert_bits_equal(got, ref, "write_db equals peak_normalize")
    assert_bits_equal(db, db0, "db untouched without write_db")
    for key in ("points", "pixels", "min"):
        assert_bits_equal(r[key], r0[key], key)
        assert_bits_equal(r_keep[key], r0[key], key)
    # against the oracle's render_curve / render_bars of the normalised rows
    nref = ref.cpu().numpy()
    o = OracleSource(settings, channels=cc)
    exp_px, exp_min = o.pixels_of(nref)
    px, mn = r["pixels"].cpu().numpy(), r["min"].cpu().numpy()
    assert np.abs(px - exp_px).max() < 2e-4, float(np.abs(px - exp_px).max())
    assert np.abs(mn[..., 0] - exp_min[..., 0]).max() < 2e-4
    assert (mn[..., 1] == exp_min[..., 1]).mean() > 0.9
    assert check_points(settings, cc, nref, r["points"].cpu().numpy()) < 2e-6
    # the gain really moved the display: the normalised rows render differently from the raw ones
    raw = eng.render(db, want_pixels=True)
    torch.cuda.synchronize()
    assert not np.array_equal(raw["pixels"].cpu().numpy(), px)


def test_host_and_device_inputs_agree():
    import torch
    from waveform_b200 import Engine

    settings = FAMILY_CASES[3][2]
    eng = Engine(settings, channels=2, max_streams=4)
    out = _spectrum(eng, settings, want_peak=True)
    db_d, peak_d = out["db"], out["peak"]
    db_h, peak_h = db_d.cpu().numpy(), peak_d.cpu().numpy()
    # no peak
    rd = eng.render(db_d, want_points=True, want_pixels=True)
    rh = eng.render(db_h, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    for key in rd:
        assert_bits_equal(rd[key], rh[key], key)
    # with a peak and write_db: device rows + device peak, device rows + host peak, host rows + host peak (in place)
    a = db_d.clone()
    ra = eng.render(a, peak_d, -6.0, 12.0, write_db=True, want_points=True, want_pixels=True)
    b = db_d.clone()
    rb = eng.render(b, peak_h, -6.0, 12.0, write_db=True, want_points=True, want_pixels=True)
    c = db_h.copy()
    rc = eng.render(c, peak_h, -6.0, 12.0, write_db=True, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert_bits_equal(a, b, "host peak")
    assert_bits_equal(a, c, "host rows")
    for key in ra:
        assert_bits_equal(ra[key], rb[key], key)
        assert_bits_equal(ra[key], rc[key], key)
    # a row base that is not 16-byte aligned takes the scalar path: same bits
    flat = torch.empty(db_d.numel() + 1, device="cuda")
    flat[1:] = db_d.reshape(-1)
    odd = flat[1:].view(db_d.shape)
    ro = eng.render(odd, peak_d, -6.0, 12.0, write_db=True, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert_bits_equal(odd, a, "unaligned rows")
    for key in ra:
        assert_bits_equal(ro[key], ra[key], key)


def test_render_on_a_side_stream_is_ordered_after_its_producer():
    import torch
    from waveform_b200 import Engine

    settings = FAMILY_CASES[1][2]
    eng = Engine(settings, channels=1, max_streams=4)
    out = _spectrum(eng, settings, want_peak=True)
    expect = eng.render(out["db"].clone(), out["peak"], -3.0, 20.0, write_db=True, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    dst = torch.full_like(out["db"], -1.0)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)     # the producer is still busy when render is enqueued
        dst.copy_(out["db"])
        r = eng.render(dst, out["peak"], -3.0, 20.0, write_db=True, want_points=True, want_pixels=True)
        after = dst.clone()
    torch.cuda.synchronize()
    for key in expect:
        assert_bits_equal(r[key], expect[key], key)
    ref = out["db"].clone()
    eng.peak_normalize(ref, out["peak"], -3.0, 20.0)
    torch.cuda.synchronize()
    assert_bits_equal(after, ref, "db written back on the side stream")


def test_render_errors():
    import torch
    from waveform_b200 import Engine, WfError
    from waveform_b200.engine import WF_ERR_ABI, WF_ERR_INVALID_ARG, WfRenderBatch

    eng = Engine({"fft_size": 1024}, channels=1, max_streams=2)
    db = torch.zeros((2, 3, 1, eng.bins), device="cuda")
    peak = torch.zeros(3, device="cuda")
    with pytest.raises(WfError) as ei:
        eng.render(db)                                           # nothing requested
    assert ei.value.status == WF_ERR_INVALID_ARG and "nothing requested" in str(ei.value)
    with pytest.raises(WfError) as ei:
        eng.render(db, None, write_db=True, want_points=True)    # write_db without a peak
    assert ei.value.status == WF_ERR_INVALID_ARG and "no peak" in str(ei.value)
    with pytest.raises(ValueError):
        eng.render(torch.zeros((2, 3, 1, eng.bins + 8), device="cuda"), want_points=True)

    def raw(**fields):
        rb = WfRenderBatch()
        rb.struct_size = C.sizeof(WfRenderBatch)
        rb.n_streams, rb.n_frames, rb.db = 2, 3, db.data_ptr()
        pts = torch.empty((2, 3, 1, eng.num_points), device="cuda")
        rb.out_points = pts.data_ptr()
        for k, v in fields.items():
            setattr(rb, k, v)
        rc = eng.L.wf_render(eng.h, C.byref(rb), torch.cuda.current_stream().cuda_stream or 1)
        torch.cuda.synchronize()
        return rc, eng.L.wf_last_error(eng.h).decode()

    assert raw()[0] == 0
    assert raw(struct_size=C.sizeof(WfRenderBatch) - 8)[0] == WF_ERR_ABI
    for k in ("n_streams", "n_frames"):
        rc, msg = raw(**{k: -1})
        assert rc == WF_ERR_INVALID_ARG and "must be >= 0" in msg, (k, msg)
    rc, msg = raw(out_points=None, write_db=1, peak=peak.data_ptr())
    assert rc == 0                                                # write_db alone is a request
    rc, msg = raw(out_points=None)
    assert rc == WF_ERR_INVALID_ARG and "nothing requested" in msg
    rc, msg = raw(db=None)
    assert rc == WF_ERR_INVALID_ARG and "db is null" in msg
    assert raw(n_streams=0)[0] == 0                               # an empty batch is a no-op


def _same_dev(a, b):
    import torch
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("settings,S,T", [
    ({"fft_size": 2048, "display_mode": "bars", "interp_mode": "catmull_rom", "bar_width": 24, "bar_gap": 6}, 4096, 16),
    ({"fft_size": 16384, "interp_mode": "lanczos", "width": 800}, 1024, 16),
], ids=["2048-bars-4096x16", "16384-curve-1024x16"])
def test_render_at_scale(settings, S, T):
    """Config 5 shapes, 4096 x 16 rows at N=2048 (26 bars) and 1024 x 16 at N=16384 (800-point curve): rendering the spectrum
    call's out_db gives the call's own display outputs, bit for bit on every row; with the peak, the write-back equals
    peak_normalize and the outputs equal a render of the normalised rows."""
    import torch
    from helpers import device_pcm
    from waveform_b200 import Engine

    N = settings["fft_size"]
    eng = Engine(settings, channels=1, max_streams=S)
    pcm = device_pcm(S, 1, (T - 1) * N + N, zero_every=7, frame_len=N)
    out = eng.process(pcm, T, N, want_peak=True, want_points=True, want_pixels=True)
    spectrum = eng.last_kernel_name()
    r = eng.render(out["db"], want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    for key in ("points", "pixels", "min"):
        assert _same_dev(r[key], out[key]), (key, spectrum, eng.last_kernel_name())
    norm = out["db"].clone()
    eng.peak_normalize(norm, out["peak"], -3.0, 30.0)
    got = out["db"]
    rn = eng.render(got, out["peak"], -3.0, 30.0, write_db=True, want_points=True, want_pixels=True)
    r0 = eng.render(norm, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert _same_dev(got, norm), "write_db at scale"
    for key in ("points", "pixels", "min"):
        assert _same_dev(rn[key], r0[key]), key


def test_process_normalized_display_equals_the_steps_by_hand():
    import torch
    from waveform_b200 import Engine
    from waveform_b200.shard import ShardedEngine

    settings = {"fft_size": 16384, "interp_mode": "lanczos", "width": 800, "filter_mode": "gauss"}
    S, T, N = 6, 5, 16384
    pcm = torch.from_numpy(synth_pcm(S, 1, (T - 1) * N + N, zero_frames=[(2, 1, 3)], frame_len=N, hop=N)).cuda()
    a = ShardedEngine(Engine(settings, channels=1, max_streams=S)).process_normalized_display(
        pcm, T, N, target_db=-3.0, max_gain=25.0, want_points=True, want_pixels=True)
    eng = Engine(settings, channels=1, max_streams=S)
    out = eng.process(pcm, T, N, want_peak=True)
    eng.peak_normalize(out["db"], out["peak"], -3.0, 25.0)
    r = eng.render(out["db"], want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert_bits_equal(a["db"], out["db"], "db")
    assert_bits_equal(a["peak"], out["peak"], "peak")
    for key in ("points", "pixels", "min"):
        assert_bits_equal(a[key], r[key], key)
