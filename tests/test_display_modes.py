"""Display outputs of the waveform and level-meter modes: what render_curve (waveform) and render_bars (meter) draw.

CPU: the waveform display tables (wf_wave_preview_table) bit-exact against the compiled reference's m_interp_indices,
m_interp_kernel.weights and m_kernel.weights; a numpy restatement of the two display stages (below) against the reference's
own render() after every tick, recorded in tests/golden/reference_display.npz; the new struct layouts and the previous struct
sizes.  GPU: the CUDA display stages against that restatement applied to the engine's own dB rows, the chunked kernel against
the per-tick one, display-only calls, the meter's fused and three-kernel paths, and the error paths.
"""
from __future__ import annotations

import ctypes as C
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

from gpu_common import clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import synth_pcm
from refdata import digest

pytestmark = pytest.mark.usefixtures("clean_knobs")

ROOT = Path(__file__).resolve().parents[1]
STORE = Path(__file__).resolve().parent / "golden" / "reference_display.npz"
RECORDING = __import__("os").environ.get("WF_RECORD_REFERENCE") == "1"
_store: dict | None = None
_recorded: dict = {}


def reference(key: str, compute) -> dict:
    """Like refdata.reference, with its own store: compute() runs against the live reference when recording."""
    global _store
    if RECORDING:
        rec = {k: np.asarray(v) for k, v in compute().items()}
        if not _recorded:
            __import__("atexit").register(_save)
        _recorded[key] = rec
        return rec
    if _store is None:
        with np.load(STORE, allow_pickle=False) as z:
            index, blob = json.loads(z["index"].tobytes()), z["data"]
            _store = {k: {f: blob[o: o + int(np.prod(sh, dtype=np.int64)) * np.dtype(dt).itemsize].view(dt).reshape(tuple(sh))
                          for f, (dt, sh, o) in fs.items()} for k, fs in index.items()}
    assert key in _store, f"{key}: not in {STORE.name}; record it with WF_RECORD_REFERENCE=1 against the reference"
    return _store[key]


def _save():
    index, parts, off = {}, [], 0
    for key in sorted(_recorded):
        index[key] = {}
        for f, v in sorted(_recorded[key].items()):
            index[key][f] = (v.dtype.str, list(v.shape), off)
            parts.append(np.ascontiguousarray(v).tobytes())
            off += v.nbytes
    np.savez_compressed(STORE, index=np.frombuffer(json.dumps(index).encode(), dtype=np.uint8),
                        data=np.frombuffer(b"".join(parts), dtype=np.uint8))


# ---- numpy restatement of the display stages (float32, the reference's operation order) -----------------------------
f32 = np.float32


def std_lerp(a, b, t):
    """std::lerp(float, float, float) as libstdc++ evaluates it, elementwise."""
    a, b, t = f32(a), f32(b), np.asarray(t, f32)
    if (a <= 0 and b >= 0) or (a >= 0 and b <= 0):
        return (t * b + (f32(1) - t) * a).astype(f32)
    x = (a + t * (b - a)).astype(f32)
    y = np.where((t > 1) == (b > a), np.where(b < x, x, b), np.where(b > x, x, b)).astype(f32)
    return np.where(t == 1, b, y).astype(f32)


def px_of(db, ceiling, rng, top, bottom):
    x = (f32(ceiling) - np.asarray(db, f32)).astype(f32)
    c = np.where(x < 0, f32(0), np.where(f32(rng) < x, f32(rng), x)).astype(f32)
    return std_lerp(top, bottom, (c / f32(rng)).astype(f32))


def first_min(px, cpos, width):
    """(miny, minpos) of the sequential scan: start at (cpos, 0), a strictly smaller value replaces it."""
    flat = px.reshape(*px.shape[:-2], -1)
    k = np.argmin(flat, axis=-1)
    v = np.take_along_axis(flat, k[..., None], -1)[..., 0]
    lt = v < f32(cpos)
    return np.stack([np.where(lt, v, f32(cpos)), np.where(lt, (k % width).astype(f32), f32(0))], -1).astype(f32)


def wave_geometry(s):
    stereo = s.get("channel_mode") == "stereo"
    floor, ceiling = int(s.get("floor", -65)), int(s.get("ceiling", 0))
    if ceiling - floor < 1:
        floor, ceiling = -120, 0
    height = int(s.get("height", 225)) or 225
    spacing = int(s.get("channel_spacing", 0))
    if not stereo or height - spacing < 1:
        spacing = 0
    cpos = f32(height) / f32(2) if stereo else f32(height)
    return ceiling, ceiling - floor, f32(cpos - f32(spacing) * f32(0.5)), f32(cpos)


def wave_display(rows, tables, settings):
    """render_curve in waveform mode for dB rows [..., dch, W]: (points, pixels, min)."""
    rows = np.asarray(rows, f32)
    W = rows.shape[-1]
    index = tables["interp_indices"].astype(np.int32)
    wts = tables["interp_weights"]
    if wts.size == 0:
        pts = rows[..., index]
    else:
        taps = wts.size // W
        wt = wts.reshape(W, taps)
        start = index - taps // 2 + 1
        pts = np.zeros(rows.shape, f32)
        for k in range(taps):
            j = start + k
            ok = (j >= 0) & (j < W)
            pts = np.where(ok, (pts + (rows[..., np.clip(j, 0, W - 1)] * wt[:, k]).astype(f32)).astype(f32), pts)
    g = tables["gauss"]
    if g.size:
        R = (g.size + 1) // 2
        i = np.arange(W)
        acc, wsum = np.zeros(pts.shape, f32), np.zeros(W, f32)
        for k in range(g.size):
            j = i - R + 1 + k
            ok = (j >= 0) & (j < W)
            acc = np.where(ok, (acc + (pts[..., np.clip(j, 0, W - 1)] * g[k]).astype(f32)).astype(f32), acc)
            wsum = np.where(ok, (wsum + g[k]).astype(f32), wsum)
        pts = (acc / wsum).astype(f32)
    ceiling, rng, hi, cpos = wave_geometry(settings)
    px = px_of(pts, ceiling, rng, 0.0, hi)
    return pts, px, first_min(px, cpos, W)


def meter_display(db, settings):
    """render_bars in meter mode for m_meter_val [..., cc]: (pixels, min)."""
    floor, ceiling = int(settings.get("floor", -65)), int(settings.get("ceiling", 0))
    if ceiling - floor < 1:
        floor, ceiling = -120, 0
    cpos = f32(int(settings.get("height", 225)) or 225)
    r = f32(int(settings.get("bar_width", 24))) / f32(2)
    caps = bool(settings.get("rounded_caps", False))
    top = r if caps else f32(0)
    bottom = f32(cpos - r) if caps else cpos
    mbh = int(settings.get("min_bar_height", 0))
    if mbh > 0:
        bottom = f32(bottom - f32(mbh))
    bottom = min(max(bottom, top), cpos)
    px = px_of(db, ceiling, ceiling - floor, top, bottom)
    return px, first_min(px[..., None, :], cpos, px.shape[-1])


# ---- cases ---------------------------------------------------------------------------------------------------------
from test_wave import CHUNK_CASES, WAVE_CASES, _case  # noqa: E402

WAVE_DISPLAY_CASES = WAVE_CASES + [
    ({"width": 800, "meter_buf": 150, "filter_mode": "gauss", "filter_radius": 2.0}, 2, 800),
    ({"width": 640, "meter_buf": 100, "channel_mode": "stereo", "channel_spacing": 20, "interp_mode": "lanczos",
      "filter_mode": "gauss"}, 2, 480),
    ({"width": 301, "meter_buf": 40, "interp_mode": "point", "height": 300, "floor": -90, "ceiling": -6}, 1, 97),
]
METER_DISPLAY_CASES = [
    ({"rms_mode": False}, 1, 800),
    ({"rms_mode": True}, 2, 800),
    ({"rms_mode": True, "rounded_caps": True, "bar_width": 30}, 2, 441),
    ({"rms_mode": False, "min_bar_height": 12, "height": 300, "floor": -80, "ceiling": -3}, 2, 800),
    ({"rms_mode": True, "rounded_caps": True, "min_bar_height": 500}, 1, 1600),  # border_bottom clamped to border_top
]
WAVE_KEYS = ("width", "meter_buf", "channel_mode", "normalize_volume")


def _tables(settings, ch=2):
    from waveform_b200.engine import make_wave_config, preview_wave_tables

    return preview_wave_tables(make_wave_config(settings, channels=ch))


# ---- CPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [64, 200, 301, 640, 800, 1000, 1920])
@pytest.mark.parametrize("interp", ["point", "lanczos", "catmull_rom"])
@pytest.mark.parametrize("gauss", [False, True])
def test_wave_display_tables_are_bit_exact_vs_compiled_reference(width, interp, gauss):
    s = {"width": width, "meter_buf": 150, "interp_mode": interp}
    if gauss:
        s.update(filter_mode="gauss", filter_radius=1.5 + width % 3)

    def live():
        from oracle import refbind

        r = refbind.RefSource({"display_mode": "waveform", **s}, channels=2)
        taps, w = r.interp_kernel()
        g = r.gauss_kernel()[0] if gauss else None
        return {"idx": digest(r.interp_indices()), "w": digest(None if interp == "point" else np.asarray(w, f32).ravel()),
                "g": digest(None if g is None else np.asarray(g, f32))}

    ref = reference(f"tables/{width}/{interp}/{int(gauss)}", live)
    t = _tables(s)
    assert np.array_equal(digest(t["interp_indices"]), ref["idx"])
    assert np.array_equal(digest(t["interp_weights"] if t["interp_weights"].size else None), ref["w"])
    assert np.array_equal(digest(t["gauss"] if t["gauss"].size else None), ref["g"])
    if interp == "point":  # std::lerp lands just below some integers: the point mode takes the sample before them
        below = t["interp_indices"].astype(np.int32) != np.arange(width)
        assert below.sum() == {800: 37, 1920: 48, 1000: 0}.get(width, below.sum())


def _ref_render_wave(settings, ch, pcm, T, hop, rms, ticks):
    from oracle import refbind

    r = refbind.RefSource({"display_mode": "waveform", **settings}, channels=ch)
    px = []
    for t in range(T):
        r.run_wave(pcm[:, t * hop:(t + 1) * hop], 1, hop, rms=None if rms is None else rms[t: t + 1])
        if t in ticks:
            r.render()
            px.append(np.stack([r.render_buf(c)[: settings['width']] for c in range(r.display_channels)]))
    return {"px": np.stack(px)}


TICKS = list(range(0, 50, 4)) + [49]


@pytest.mark.parametrize("settings,ch,hop", WAVE_DISPLAY_CASES)
def test_wave_display_restatement_matches_reference_render(settings, ch, hop):
    """The numpy restatement, fed the oracle's dB rows (bit-exact against the reference's m_decibels, test_wave.py), against
    the pixels the reference's render() leaves in m_interp_bufs after the same tick."""
    from oracle.oraclebind import OracleWave

    T = 50
    pcm, rms = _case(settings, ch, hop, T)
    rms = None if rms is None else rms[0]
    key = f"wave/{WAVE_DISPLAY_CASES.index((settings, ch, hop))}"
    ref = reference(key, lambda: _ref_render_wave(settings, ch, pcm[0], T, hop, rms, TICKS))
    ws = {k: v for k, v in settings.items() if k in WAVE_KEYS}
    rows = OracleWave(ws, channels=ch).run(pcm[0], T, hop, rms=rms)["out"][TICKS]
    tables = _tables(settings, ch)
    _, px, mn = wave_display(rows, tables, settings)
    W = px.shape[-1]
    rp = ref["px"]
    ok = np.ones(px.shape, bool)
    if tables["gauss"].size:
        # From the second render on, the reference's Gaussian runs over a swapped-in buffer of 2 * width floats
        # (apply_filter sizes the loop by the buffer, src/filter.hpp:172-180), so its last radius - 1 points mix in stale
        # entries past the row.  The engine renormalises at the row's end, as the reference does on its first render.
        R = (tables["gauss"].size + 1) // 2
        ok[1:, :, W - R + 1:] = False
    assert np.abs(px - rp)[ok].max() < 5e-4
    # (miny, minpos) over the points both sides define: miny to the same tolerance, and the point the restatement picks is a
    # minimum of the reference's row to that tolerance too (near-ties may pick either)
    _, _, hi, cpos = wave_geometry(settings)
    inf = np.float32(np.inf)
    mn_ok = first_min(np.where(ok, px, inf), cpos, W)
    ref_mn = first_min(np.where(ok, rp, inf), cpos, W)
    assert np.abs(mn_ok[:, 0] - ref_mn[:, 0]).max() < 5e-4
    for t in range(len(TICKS)):
        if mn_ok[t, 0] < cpos:
            i = int(mn_ok[t, 1])
            picked = min(rp[t, d, i] for d in range(rp.shape[1]) if ok[t, d, i])
            assert picked - ref_mn[t, 0] < 1e-3, t
        else:
            assert ref_mn[t, 0] > cpos - 5e-4, t
    if ok.all():
        assert np.array_equal(mn_ok, mn)


def _ref_render_meter(settings, ch, pcm, T, hop):
    from oracle import refbind

    r = refbind.RefSource({"display_mode": "level_meter", **settings}, channels=ch)
    px, db = [], []
    for t in range(T):
        d = r.run_meter(pcm[:, t * hop:(t + 1) * hop], 1, hop)["db"]
        r.render()
        px.append(r.render_buf(0))
        db.append(d[0])
    return {"px": np.stack(px), "db": np.stack(db)}


@pytest.mark.parametrize("settings,ch,hop", METER_DISPLAY_CASES)
def test_meter_display_restatement_matches_reference_render(settings, ch, hop):
    from oracle.oraclebind import OracleMeter

    T = 40
    pcm = synth_pcm(1, ch, T * hop, seed=11)[0]
    pcm[:, 10 * hop: 20 * hop] = 0.0
    ref = reference(f"meter/{METER_DISPLAY_CASES.index((settings, ch, hop))}", lambda: _ref_render_meter(settings, ch, pcm, T, hop))
    px, _ = meter_display(ref["db"], settings)          # the reference's own m_meter_val
    assert np.abs(px - ref["px"]).max() < 1e-4
    ms = {k: v for k, v in settings.items() if k in ("rms_mode", "floor")}
    db = OracleMeter(ms, channels=ch).run(pcm, T, hop)["db"]
    px2, _ = meter_display(db, settings)
    assert np.abs(px2 - ref["px"]).max() < 5e-4


def test_display_struct_layouts_and_previous_sizes(tmp_path):
    from waveform_b200.engine import (WF_ERR_ABI, WF_ERR_INVALID_ARG, WfMeterBatch, WfMeterConfig, WfWaveBatch, WfWaveConfig, load_library,
                                      make_wave_config, TABLE_INTERP_INDICES)

    src = tmp_path / "sz3.c"
    fields = [("wf_wave_config", "interp_mode"), ("wf_wave_config", "channel_spacing"), ("wf_wave_batch", "out_points"),
              ("wf_wave_batch", "out_min"), ("wf_meter_config", "height"), ("wf_meter_config", "min_bar_height"),
              ("wf_meter_batch", "out_pixels"), ("wf_meter_batch", "out_min")]
    body = ", ".join(f"offsetof({s},{f})" for s, f in fields)
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   f'int main(){{printf("{" ".join(["%zu"] * len(fields))}\\n", {body});return 0;}}\n')
    exe = tmp_path / "sz3"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    types = {"wf_wave_config": WfWaveConfig, "wf_wave_batch": WfWaveBatch, "wf_meter_config": WfMeterConfig,
             "wf_meter_batch": WfMeterBatch}
    assert out == [getattr(types[s], f).offset for s, f in fields]
    # the previous structs end where the new fields begin
    assert (WfWaveConfig.interp_mode.offset, WfWaveBatch.out_points.offset) == (44, 64)
    assert (WfMeterConfig.height.offset, WfMeterBatch.out_pixels.offset) == (44, 72)
    L = load_library()
    cfg = make_wave_config({"width": 800}, channels=1)
    cfg.struct_size = WfWaveConfig.interp_mode.offset
    counts = np.zeros(4, np.int32)
    assert L.wf_wave_preview_plan(C.byref(cfg), 4, 800, counts.ctypes.data, None, 0) > 0
    assert L.wf_wave_preview_table(C.byref(cfg), TABLE_INTERP_INDICES, None, 0) == 0  # no display settings, no tables
    cfg.struct_size = 40
    assert L.wf_wave_preview_table(C.byref(cfg), TABLE_INTERP_INDICES, None, 0) == WF_ERR_ABI
    # the engine's limits come first: a width it refuses has no tables either (nothing is sized by it)
    big = make_wave_config({"width": 100000, "meter_buf": 150000}, channels=1)
    assert L.wf_wave_preview_table(C.byref(big), TABLE_INTERP_INDICES, None, 0) == WF_ERR_INVALID_ARG


# ---- GPU -----------------------------------------------------------------------------------------------------------
GPU_WAVE_CASES = CHUNK_CASES + WAVE_DISPLAY_CASES[len(WAVE_CASES):]


@pytest.mark.gpu
@pytest.mark.parametrize("device_ptrs", [False, True])
@pytest.mark.parametrize("settings,ch,hop", GPU_WAVE_CASES)
def test_gpu_wave_display_vs_restatement(settings, ch, hop, device_ptrs):
    from waveform_b200 import WaveEngine

    S, T = 4, 40
    pcm, rms = _case(settings, ch, hop, T, S)
    eng = WaveEngine(settings, channels=ch, max_streams=S)
    if device_ptrs:
        import torch

        o = eng.process(torch.from_numpy(pcm).cuda(), T, hop, input_rms=None if rms is None else torch.from_numpy(rms),
                        want_points=True, want_pixels=True)
        o = {k: v.cpu().numpy() for k, v in o.items()}
    else:
        o = eng.process(pcm, T, hop, input_rms=rms, want_points=True, want_pixels=True)
    pts, px, mn = wave_display(o["out"], _tables(settings, ch), settings)
    assert np.abs(o["points"] - pts).max() < 1e-3
    assert np.abs(o["pixels"] - px).max() < 2e-4
    assert np.array_equal(o["min"][..., 1], mn[..., 1])
    assert np.abs(o["min"][..., 0] - mn[..., 0]).max() < 2e-4
    # the full chain against the oracle: the dB tolerance of test_wave.py scaled to pixels
    from test_wave import _oracle_batch

    ref, _ = _oracle_batch({k: v for k, v in settings.items() if k in WAVE_KEYS}, ch, pcm, T, hop, rms)
    _, px_ref, _ = wave_display(ref, _tables(settings, ch), settings)
    ceiling, rng, hi, _ = wave_geometry(settings)
    assert np.abs(o["pixels"] - px_ref).max() <= 1e-3 * float(hi) / rng + 2e-4


def _wave_runs(settings, ch, hop, S, T, monkeypatch, chunk, want_db=True):
    from waveform_b200 import WaveEngine

    pcm, rms = _case(settings, ch, hop, T, S)
    pcm[1] = 0.0
    pcm[2, :, : 30 * hop] = 1.0
    set_knobs(monkeypatch, {"WF_WAVE_CHUNK": chunk})
    eng = WaveEngine(settings, channels=ch, max_streams=S)
    parts = [eng.process(pcm[:, :, : 13 * hop], 13, hop, input_rms=None if rms is None else rms[:, :13], want_db=want_db,
                         want_points=True, want_pixels=True),
             eng.process(pcm[:, :, 13 * hop:], T - 13, hop, input_rms=None if rms is None else rms[:, 13:], want_db=want_db,
                         want_points=True, want_pixels=True)]
    return {k: np.concatenate([p[k] for p in parts], axis=1) for k in parts[0]}


@pytest.mark.gpu
@pytest.mark.parametrize("settings,ch,hop", GPU_WAVE_CASES)
def test_gpu_wave_display_chunked_equals_per_tick_and_display_only(settings, ch, hop, monkeypatch):
    a = _wave_runs(settings, ch, hop, 5, 60, monkeypatch, "1")
    b = _wave_runs(settings, ch, hop, 5, 60, monkeypatch, "0")
    c = _wave_runs(settings, ch, hop, 5, 60, monkeypatch, "1", want_db=False)
    for k in ("points", "pixels", "min"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
        assert np.array_equal(a[k].view(np.uint32), c[k].view(np.uint32)), k
    assert "out" not in c and np.array_equal(a["silent"], c["silent"])


@pytest.mark.gpu
@pytest.mark.parametrize("settings,ch,hop", [CHUNK_CASES[0], CHUNK_CASES[1], CHUNK_CASES[5], WAVE_DISPLAY_CASES[-2]])
def test_gpu_wave_display_chunked_many_streams(settings, ch, hop, monkeypatch):
    a = _wave_runs(settings, ch, hop, 1700, 24, monkeypatch, "1")
    b = _wave_runs(settings, ch, hop, 1700, 24, monkeypatch, "0")
    for k in ("out", "points", "pixels", "min"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k


@pytest.mark.gpu
@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("settings,ch,hop", METER_DISPLAY_CASES)
def test_gpu_meter_display_vs_restatement(settings, ch, hop, fused, monkeypatch):
    import torch
    from waveform_b200 import MeterEngine

    set_knobs(monkeypatch, {"WF_METER_FUSED": fused})
    S, T = 6, 30
    pcm = synth_pcm(S, ch, T * hop, seed=5)
    pcm[1] = 0.0
    eng = MeterEngine(settings, channels=ch, max_streams=S)
    o = eng.process(pcm, T, hop, want_pixels=True)
    px, mn = meter_display(o["db"], settings)
    assert np.array_equal(o["pixels"], px) and np.array_equal(o["min"], mn)
    eng2 = MeterEngine(settings, channels=ch, max_streams=S)
    d = eng2.process(torch.from_numpy(pcm).cuda(), T, hop, want_pixels=True)
    assert np.array_equal(d["pixels"].cpu().numpy(), o["pixels"]) and np.array_equal(d["min"].cpu().numpy(), o["min"])


@pytest.mark.gpu
def test_gpu_display_error_paths():
    from waveform_b200 import MeterEngine, WaveEngine, WfError
    from waveform_b200.engine import (METER_INPUT_RMS, WF_ERR_INVALID_ARG, WF_OK, WfMeterBatch, WfMeterConfig, WfWaveBatch,
                                      WfWaveConfig, load_library, make_meter_config, make_wave_config)

    pcm = synth_pcm(2, 2, 4 * 800)
    with pytest.raises(WfError) as e:
        MeterEngine({}, channels=2, max_streams=2, mode=METER_INPUT_RMS).process(pcm, 4, 800, want_pixels=True)
    assert e.value.status == WF_ERR_INVALID_ARG
    L = load_library()
    # engines created from the previous struct sizes have no display settings
    mcfg = make_meter_config({}, channels=2, max_streams=2)
    mcfg.struct_size = WfMeterConfig.height.offset
    h = C.c_void_p()
    assert L.wf_meter_create(C.byref(mcfg), C.byref(h)) == WF_OK
    px = np.zeros((2, 4, 2), np.float32)
    mb = WfMeterBatch(struct_size=C.sizeof(WfMeterBatch), n_streams=2, n_ticks=4, hop=800, pcm=pcm.ctypes.data,
                      stream_stride=2 * 4 * 800, channel_stride=4 * 800, out_db=px.ctypes.data, out_pixels=px.ctypes.data)
    assert L.wf_meter_process(h, C.byref(mb)) == WF_ERR_INVALID_ARG
    mb.out_pixels = None
    mb.out_min = px.ctypes.data
    assert L.wf_meter_process(h, C.byref(mb)) == WF_ERR_INVALID_ARG
    mb.out_min = None
    mb.struct_size = WfMeterBatch.out_pixels.offset  # a caller built against the previous header
    assert L.wf_meter_process(h, C.byref(mb)) == WF_OK
    L.wf_meter_destroy(h)
    assert np.array_equal(MeterEngine({}, channels=2, max_streams=2).process(pcm, 4, 800)["db"], px)
    weng = WaveEngine({}, channels=2, max_streams=2)
    cfg = make_wave_config({}, channels=2, max_streams=2)
    cfg.struct_size = WfWaveConfig.interp_mode.offset
    h = C.c_void_p()
    assert L.wf_wave_create(C.byref(cfg), C.byref(h)) == WF_OK
    out = np.zeros((2, 4, 1, 800), np.float32)
    b = WfWaveBatch(struct_size=C.sizeof(WfWaveBatch), n_streams=2, n_ticks=4, hop=800, pcm=pcm.ctypes.data,
                    stream_stride=2 * 4 * 800, channel_stride=4 * 800, out=out.ctypes.data, out_pixels=out.ctypes.data)
    assert L.wf_wave_process(h, C.byref(b)) == WF_ERR_INVALID_ARG
    b.out_pixels = None
    b.struct_size = WfWaveBatch.out_points.offset  # a caller built against the previous header
    assert L.wf_wave_process(h, C.byref(b)) == WF_OK
    L.wf_wave_destroy(h)
    assert np.array_equal(weng.process(pcm, 4, 800)["out"], out)
