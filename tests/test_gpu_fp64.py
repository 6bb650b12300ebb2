"""Every spectrum kernel family and FFT plan against the float64 restatement of tick_spectrum (tests/fp64_spectrum.py),
and the level meter's RMS against a float64 sum of squares.

The oracle is a float32 restatement, so a kernel-vs-oracle test cannot say whose error it sees.  Here each kernel is
routed explicitly (environment knobs, asserted through last_kernel_name()), fed the usual noise-plus-sines signal and the
edge signals (impulses at the first and last sample, exact-bin sines at k = 1 and k = B-1, DC, full-scale ±1, input scaled
by 2^-20 and 2^-60), with plain and all options, three hops and a call boundary, and held per frame, in the linear domain,
to normwise < 1e-6 against float64, beyond what the documented float32 approximations cannot avoid (fp64_spectrum.compare:
the dB steps' rounding and the approximate logarithm's error floor, and magnitudes below 1e-19 flushed to zero).
Where the compiled reference has a fixture at that size (tests/golden/fp64_*), the plain noise-plus-sines runs are also
held, on the raw normwise metric the reference was measured with, to at most 4x the reference's own error + 2e-7.  The
linear EMA state from get_state() is held to 1e-6 normwise.

Run on an H100:  python -m pytest tests/test_gpu_fp64.py -m gpu -q
"""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import pytest

from fp64_spectrum import Fp64Spectrum, compare, normwise_vs_truth
from helpers import synth_pcm

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).parent / "golden"
T = 8               # ticks per run, in two calls of 4

FAMILIES = ["stft2048_fast_kernel", "stft2048_team_kernel", "stft_warp2_kernel", "stft_warp2_kernel/display",
            "stft_v3_kernel", "stft16384_parity_kernel", "stft_wide_kernel", "stft_fused_kernel",
            "stft_anyn_kernel/smem", "stft_anyn_kernel/L2"]

# (family, N, channels, stereo, environment, display outputs)
ROUTES = [
    ("stft2048_fast_kernel", 2048, 1, False, {"WF_TEAM_W": "1"}, False),
    ("stft2048_team_kernel", 2048, 1, False, {"WF_TEAM_W": "4"}, False),
    *[("stft_warp2_kernel", n, 1, False, {}, False) for n in (800, 1456, 1664, 1408, 1792)],
    *[("stft_warp2_kernel/display", n, 1, False, {}, True) for n in (800, 1456, 1024)],
    ("stft_v3_kernel", 1024, 1, False, {}, False),
    ("stft_v3_kernel", 2048, 1, False, {"WF_FORCE_GENERIC": "1"}, False),
    ("stft_v3_kernel", 4096, 2, True, {}, False),
    ("stft_v3_kernel", 4096, 2, False, {}, False),
    ("stft_v3_kernel", 8192, 1, False, {}, False),
    ("stft_v3_kernel", 16384, 1, False, {"WF_PAR16384": "0"}, False),
    ("stft16384_parity_kernel", 16384, 1, False, {}, False),
    ("stft_wide_kernel", 4096, 1, False, {"WF_V3": "0", "WF_WIDE_R": "2"}, False),
    ("stft_wide_kernel", 32768, 1, False, {"WF_WIDE_R": "2"}, False),
    *[("stft_fused_kernel", n, 1, False, {}, False) for n in (128, 256, 512)],
    ("stft_fused_kernel", 2048, 1, False, {"WF_FORCE_GENERIC": "1", "WF_V3": "0", "WF_WIDE_R": "1"}, False),
    ("stft_fused_kernel", 32768, 1, False, {"WF_WIDE_R": "1"}, False),
    *[("stft_anyn_kernel/smem", n, 1, False, {"WF_WARP2": "0"}, False) for n in (800, 1456, 1664)],
    ("stft_anyn_kernel/smem", 8128, 1, False, {}, False),
    *[("stft_anyn_kernel/L2", n, 1, False, {}, False) for n in (40000, 65344, 65488, 65536)],
]

SEEN: dict[str, list] = {}      # family -> [(N, max error against float64, error of the reference)]


def _route_id(r):
    fam, N, cc, stereo, env, disp = r
    return f"{fam.replace('/', '-')}-{N}{'-stereo' if stereo else ('-mix' if cc == 2 else '')}"


def _yardstick(N):
    """The compiled reference's own normwise error against float64 at this size (max over the fixture's frames)."""
    from oracle.oraclebind import OracleSource

    for p in GOLDEN.glob("fp64_*.npz"):
        z = np.load(p, allow_pickle=False)
        s = json.loads(str(z["settings"]))
        if s["fft_size"] != N:
            continue
        cc = int(z["channels"])
        truth = Fp64Spectrum(s, channels=cc).run(z["pcm"], int(z["n_frames"]), int(z["hop"]),
                                                 OracleSource(s, channels=cc).gravity(float(z["seconds"])))
        return float(normwise_vs_truth(z["db"], truth["db"], float(z["db_min"])).max())
    return None


def _signals(N, cc, hop):
    """[9, cc, samples] float32: noise + sines, then the edge set."""
    ns = (T - 1) * hop + N
    B = N // 2
    n = np.arange(ns, dtype=np.float64)
    base = synth_pcm(1, cc, ns, seed=0xF64 + N)[0]
    x = np.zeros((9, cc, ns), np.float32)
    x[0] = base
    for t in range(T):                       # an impulse at the first / last sample of every frame
        x[1, :, t * hop] = 1.0
        x[2, :, t * hop + N - 1] = 1.0
    x[3] = (0.5 * np.sin(2 * np.pi * 1 * n / N)).astype(np.float32)         # exact-bin sine, k = 1
    x[4] = (0.5 * np.sin(2 * np.pi * (B - 1) * n / N)).astype(np.float32)   # k = B - 1
    x[5] = 0.25                                                               # DC
    x[6] = np.where(np.random.default_rng(N).uniform(size=(cc, ns)) < 0.5, -1.0, 1.0)   # full scale ±1
    x[7] = base * np.float32(2.0 ** -20)
    x[8] = base * np.float32(2.0 ** -60)    # near the documented flush: |X|·coef ~ 1e-21 ... 4e-19
    return x


def _options(N, all_options):
    if not all_options:
        return {"fft_size": N, "window": "hann"}, None
    return ({"fft_size": N, "window": "blackman_harris", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0,
             "fast_peaks": True, "normalize_volume": True, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5},
            True)


@pytest.mark.parametrize("route", ROUTES, ids=[_route_id(r) for r in ROUTES])
def test_kernel_against_float64(route, monkeypatch):
    import torch
    from waveform_b200 import Engine

    fam, N, cc, stereo, env, disp = route
    for k in ("WF_TEAM_W", "WF_WIDE_R", "WF_V3", "WF_PAR16384", "WF_WARP2", "WF_WARP2_DISPLAY", "WF_FORCE_GENERIC"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    yard = _yardstick(N)
    hops = sorted({N, N // 4} | ({800} if N >= 1024 else set()), reverse=True)
    worst = 0.0
    for hop in hops:
        x = _signals(N, cc, hop)
        S = x.shape[0]
        for all_opt in (False, True):
            settings, _ = _options(N, all_opt)
            if stereo:
                settings["channel_mode"] = "stereo"
            eng = Engine(settings, channels=cc, max_streams=S)
            db_min = float(eng.db_min)
            rng = np.random.default_rng(N + hop)
            secs = rms = skip = None
            if all_opt:
                secs = (1.0 / 60.0 * (0.5 + rng.uniform(size=T))).astype(np.float32)
                rms = (0.02 + 0.3 * rng.uniform(size=(S, T))).astype(np.float32)
                skip = np.zeros((S, T), np.uint8)
                skip[1::2, 5] = 1          # a "not enough audio" tick right after the call boundary on odd streams
                skip[2::3, 2] = 1
            xd = torch.from_numpy(x).cuda()
            outs = []
            for a, b in ((0, 4), (4, T)):
                kw = {}
                if all_opt:
                    kw = dict(frame_seconds=secs[a:b], input_rms=torch.from_numpy(rms[:, a:b].copy()).cuda(),
                              skip_mask=torch.from_numpy(skip[:, a:b].copy()).cuda())
                outs.append(eng.process(xd[:, :, a * hop:].contiguous(), b - a, hop, want_points=disp, **kw))
            torch.cuda.synchronize()
            name = eng.last_kernel_name()
            assert name.startswith(fam.split("/")[0] + "<"), (fam, name)
            assert ("display" in name) == disp, name
            got = torch.cat([o["db"] for o in outs], dim=1).cpu().numpy()
            sil = torch.cat([o["silent"] for o in outs], dim=1).cpu().numpy()
            state = eng.get_state()["tsmooth"]
            gvals = np.array([eng.gravity(float(s)) for s in secs], np.float32) if all_opt else \
                np.float32(eng.gravity(1.0 / 60.0))
            f = Fp64Spectrum(settings, channels=cc)
            slope = f.slope if f.slope is not None else 1.0     # the EMA state carries the slope factor
            for s in range(S):
                f.reset()
                tr = f.run(x[s], T, hop, gvals, input_rms=None if rms is None else rms[s],
                           skip_mask=None if skip is None else skip[s])
                err, bad_floor = compare(got[s], tr, db_min)
                ctx = (fam, N, hop, all_opt, s, name)
                assert not bad_floor, ("DB_MIN above the flush level", ctx)
                assert np.array_equal(sil[s].astype(bool), tr["silent"]), ctx
                assert err.max() < 1e-6, (err.max(), yard, ctx)
                if yard is not None and s == 0 and not all_opt:
                    # the reference's yardstick, on the metric and signal family it was measured with
                    raw = float(normwise_vs_truth(got[s], tr["db"], db_min).max())
                    assert raw <= 4 * yard + 2e-7, (raw, yard, ctx)
                # the linear EMA state after the last tick, per capture channel
                ts, tt = state[s].astype(np.float64) / slope, tr["tsmooth"] / slope
                dstate = np.maximum(np.abs(ts - tt) - tr["tsmooth_flush"] / slope, 0.0).max(axis=-1) / np.maximum(tt.max(axis=-1), 1e-300)
                assert dstate.max() < 1e-6, (dstate.max(), ctx)
                worst = max(worst, float(err.max()), float(dstate.max()))
    SEEN.setdefault(fam, []).append((N, worst, yard))
    print(f"{fam} N={N}: max normwise vs float64 {worst:.2e} (reference {yard if yard is None else f'{yard:.2e}'})")


def test_every_kernel_family_ran(monkeypatch):
    """Each route of ROUTES reaches the kernel family it names, and together they cover every family."""
    import torch
    from waveform_b200 import Engine

    seen = set()
    for fam, N, cc, stereo, env, disp in ROUTES:
        for k in ("WF_TEAM_W", "WF_WIDE_R", "WF_V3", "WF_PAR16384", "WF_WARP2", "WF_WARP2_DISPLAY", "WF_FORCE_GENERIC"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        settings = {"fft_size": N, **({"channel_mode": "stereo"} if stereo else {})}
        eng = Engine(settings, channels=cc, max_streams=2)
        x = torch.from_numpy(synth_pcm(2, cc, 3 * N + N)).cuda()
        eng.process(x, 4, N, want_points=disp)
        torch.cuda.synchronize()
        name = eng.last_kernel_name()
        assert name.startswith(fam.split("/")[0] + "<") and (("display" in name) == disp), (fam, N, name)
        seen.add(fam)
    assert seen == set(FAMILIES), sorted(set(FAMILIES) - seen)
    for fam in FAMILIES:             # the measured table, when the matrix ran in the same session (pytest -s)
        for N, err, yard in SEEN.get(fam, []):
            print(f"| {fam} | {N} | {err:.2e} | {'—' if yard is None else f'{yard:.2e}'} |")


# ---- level meter RMS (wf_meter.cu) against a float64 sum of squares ----

@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("kind,hop", [("rms", 800), ("rms", 700), ("feed", 800), ("feed", 700)])
def test_meter_rms_against_float64(kind, hop, fused, monkeypatch):
    """2000 ticks over several calls: the carried block partials and the ring must not drift.  On every tick the GPU's
    relative error against float64 is at most the oracle's (a single sequential float32 sum, as the reference's generic
    path) + 4 ulp.  Stream 1 goes quiet -> loud -> quiet by 2^-20: a sum carried by subtracting the samples that leave the
    window would show its cancellation there; stream 2 has a stretch of digital silence longer than the window."""
    from oracle.oraclebind import OracleMeter
    from waveform_b200 import MeterEngine
    from waveform_b200.engine import METER_INPUT_RMS

    monkeypatch.setenv("WF_METER_FUSED", fused)
    S, ch, n_ticks = 3, 2, 2000
    settings = {} if kind == "feed" else {"meter_buf": 1000, "rms_mode": True, "temporal_smoothing": "none"}
    eng = MeterEngine(settings, channels=ch, max_streams=S, mode=METER_INPUT_RMS if kind == "feed" else None)
    W = eng.window
    assert W == 48000
    pcm = synth_pcm(S, ch, n_ticks * hop, seed=0x5EED + hop)
    pcm[1, :, : 300 * hop] *= np.float32(2.0 ** -20)
    pcm[1, :, 1300 * hop:] *= np.float32(2.0 ** -20)
    pcm[2, :, 900 * hop: 1100 * hop] = 0.0
    calls = [1, 7, 192, 300, 500, 1000]
    assert sum(calls) == n_ticks
    got, t0 = [], 0
    for n in calls:
        out = eng.process(np.ascontiguousarray(pcm[:, :, t0 * hop:(t0 + n) * hop]), n, hop)
        got.append(out["rms"] if kind == "feed" else out["lin"])
        t0 += n
    got = np.concatenate(got, axis=1).astype(np.float64)
    ulp4 = 4 * 2.0 ** -24
    for s in range(S):
        if kind == "feed":
            sq = np.square(np.abs(pcm[s]).max(axis=0).astype(np.float32)).astype(np.float64)[None]   # val*val in float32
            orc = OracleMeter({}, channels=ch).run(pcm[s], n_ticks, hop, meter=False, rms=True)["rms"][:, None]
        else:
            sq = np.square(pcm[s].astype(np.float64))
            orc = OracleMeter(settings, channels=ch).run(pcm[s], n_ticks, hop)["lin"]
        # each tick's window summed on its own (a running sum would cancel in the quiet stretches)
        truth = np.stack([np.sqrt(sq[:, max(0, e - W): e].sum(axis=1) / W) for e in (np.arange(n_ticks) + 1) * hop])
        g = got[s] if kind != "feed" else got[s][:, None]
        scale = np.maximum(truth, 1e-30)
        e_gpu = np.abs(g - truth) / scale
        e_orc = np.abs(orc.astype(np.float64) - truth) / scale
        live = truth > 0
        over = live & (e_gpu > e_orc + ulp4)
        assert not over.any(), (s, np.argwhere(over)[:5].tolist(), float(e_gpu[over].max()))
        assert np.all(g[~live] == 0.0)
