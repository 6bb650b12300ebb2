"""GPU parity at the launch geometries that are actually MEASURED (bench.py, tools/bench_shapes.py), not toy shapes.

The small-shape tests (test_gpu_parity.py) run 1-37 streams, which the N=2048 warp-per-stream kernel maps to one warp
per CTA and one round.  The headline launch is 132 CTAs x 16 warps x 2 rounds with SM-interleaved stream indices and
next-stream TMA prefetch; the CTA-per-tick kernel picks its cluster size from the stream count.  These tests run the
real geometries on the device and compare a strided sample of streams (first / last warp of several CTAs, every round,
plus random ones: >= 64 streams) against the oracle, and every stream against a cheap whole-batch invariant.

Run on an H100:  python -m pytest tests -m gpu -x -q
"""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import pytest

from fp64_spectrum import Fp64Spectrum, compare
from helpers import check_points, device_pcm, parity_report, synth_pcm

pytestmark = pytest.mark.gpu

SMS = 132  # H100 SXM: the N=2048 kernel launches one CTA per SM


def _sample_streams(S: int, n_random: int = 40, seed: int = 1) -> list[int]:
    """Streams at the corners of the N=2048 kernel's decomposition (stream s -> CTA s % SMS, local index s // SMS,
    warp = local % 16, round = local // 16) + the first/last few + random ones."""
    per_cta = (S + SMS - 1) // SMS
    locals_ = sorted({0, 1, 15, 16, 17, per_cta - 2, per_cta - 1} & set(range(per_cta)))
    ctas = [0, 1, 2, SMS // 2 - 1, SMS // 2, SMS - 2, SMS - 1]
    pick = {c + li * SMS for li in locals_ for c in ctas}
    pick |= {0, 1, 2, S - 1, S - 2, S // 2}
    rng = np.random.default_rng(seed)
    pick |= set(int(x) for x in rng.integers(0, S, n_random))
    return sorted(s for s in pick if 0 <= s < S)


def _oracle_rows(settings, channels, pcm_rows, T, hop, want_points=False):
    from oracle.oraclebind import OracleSource

    db, pts, sil = [], [], []
    for row in pcm_rows:
        r = OracleSource(settings, channels=channels).run_stft(row, T, hop, want_points=want_points)
        db.append(r["db"])
        pts.append(r["points"])
        sil.append(r["silent"])
    return np.stack(db), (np.stack(pts) if want_points else None), np.stack(sil)


def _run_and_check(settings, channels, S, T, hop_div=1, zero_every=7, want_points=False, n_random=40, calls=1):
    import torch
    from waveform_b200 import Engine

    eng = Engine(settings, channels=channels, max_streams=S)
    N, cc = eng.fft_size, eng.capture_channels
    hop = N // hop_div
    ns = (T - 1) * hop + N
    pcm = device_pcm(S, cc, ns, seed=0xB200 + S + T, zero_every=zero_every, frame_len=hop)
    if calls == 1:
        out = eng.process(pcm, T, hop, want_points=want_points)
    else:  # the same ticks in `calls` consecutive launches: state, hold and flags cross the call boundary
        parts, t0 = [], 0
        for c in range(calls):
            n = T // calls + (1 if c < T % calls else 0)
            parts.append(eng.process(pcm[:, :, t0 * hop:].contiguous(), n, hop, want_points=want_points))
            t0 += n
        out = {k: torch.cat([p[k] for p in parts], dim=1) for k in parts[0]}
    torch.cuda.synchronize()
    pick = _sample_streams(S, n_random=n_random)
    assert len(pick) >= min(S, 16)
    idx = torch.tensor(pick, device="cuda")
    got_db = out["db"][idx].cpu().numpy()
    got_sil = out["silent"][idx].cpu().numpy()
    ref_db, ref_pts, ref_sil = _oracle_rows(settings, channels, pcm[idx].cpu().numpy(), T, hop, want_points=want_points)
    rep = parity_report(got_db, ref_db, db_min=eng.db_min)
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(got_sil, ref_sil)
    if want_points:
        gp = out["points"][idx].cpu().numpy()
        assert check_points(settings, channels, got_db, gp) < 2e-6
        d = np.abs(gp.astype(np.float64) - ref_pts.astype(np.float64))
        assert np.median(d) < 1e-4 and np.nanmax(d) < 2e-2
    # whole-batch invariants over EVERY stream (cheap, size independent): finite, >= DB_MIN, and no stream left unwritten
    db = out["db"]
    assert bool(torch.isfinite(db).all()) and float(db.min()) >= eng.db_min - 1e-3
    row_max = db.amax(dim=(1, 2, 3))
    audible = pcm[:, :, : ns].abs().amax(dim=(1, 2)) > 0          # a stream of pure digital silence stays at DB_MIN
    assert float(row_max[audible].min()) > -200.0, "a stream's outputs were never written"
    return eng, out, pcm


FAST_SHAPES = [
    # (S, T, calls): 300 -> 3 warps/CTA; 2500 -> 16 warps + a ragged second round; 4096x16 = the bench launch;
    # 65536x1 and 1024x64 = two more layouts of profiles/r0x_layouts.txt; 2113 -> one stream more than 132 x 16; 2369 -> a ragged second round
    (300, 9, 1), (2500, 5, 2), (4096, 16, 1), (2369, 3, 1), (2113, 3, 1), (65536, 1, 1), (1024, 40, 2), (768, 33, 3),
]


@pytest.mark.parametrize("S,T,calls", FAST_SHAPES)
def test_fast2048_parity_at_measured_geometry(S, T, calls, monkeypatch):
    """The warp-per-stream kernel at its real launch geometries (WF_TEAM_W=1 keeps the small shapes on it too)."""
    monkeypatch.setenv("WF_TEAM_W", "1")
    settings = {"fft_size": 2048, "window": "hann", "gravity": 0.65}
    eng, out, _ = _run_and_check(settings, 1, S, T, calls=calls)
    assert eng.last_kernel_name().startswith("stft2048_fast"), eng.last_kernel_name()


@pytest.mark.parametrize("S,T,calls,opts", [
    (4096, 16, 1, {}), (2500, 5, 2, {}), (2369, 3, 1, {}), (8192, 8, 1, {}), (4000, 9, 2, {"slope": 0.5, "fast_peaks": True, "rolloff_q": 1.0, "rolloff_rate": 6.0}),
    (3000, 12, 1, {"gravity": 0.2, "floor": -40}), (2113, 3, 1, {}),
])
def test_fast2048_split_runs_are_bit_identical_to_whole_streams(S, T, calls, opts, monkeypatch):
    """Split mode of the warp-per-stream kernel (an SM's frames cut into 16 equal runs: a stream changes warps mid-call through
    global memory, as it would between two calls) against whole streams per warp (WF_SPLIT=0): every output row, silent flag and
    the state after the call must be identical — streams with silent stretches (gate: decay -> freeze -> wake) included."""
    import torch
    from waveform_b200 import Engine

    monkeypatch.setenv("WF_TEAM_W", "1")
    settings = {"fft_size": 2048, "window": "hann", "gravity": 0.65, **opts}
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("WF_SPLIT", mode)
        eng = Engine(settings, channels=1, max_streams=S)
        pcm = device_pcm(S, 1, (T - 1) * 2048 + 2048, seed=77 + S, zero_every=3, frame_len=2048 * max(1, T // 3))
        parts, t0 = [], 0
        for c in range(calls):
            n = T // calls + (1 if c < T % calls else 0)
            parts.append(eng.process(pcm[:, :, t0 * 2048:].contiguous(), n, 2048, want_peak=bool(opts)))
            t0 += n
        torch.cuda.synchronize()
        assert eng.last_kernel_name().startswith("stft2048_fast"), eng.last_kernel_name()
        res[mode] = ({k: torch.cat([q[k] for q in parts], dim=1) for k in ("db", "silent")}, eng.get_state())
    assert torch.equal(res["1"][0]["db"], res["0"][0]["db"])
    assert torch.equal(res["1"][0]["silent"], res["0"][0]["silent"])
    for key in ("tsmooth", "hold_db", "flags"):
        assert np.array_equal(res["1"][1][key], res["0"][1][key]), key


@pytest.mark.parametrize("N,S,T,points", [(800, 4096, 16, False), (1920, 2500, 5, False), (1456, 3000, 7, False), (800, 4000, 6, True),
                                          (1024, 2500, 5, True)])
def test_warp2_split_runs_are_bit_identical_to_whole_streams(N, S, T, points, monkeypatch):
    """The same equal-runs split in stft_warp2_kernel (non-power-of-two sizes and the display variant, where the first tick of a
    continued stream takes its previous row from the mirror instead of the warp's shared-memory row)."""
    import torch
    from waveform_b200 import Engine

    settings = {"fft_size": N, "window": "hann", "gravity": 0.3, "floor": -40}
    if points:
        settings["interp_mode"] = "catmull_rom"
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("WF_SPLIT", mode)
        eng = Engine(settings, channels=1, max_streams=S)
        pcm = device_pcm(S, 1, T * N, seed=5 + N, zero_every=3, frame_len=N * max(1, T // 3))
        a = eng.process(pcm[:, :, : 2 * N].contiguous(), 2, N, want_points=points, want_pixels=points)
        b = eng.process(pcm[:, :, 2 * N:].contiguous(), T - 2, N, want_points=points, want_pixels=points)
        torch.cuda.synchronize()
        assert eng.last_kernel_name().startswith("stft_warp2"), eng.last_kernel_name()
        res[mode] = ({k: torch.cat([a[k], b[k]], dim=1) for k in a}, eng.get_state())
    for k in res["1"][0]:
        assert torch.equal(res["1"][0][k], res["0"][0][k]), k
    for key in ("tsmooth", "hold_db", "flags"):
        assert np.array_equal(res["1"][1][key], res["0"][1][key]), key


TEAM_SHAPES = [
    # (S, T, calls, W expected): few streams x many ticks (SURVEY §8(d) C3 '256 x 256' family) -> a team of W warps per stream
    # W follows the streams per SM (132 SMs): 1 -> 16, 2 -> 8, 3..8 -> 4
    (256, 64, 2, 8), (512, 48, 2, 4), (132, 48, 3, 16), (1024, 21, 2, 4), (300, 9, 1, 4), (37, 5, 1, 4), (600, 8, 2, 4), (1056, 6, 1, 4),
]


@pytest.mark.parametrize("S,T,calls,W", TEAM_SHAPES)
def test_team2048_parity_and_bit_identity(S, T, calls, W, monkeypatch):
    """wf_team2048.cuh under the engine's own routing: parity against the oracle on the sampled streams, and bit-identical
    outputs / state to the warp-per-stream kernel on EVERY stream (the recurrences are only distributed over bins)."""
    import torch
    from waveform_b200 import Engine

    settings = {"fft_size": 2048, "window": "hann", "gravity": 0.65}
    eng, out, pcm = _run_and_check(settings, 1, S, T, calls=calls)
    assert eng.last_kernel_name().startswith(f"stft2048_team_kernel<{W},"), eng.last_kernel_name()
    monkeypatch.setenv("WF_TEAM_W", "1")
    ref_eng = Engine(settings, channels=1, max_streams=S)
    ref = ref_eng.process(pcm, T, 2048)
    torch.cuda.synchronize()
    assert ref_eng.last_kernel_name().startswith("stft2048_fast")
    assert torch.equal(out["db"], ref["db"]) and torch.equal(out["silent"], ref["silent"])
    a, b = eng.get_state(), ref_eng.get_state()
    for key in ("tsmooth", "hold_db", "flags"):
        assert np.array_equal(a[key], b[key]), key


@pytest.mark.parametrize("W", [4, 8, 16])
def test_team2048_all_options_match_fast_kernel(W, monkeypatch):
    """Slope, fast peaks, roll-off, volume normalisation, skip mask and the peak output through the team kernel's EXTRA
    variant: bit-identical to the warp-per-stream kernel, and within parity of the oracle."""
    import torch
    from waveform_b200 import Engine

    settings = {"fft_size": 2048, "window": "hamming", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "fast_peaks": True,
                "normalize_volume": True, "gravity": 0.4, "floor": -45}
    S, T, N = 21, 35, 2048
    pcm = synth_pcm(S, 1, T * N, zero_frames=[(1, 3, 9), (2, 0, 35), (5, 10, 12), (7, 14, 30)], frame_len=N, hop=N)
    rng = np.random.default_rng(3)
    rms = (0.02 + 0.3 * rng.uniform(size=(S, T))).astype(np.float32)
    skip = (rng.uniform(size=(S, T)) < 0.1).astype(np.uint8)
    x, r, k = torch.from_numpy(pcm).cuda(), torch.from_numpy(rms).cuda(), torch.from_numpy(skip).cuda()
    outs = []
    for w in (W, 1):
        monkeypatch.setenv("WF_TEAM_W", str(w))
        eng = Engine(settings, channels=1, max_streams=S)
        a = eng.process(x[:, :, : 16 * N].contiguous(), 16, N, input_rms=r[:, :16].contiguous(), skip_mask=k[:, :16].contiguous(), want_peak=True)
        b = eng.process(x[:, :, 16 * N:].contiguous(), T - 16, N, input_rms=r[:, 16:].contiguous(), skip_mask=k[:, 16:].contiguous(), want_peak=True)
        torch.cuda.synchronize()
        name = eng.last_kernel_name()
        assert name.startswith(f"stft2048_team_kernel<{w},1>" if w > 1 else "stft2048_fast"), name
        outs.append(({key: torch.cat([a[key], b[key]], dim=1 if key != "peak" else 0).cpu().numpy() for key in ("db", "silent", "peak")},
                     eng.get_state()))
    for key in ("db", "silent", "peak"):
        assert np.array_equal(outs[0][0][key], outs[1][0][key]), key
    for key in ("tsmooth", "hold_db", "flags"):
        assert np.array_equal(outs[0][1][key], outs[1][1][key]), key


V3_SHAPES = [
    # (settings, channels, S, T, hop_div, want_points)
    ({"fft_size": 4096, "window": "hann"}, 1, 1024, 4, 1, False),
    ({"fft_size": 4096, "window": "blackman_harris", "channel_mode": "stereo"}, 2, 1100, 6, 4, False),   # config 2 at scale
    ({"fft_size": 2048, "window": "hann", "channel_mode": "stereo"}, 2, 1200, 3, 1, False),
    ({"fft_size": 8192, "window": "hann", "interp_mode": "lanczos"}, 1, 256, 16, 4, True),               # config 4 shape
    ({"fft_size": 8192, "window": "hann"}, 1, 1024, 3, 1, False),
    ({"fft_size": 16384, "window": "hann"}, 1, 128, 12, 1, False),                                       # config 5 shape (per GPU)
    ({"fft_size": 1024, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 1, 2048, 4, 1, True),
    ({"fft_size": 800, "window": "hann"}, 1, 1500, 4, 1, False),                                         # the automatic size
    ({"fft_size": 1920, "window": "blackman"}, 1, 600, 4, 2, False),
]


@pytest.mark.parametrize("settings,channels,S,T,hop_div,want_points", V3_SHAPES)
def test_other_kernels_parity_at_scale(settings, channels, S, T, hop_div, want_points):
    """>= 1024 streams (cluster size 1) and few-stream shapes (clusters of 2-8 CTAs per stream) of the CTA-per-tick
    kernel, the stereo path, display epilogues and the mixed-radix sizes, all at real stream counts."""
    _run_and_check(settings, channels, S, T, hop_div=hop_div, want_points=want_points, n_random=24, calls=2)


WARP2_DISPLAY_CASES = [
    # (settings, S, T): BASELINE config 1 (N=1024, 26 Catmull-Rom bars), the automatic size with a filtered Lanczos curve,
    # N=2048 curve, a radix-7/13 size with bars, nearest-point interpolation
    ({"fft_size": 1024, "window": "hann", "display_mode": "bars", "interp_mode": "catmull_rom"}, 2048, 6),
    ({"fft_size": 800, "window": "hann", "interp_mode": "lanczos", "filter_mode": "gauss"}, 1500, 5),
    ({"fft_size": 2048, "window": "hann", "interp_mode": "catmull_rom", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0}, 300, 7),
    ({"fft_size": 1456, "window": "blackman", "display_mode": "bars", "interp_mode": "lanczos", "floor": -40, "gravity": 0.2}, 700, 9),
    ({"fft_size": 512, "window": "hann", "interp_mode": "point"}, 37, 4),
]


@pytest.mark.parametrize("settings,S,T", WARP2_DISPLAY_CASES)
def test_warp2_display_variant(settings, S, T, monkeypatch):
    """Display outputs of one-channel sources on the warp-per-stream kernel (stft_warp2_kernel<L,P,display>: the render-time
    stages run per warp on a dB row kept in shared memory): parity of spectrum, points and silent flags with the oracle at
    real stream counts with silent stretches; identical points / pixels / minimum with and without the dB output (the hold
    paths then read the shared-memory row instead of the previous output row); and against the CTA-per-tick / any-N path."""
    import torch
    from waveform_b200 import Engine

    eng, out, pcm = _run_and_check(settings, 1, S, T, want_points=True, n_random=24, calls=2)
    assert "display" in eng.last_kernel_name(), eng.last_kernel_name()
    N = eng.fft_size
    a = Engine(settings, channels=1, max_streams=S).process(pcm, T, N, want_points=True, want_pixels=True)
    e2 = Engine(settings, channels=1, max_streams=S)
    b = e2.process(pcm, T, N, want_db=False, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert "display" in e2.last_kernel_name()
    for key in ("points", "pixels", "min", "silent"):
        assert torch.equal(a[key], b[key]), key
    monkeypatch.setenv("WF_WARP2_DISPLAY", "0")
    e3 = Engine(settings, channels=1, max_streams=S)
    c = e3.process(pcm, T, N, want_points=True, want_pixels=True)
    torch.cuda.synchronize()
    assert "display" not in e3.last_kernel_name()
    assert torch.equal(a["silent"], c["silent"])
    d = (a["points"] - c["points"]).abs()
    assert float(d.median()) < 1e-4 and float(d.max()) < 5e-2, (float(d.median()), float(d.max()))
    dp = (a["pixels"] - c["pixels"]).abs()
    assert float(dp.max()) < 5e-2 * max(1.0, float(c["pixels"].abs().max()) / 100.0), float(dp.max())
    same_min = (a["min"][..., 1] == c["min"][..., 1]).float().mean()
    assert float(same_min) > 0.98, float(same_min)   # the arg-min position can move between two near-equal pixels


GOLD = sorted((Path(__file__).parent / "golden").glob("case_*.npz"))


@pytest.mark.parametrize("team_w", ["1", "0"])
@pytest.mark.parametrize("path", GOLD, ids=[p.stem for p in GOLD])
def test_golden_vectors_spectrum_only(path, team_w, monkeypatch):
    """The reference's golden vectors WITHOUT display outputs: for case_c3_mono_2048_hann this is the headline
    stft2048_fast_kernel (the display-points variant of this test in test_gpu_parity.py routes to the CTA-per-tick kernel)."""
    z = np.load(path, allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    from waveform_b200 import Engine

    monkeypatch.setenv("WF_TEAM_W", team_w)   # "1": warp-per-stream kernel; "0": the engine's routing (one stream -> a team)
    eng = Engine(settings, channels=int(z["channels"]), max_streams=1)
    rms = z["rms"][None, :] if z["rms"].size else None
    out = eng.process(z["pcm"][None], int(z["n_frames"]), int(z["hop"]), seconds=float(z["seconds"]), input_rms=rms)
    rep = parity_report(out["db"][0], z["db"], db_min=float(z["db_min"]))
    assert rep["ok"] and rep["normwise"] < 1e-6, rep
    assert np.array_equal(out["silent"][0], z["silent"])
    if path.stem == "case_c3_mono_2048_hann":
        want = "stft2048_fast" if team_w == "1" else "stft2048_team"
        assert eng.last_kernel_name().startswith(want), eng.last_kernel_name()


@pytest.mark.parametrize("team_w", [1, 4, 8, 16])
@pytest.mark.parametrize("split", [None, 7, 12])
def test_fast2048_gate_decay_freeze_wake(split, team_w, monkeypatch):
    """Decay -> freeze -> wake-up on the warp-per-stream kernel (team_w = 1) and on the team kernel (lazy team-wide gate
    reduction), with the call boundary inside the decay (7) and inside the frozen stretch (12): the next call must see the
    held dB row and both gate flags."""
    monkeypatch.setenv("WF_TEAM_W", str(team_w))
    settings = {"fft_size": 2048, "window": "hann", "gravity": 0.3, "floor": -40}
    S, T, N = 5, 30, 2048
    pcm = synth_pcm(S, 1, T * N)
    pcm[:, :, 4 * N:] = 0.0
    pcm[2, :, 20 * N: 22 * N] = 0.1   # wakes up again
    pcm[4, :, 9 * N: 10 * N] = 0.2    # wakes up while still decaying
    from waveform_b200 import Engine

    eng = Engine(settings, channels=1, max_streams=S)
    if split is None:
        out = eng.process(pcm, T, N)
    else:
        a = eng.process(pcm[:, :, : split * N], split, N)
        b = eng.process(pcm[:, :, split * N:], T - split, N)
        out = {k: np.concatenate([a[k], b[k]], axis=1) for k in ("db", "silent")}
    assert eng.last_kernel_name().startswith("stft2048_fast" if team_w == 1 else f"stft2048_team_kernel<{team_w},"), eng.last_kernel_name()
    ref_db, _, ref_sil = _oracle_rows(settings, 1, pcm, T, N)
    assert ref_sil.sum() > 10 and ref_sil[2, 21] == 0 and ref_sil[2, -1] == 1, "test must exercise freeze and wake-up"
    assert np.array_equal(out["silent"], ref_sil)
    rep = parity_report(out["db"], ref_db, db_min=eng.db_min)
    assert rep["ok"], rep
    s, t = np.argwhere(ref_sil == 1)[3]
    assert np.array_equal(out["db"][s, t], out["db"][s, t - 1])  # held rows are bit-identical copies


STALL = sorted((Path(__file__).parent / "golden").glob("stall_*.npz"))


@pytest.mark.parametrize("device_ptrs", [False, True])
@pytest.mark.parametrize("path", STALL, ids=[p.stem for p in STALL])
def test_skip_mask_against_reference_not_enough_audio(path, device_ptrs):
    """A real, non-zero skip_mask: the ticks on which the compiled reference had 'not enough audio'
    (src/source_generic.cpp:55-61; fixtures from tests/golden/make_golden.py --stall-only).  While a channel is skipped
    with m_last_silent == false the reference pushes the stale dB values through dbfs() again (:138-159)."""
    import torch
    from test_oracle_golden import stall_calls
    from waveform_b200 import Engine

    z = np.load(path, allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    eng = Engine(settings, channels=int(z["channels"]), max_streams=3)
    hop = int(z["hop"])
    dbs, sils = [], []
    for pcm, n, skip in stall_calls(z):
        # three streams: 0 and 2 follow the fixture, stream 1 is never skipped (the mask is per stream and tick)
        batch = np.ascontiguousarray(np.stack([pcm, pcm, pcm]))
        mask = np.stack([skip, np.zeros_like(skip), skip])
        if device_ptrs:
            out = eng.process(torch.from_numpy(batch).cuda(), n, hop, seconds=float(z["seconds"]),
                              skip_mask=torch.from_numpy(mask).cuda())
            torch.cuda.synchronize()
            out = {k: v.cpu().numpy() for k, v in out.items()}
        else:
            out = eng.process(batch, n, hop, seconds=float(z["seconds"]), skip_mask=mask)
        dbs.append(out["db"])
        sils.append(out["silent"])
    db, sil = np.concatenate(dbs, axis=1), np.concatenate(sils, axis=1)
    skipped = np.concatenate([s for _, _, s in stall_calls(z)]).astype(bool)
    assert skipped.sum() >= 2
    for s in (0, 2):
        rep = parity_report(db[s], z["db"], db_min=float(z["db_min"]))
        assert rep["ok"] and rep["normwise"] < 1e-6, (s, rep)
        assert np.array_equal(sil[s], z["silent"])
        assert (db[s][skipped] <= float(z["db_min"]) + 1e-3).all()      # stale dB -> dbfs() -> DB_MIN
    assert (db[1][skipped].max(axis=(-1, -2)) > -100).all()             # the unmasked stream kept going


def test_fp64_arbiter_gpu_and_reference_errors():
    """SURVEY §4(ii)/§7: both implementations' error against a double-precision ground truth.  The CUDA path must be as
    close to the truth as the reference's own FFTW path is (both are fp32 FFTs; normwise ~1e-7), on the golden PCM."""
    z = np.load(Path(__file__).parent / "golden" / "case_c3_mono_2048_hann.npz", allow_pickle=False)
    settings = json.loads(str(z["settings"]))
    from waveform_b200 import Engine

    T, hop = int(z["n_frames"]), int(z["hop"])
    eng = Engine(settings, channels=1, max_streams=1)
    got = eng.process(z["pcm"][None], T, hop, seconds=float(z["seconds"]))["db"][0, :, 0]
    truth = Fp64Spectrum(settings, channels=1).run(z["pcm"], T, hop, eng.gravity(float(z["seconds"])))["db"][:, 0]
    lin = lambda d: np.power(10.0, np.asarray(d, np.float64) / 20.0)
    peak = lin(truth).max(axis=-1, keepdims=True)
    err_gpu = (np.abs(lin(got) - lin(truth)) / peak).max()
    err_ref = (np.abs(lin(z["db"][:, 0]) - lin(truth)) / peak).max()
    assert err_ref < 1e-6 and err_gpu < 1e-6, (err_gpu, err_ref)
    assert err_gpu < 4 * err_ref + 2e-7, (err_gpu, err_ref)
    # and in dB on the bins that matter (within 60 dB of the frame peak)
    strong = lin(truth) >= peak * 1e-3
    assert np.abs(got - truth)[strong].max() < 1e-3


WARP2_SIZES = [400, 720, 800, 960, 1456, 1600, 640, 1152, 1280, 1536, 1792, 1920, 192, 320, 384, 448, 576, 704, 768, 832, 896,
               1344, 1408, 1664, 1728, 880, 480, 528, 352, 288]


@pytest.mark.parametrize("N", WARP2_SIZES)
def test_warp2_nonpow2_sizes_parity(N, monkeypatch):
    """wf_warp2.cuh (two register-DFT passes per warp: radix 2/3/5/7/13 butterflies) for the plugin's non-power-of-two
    sizes: parity against the oracle (plain and all-options settings, gate, call boundary) and agreement with the
    first-generation any-N kernel."""
    import torch
    from waveform_b200 import Engine

    for settings in ({"fft_size": N, "window": "hann", "gravity": 0.3, "floor": -40},
                     {"fft_size": N, "window": "blackman_harris", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0,
                      "fast_peaks": True, "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5}):
        S, T = 37, 26
        pcm = synth_pcm(S, 1, T * N, zero_frames=[(1, 3, 7), (2, 0, 26), (5, 4, 26)], frame_len=N, hop=N)
        pcm[5, :, 20 * N: 21 * N] = 0.1
        x = torch.from_numpy(pcm).cuda()
        eng = Engine(settings, channels=1, max_streams=S)
        a = eng.process(x[:, :, : 9 * N].contiguous(), 9, N)
        b = eng.process(x[:, :, 9 * N:].contiguous(), T - 9, N)
        torch.cuda.synchronize()
        assert eng.last_kernel_name().startswith("stft_warp2_kernel<"), eng.last_kernel_name()
        got = torch.cat([a["db"], b["db"]], dim=1).cpu().numpy()
        sil = torch.cat([a["silent"], b["silent"]], dim=1).cpu().numpy()
        ref_db, _, ref_sil = _oracle_rows(settings, 1, pcm, T, N)
        rep = parity_report(got, ref_db, db_min=eng.db_min)
        assert rep["ok"], (settings, rep)
        # every stream (gate, zero frames, stream 5's constant frame) against float64: the warp2 plans, radix 7 / 13
        # included, are held to the same 1e-6 as every other kernel (tests/test_gpu_fp64.py)
        f = Fp64Spectrum(settings, channels=1)
        for s in range(S):
            f.reset()
            tr = f.run(pcm[s], T, N, eng.gravity(1.0 / 60.0))
            err, bad_floor = compare(got[s], tr, eng.db_min)
            assert err.max() < 1e-6 and not bad_floor, (settings, s, err.max())
            assert np.array_equal(sil[s].astype(bool), tr["silent"]), (settings, s)
        assert np.array_equal(sil, ref_sil) and ref_sil.sum() > 10
        monkeypatch.setenv("WF_WARP2", "0")
        old = Engine(settings, channels=1, max_streams=S)
        c = old.process(x, T, N)
        torch.cuda.synchronize()
        monkeypatch.delenv("WF_WARP2")
        assert old.last_kernel_name().startswith("stft_anyn"), old.last_kernel_name()
        rep2 = parity_report(got, c["db"].cpu().numpy(), db_min=eng.db_min)
        assert rep2["ok"], rep2
        assert np.array_equal(sil, c["silent"].cpu().numpy())


@pytest.mark.parametrize("N,S,team_w", [(2048, 3, "1"), (2048, 3, "0"), (4096, 2, "0"), (4096, 160, "0"), (800, 3, "0"), (4160, 2, "0"),
                                         (512, 3, "0"), (32768, 2, "0")])
def test_per_tick_seconds_tv_exponential(N, S, team_w, monkeypatch):
    """wf_batch.frame_seconds: the reference evaluates get_gravity(seconds) on every tick (src/source.hpp:301-312); a batch
    recorded with jittering frame times replays exactly.  Every kernel family, against the oracle ticked with the same times."""
    from oracle.oraclebind import OracleSource
    from waveform_b200 import Engine

    monkeypatch.setenv("WF_TEAM_W", team_w)
    settings = {"fft_size": N, "window": "hann", "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5}
    T = 12
    rng = np.random.default_rng(11)
    secs = (1.0 / 60.0 * (0.4 + 1.6 * rng.uniform(size=T))).astype(np.float32)
    pcm = synth_pcm(min(S, 3), 1, T * N)
    if S > 3:
        pcm = np.tile(pcm, ((S + 2) // 3, 1, 1))[:S]
    eng = Engine(settings, channels=1, max_streams=S)
    out = eng.process(pcm, T, N, frame_seconds=secs)
    const = Engine(settings, channels=1, max_streams=S).process(pcm, T, N, seconds=float(secs[0]))
    assert not np.array_equal(out["db"], const["db"])          # the table is really used ...
    assert np.array_equal(out["db"][:, 0], const["db"][:, 0])  # ... and tick 0 agrees with the scalar path
    for s in range(min(S, 3)):
        o = OracleSource(settings, channels=1)
        for t in range(T):
            o.tick([pcm[s, 0, t * N:(t + 1) * N]], float(secs[t]))
            rep = parity_report(out["db"][s, t], np.stack([o.decibels(0)]), db_min=eng.db_min)
            assert rep["ok"] and rep["normwise"] < 1e-6, (eng.last_kernel_name(), s, t, rep)


@pytest.mark.parametrize("variant", ["plain", "options", "odd_hop"])
def test_par16384_bin_parity_cluster(variant, monkeypatch):
    """wf_par16384.cuh (N = 16384: a cluster of two CTAs per stream, even / odd bins, each on the N=8192 plan): parity against
    the oracle incl. the gate's freeze / wake-up across a call boundary (cluster-wide flag reduction), skip mask, per-tick
    gravity, the option set and the peak output; agreement with the CTA-per-tick kernel it replaces."""
    import torch
    from waveform_b200 import Engine

    N = 16384
    if variant == "options":
        settings = {"fft_size": N, "window": "blackman_harris", "slope": 0.5, "rolloff_q": 1.0, "rolloff_rate": 6.0, "fast_peaks": True,
                    "temporal_smoothing": "tv_exp_moving_avg", "gravity": 0.5, "normalize_volume": True}
    else:
        settings = {"fft_size": N, "window": "hann", "gravity": 0.3, "floor": -40}
    hop = N if variant != "odd_hop" else 4097   # an odd hop: scalar loads instead of 64-bit ones
    S, T = 7, 24
    pcm = synth_pcm(S, 1, (T - 1) * hop + N, zero_frames=[(1, 3, 7), (2, 0, 24), (5, 4, 24)], frame_len=N, hop=hop)
    if variant != "odd_hop":
        pcm[5, :, 18 * N: 19 * N] = 0.1
    rng = np.random.default_rng(4)
    rms = (0.02 + 0.3 * rng.uniform(size=(S, T))).astype(np.float32) if variant == "options" else None
    secs = (1.0 / 60.0 * (0.5 + rng.uniform(size=T))).astype(np.float32) if variant == "options" else None
    skip = (rng.uniform(size=(S, T)) < 0.08).astype(np.uint8) if variant == "options" else None
    x = torch.from_numpy(pcm).cuda()
    outs = {}
    for name, flag in (("par", "1"), ("v3", "0")):
        monkeypatch.setenv("WF_PAR16384", flag)
        eng = Engine(settings, channels=1, max_streams=S)

        def kw(a, b):
            return dict(input_rms=None if rms is None else torch.from_numpy(rms[:, a:b].copy()).cuda(),
                        skip_mask=None if skip is None else torch.from_numpy(skip[:, a:b].copy()).cuda(),
                        frame_seconds=None if secs is None else secs[a:b], want_peak=True)
        a = eng.process(x[:, :, : 8 * hop + N].contiguous(), 9, hop, **kw(0, 9))
        b = eng.process(x[:, :, 9 * hop:].contiguous(), T - 9, hop, **kw(9, T))
        torch.cuda.synchronize()
        want = "stft16384_parity_kernel" if name == "par" else "stft_v3_kernel<16384"
        assert eng.last_kernel_name().startswith(want), eng.last_kernel_name()
        outs[name] = ({k: torch.cat([a[k], b[k]], dim=1 if k != "peak" else 0).cpu().numpy() for k in ("db", "silent", "peak")},
                      eng.get_state())
    got, st = outs["par"]
    assert np.array_equal(got["silent"], outs["v3"][0]["silent"])
    rep = parity_report(got["db"], outs["v3"][0]["db"], db_min=-758.0)
    assert rep["ok"], rep
    assert np.allclose(got["peak"], outs["v3"][0]["peak"], atol=2e-3)
    assert np.array_equal(st["flags"], outs["v3"][1]["flags"])
    if variant != "options":
        ref_db, _, ref_sil = _oracle_rows(settings, 1, pcm, T, hop)
        assert np.array_equal(got["silent"], ref_sil) and ref_sil.sum() > 10
        rep = parity_report(got["db"], ref_db, db_min=-758.0)
        assert rep["ok"] and rep["normwise"] < 2e-6, rep
        assert parity_report(st["hold_db"][:, 0], ref_db[:, -1, 0], db_min=-758.0)["ok"]   # m_decibels mirror after the call


def test_zero_copy_live_path_equals_staged_path(monkeypatch):
    """wf_host_alloc: a small batch whose buffers all live in page-locked, device-mapped host memory is processed in place
    (one launch, no staging copies — the live tick of host/source_cuda.hpp); the same call with WF_ZERO_COPY=0, and with
    pageable numpy buffers, must give identical bits.  A batch above 1 MiB of PCM in the same kind of memory is staged."""
    import ctypes as C
    from waveform_b200 import Engine

    N, cc = 4096, 2
    settings = {"fft_size": N, "channel_mode": "stereo", "window": "blackman_harris"}
    pcm = synth_pcm(1, cc, 6 * N, seed=2)[0]
    outs = {}
    for name, zc in (("zero_copy", "1"), ("staged", "0")):
        monkeypatch.setenv("WF_ZERO_COPY", zc)
        eng = Engine(settings, channels=cc, max_streams=1)
        L, B, dch = eng.L, eng.bins, eng.display_channels
        pin = L.wf_host_alloc(cc * N * 4)
        pout = L.wf_host_alloc(dch * B * 4)
        pfl = L.wf_host_alloc(16)
        assert pin and pout and pfl
        rows = []
        launches0 = eng.launch_count
        for t in range(6):
            frame = np.ascontiguousarray(pcm[:, t * N:(t + 1) * N])
            C.memmove(pin, frame.ctypes.data, frame.nbytes)
            C.memset(pfl, 0, 16)
            eng.process_raw(pin, 1, 1, N, cc * N, N, out_db=pout, out_silent=pfl + 1, skip_mask=pfl)
            rows.append(np.ctypeslib.as_array(C.cast(pout, C.POINTER(C.c_float)), shape=(dch, B)).copy())
        outs[name] = np.stack(rows)
        assert eng.launch_count - launches0 == 6
        for q in (pin, pout, pfl):
            L.wf_host_free(q)
    assert np.array_equal(outs["zero_copy"], outs["staged"])
    ref = Engine(settings, channels=cc, max_streams=1).process(pcm[None], 6, N)["db"][0]
    assert np.array_equal(outs["zero_copy"], ref)


@pytest.mark.parametrize("seed", range(24))
def test_randomised_configs_against_oracle(seed):
    """Differential fuzz over the whole dispatch table: random size (powers of two, mixed-radix plans, sizes without a plan),
    window, channel mode, smoothing, options, hop, stream / tick counts (which select warp / team / cluster kernels), silent
    stretches, skip masks, per-tick frame times and call boundaries — every draw must match the oracle tick for tick."""
    from oracle.oraclebind import OracleSource
    from waveform_b200 import Engine

    rng = np.random.default_rng(1000 + seed)
    N = int(rng.choice([128, 512, 1024, 2048, 2048, 4096, 8192, 16384, 800, 720, 1600, 1920, 1456, 352, 2000, 4160, 1088]))
    mode = str(rng.choice(["mono", "mono", "stereo"]))
    channels = 2 if mode == "stereo" or rng.uniform() < 0.25 else 1
    settings = {"fft_size": N, "channel_mode": mode,
                "window": str(rng.choice(["none", "hann", "hamming", "blackman", "blackman_harris", "power_of_sine"])),
                "temporal_smoothing": str(rng.choice(["none", "exp_moving_avg", "exp_moving_avg", "tv_exp_moving_avg"])),
                "gravity": float(rng.choice([0.2, 0.5, 0.65, 0.9])), "floor": int(rng.choice([-30, -45, -65]))}
    if rng.uniform() < 0.3:
        settings.update(slope=float(rng.choice([0.25, 1.0])), fast_peaks=bool(rng.uniform() < 0.5))
    if rng.uniform() < 0.3:
        settings.update(rolloff_q=1.0, rolloff_rate=float(rng.choice([3.0, 9.0])))
    hop = int(N // int(rng.choice([1, 1, 2, 4]))) if rng.uniform() < 0.8 else int(rng.integers(N // 4, N)) // 2 * 2 + 1  # odd hop sometimes
    S = int(rng.choice([1, 3, 9, 40, 170]))
    T = int(rng.choice([1, 5, 11, 23]))
    eng = Engine(settings, channels=channels, max_streams=S)
    cc = eng.capture_channels
    ns = (T - 1) * hop + N
    pcm = synth_pcm(min(S, 6), cc, ns, seed=seed)
    for s in range(pcm.shape[0]):       # silent stretches: decay, freeze, wake-up
        if rng.uniform() < 0.6:
            a = int(rng.integers(0, ns // 2))
            pcm[s, :, a: a + int(rng.integers(N, 4 * N + 1))] = 0.0
    if S > pcm.shape[0]:
        pcm = np.concatenate([pcm] * (-(-S // pcm.shape[0])))[:S]
    skip = (rng.uniform(size=(S, T)) < 0.1).astype(np.uint8) if rng.uniform() < 0.3 else None
    secs = (1.0 / 60.0 * (0.5 + rng.uniform(size=T))).astype(np.float32) if rng.uniform() < 0.4 else None
    cut = int(rng.integers(1, T)) if T > 1 and rng.uniform() < 0.6 else None
    if cut is None:
        out = eng.process(pcm, T, hop, skip_mask=skip, frame_seconds=secs)
        db, sil = out["db"], out["silent"]
    else:
        a = eng.process(pcm[:, :, : (cut - 1) * hop + N], cut, hop, skip_mask=None if skip is None else skip[:, :cut],
                        frame_seconds=None if secs is None else secs[:cut])
        b = eng.process(pcm[:, :, cut * hop:], T - cut, hop, skip_mask=None if skip is None else skip[:, cut:],
                        frame_seconds=None if secs is None else secs[cut:])
        db, sil = np.concatenate([a["db"], b["db"]], axis=1), np.concatenate([a["silent"], b["silent"]], axis=1)
    kernel = eng.last_kernel_name()
    for s in sorted(set([0, S // 2, S - 1])):
        o = OracleSource(settings, channels=channels)
        for t in range(T):
            frames = [None if (skip is not None and skip[s, t]) else pcm[s, c, t * hop: t * hop + N] for c in range(cc)]
            o.tick(frames, float(secs[t]) if secs is not None else 1.0 / 60.0)
            ref = np.stack([o.decibels(d) for d in range(o.display_channels)])
            rep = parity_report(db[s, t], ref, db_min=eng.db_min)
            # `ok` is the parity criterion; the normwise bound only guards against gross errors here (two independent fp32
            # FFTs on frames with inserted silence: up to 2.1e-6 seen, typical 4e-7)
            assert rep["ok"] and rep["normwise"] < 5e-6, (kernel, settings, S, T, hop, s, t, rep)
            assert bool(sil[s, t]) == o.last_silent, (kernel, settings, S, T, hop, s, t)
