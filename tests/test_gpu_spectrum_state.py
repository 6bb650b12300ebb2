"""wf_get_state / wf_set_state of the spectrum engine on every kernel route of gpu_common.CATALOGUE, including the N=2048
fast and team routes, whose hold mirrors stay implicit until a state call writes them out.

- Round trip: a checkpoint of engine A restored into a fresh engine B makes the next call on both bit-identical.
- Flag rule: every non-empty combination of tsmooth / hold_db / flags restores what it names, and restored hold rows set
  the display bits the silence gate reads (bit 2 << d when every bin of display row d is <= floor_db - 10, bit 2 always
  with one display channel).  A gated call on digital silence shows them: a slot whose rows are all below goes silent
  and repeats its rows, one that is not processes the silence as the oracle started from the same state does.
- Ordering: get_state after an asynchronous call on torch's default stream, with no synchronise, reads the state that
  call left.

Run on an H100:  python -m pytest tests/test_gpu_spectrum_state.py -m gpu -q
"""
from __future__ import annotations

import itertools

import numpy as np
import pytest

from gpu_common import CATALOGUE, assert_bits_equal, clean_knobs, set_knobs  # noqa: F401 (fixture)
from helpers import parity_report, synth_pcm

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("clean_knobs")]

NAMES = list(CATALOGUE)
PARTS = ("tsmooth", "hold_db", "flags")
COMBOS = [c for c in itertools.product((False, True), repeat=3) if any(c)]
T = 4  # ticks per call: the N=2048 team kernel needs at least as many as its team has warps


def _engine(name, monkeypatch, gate=False):
    """An engine on the route `name` (300 streams for the split route, which needs more streams than SMs; else 5, which
    keeps the N=2048 team route off the warp-per-stream kernel)."""
    from waveform_b200 import Engine

    fam, N, cc, stereo, env, disp = CATALOGUE[name]
    set_knobs(monkeypatch, env)
    settings = {"fft_size": N, "window": "hann", "silence_gate": gate, **({"channel_mode": "stereo"} if stereo else {})}
    S = 300 if name.endswith("-split") else 5
    return Engine(settings, channels=cc, max_streams=S), settings, S


def _audio(name, S, calls):
    """The PCM of `calls` calls of T ticks at hop N/2 ([S, cc, n] each), and the hop."""
    fam, N, cc, stereo, env, disp = CATALOGUE[name]
    hop = N // 2
    x = synth_pcm(S, cc, (T * calls - 1) * hop + N, seed=0x5747 + N)
    return [np.ascontiguousarray(x[:, :, T * i * hop:T * i * hop + (T - 1) * hop + N]) for i in range(calls)], hop


def _check_route(eng, name):
    fam = CATALOGUE[name].family
    assert eng.last_kernel_name().startswith(fam.split("/")[0] + "<"), (name, eng.last_kernel_name())


@pytest.mark.parametrize("name", NAMES)
def test_checkpoint_round_trip(name, monkeypatch):
    disp = CATALOGUE[name].display
    a, _, S = _engine(name, monkeypatch)
    b, _, _ = _engine(name, monkeypatch)
    xs, hop = _audio(name, S, 3)
    for x in xs[:2]:
        a.process(x, T, hop, want_points=disp)
    _check_route(a, name)
    b.set_state(a.get_state())
    out_a = a.process(xs[2], T, hop, want_points=disp)
    out_b = b.process(xs[2], T, hop, want_points=disp)
    assert_bits_equal(out_b, out_a, (name, "outputs"))
    assert_bits_equal(b.get_state(), a.get_state(), (name, "state"))


def _restore_rows(base, dch, thr):
    """hold_db rows in which, slot by slot (mod 3), display channel 0 lies at or below thr and channel 1 does not, the
    other way round, or both below (one display channel: below, one bin above, below)."""
    hold = base.copy()
    B = hold.shape[-1]
    for s in range(hold.shape[0]):
        below = [(True, False), (False, True), (True, True)][s % 3] if dch == 2 else [(True,), (False,), (True,)][s % 3]
        for d in range(dch):
            hold[s, d] = thr if s % 2 == 0 else thr - 7.5  # exactly at the threshold, or under it
            if not below[d]:
                hold[s, d, (7 * s + 3 * d) % B] = thr + 0.25
    return hold


def _display_bits(hold, dch, thr):
    """The host rule the display bits restate: bit 2 << d when every bin of display row d is <= thr; bit 2 with one
    display channel."""
    bits = np.full(hold.shape[0], 4 if dch == 1 else 0, np.uint8)
    for d in range(dch):
        bits |= np.where((hold[:, d] > thr).any(axis=-1), 0, 2 << d).astype(np.uint8)
    return bits


def _oracle_tick(settings, cc, och, state, s, pcm):
    """The oracle's one gated tick on `pcm` from slot s of `state`."""
    from oracle.oraclebind import OracleSource, _fp

    o = OracleSource(settings, channels=cc)
    if state["flags"][s] & 1:
        o.reset()
    for ch in range(max(cc, och)):
        ts = np.ascontiguousarray(state["tsmooth"][s, ch]) if ch < cc else None
        db = np.ascontiguousarray(state["hold_db"][s, ch]) if ch < och else None
        o.L.wfo_set_state(o.h, ch, _fp(ts), _fp(db))
    return o.run_stft(pcm, 1, pcm.shape[-1])


@pytest.mark.parametrize("name", NAMES)
def test_restore_sets_the_display_bits(name, monkeypatch):
    fam, N, cc, stereo, env, disp = CATALOGUE[name]
    eng, settings, S = _engine(name, monkeypatch, gate=True)
    xs, hop = _audio(name, S, 1)
    eng.process(xs[0], T, hop, want_points=disp)
    # with the gate on, the wide routes take the fused kernel; every gated call here takes the same kernel as this one
    kernel = eng.last_kernel_name().split("<")[0]
    base = eng.get_state()
    assert not (base["flags"] & 1).any()
    dch, och, thr = eng.display_channels, eng.output_channels, np.float32(eng.cfg.floor_db - 10)
    new = {"tsmooth": base["tsmooth"] * np.float32(0.5), "hold_db": _restore_rows(base["hold_db"], dch, thr),
           "flags": np.array([0xFE, 0x00, 0xFF] * S, np.uint8)[:S]}
    silence = np.zeros((S, cc, T * N + 16), np.float32)
    for combo in COMBOS:
        eng.set_state(base)
        part = {k: new[k] for k, on in zip(PARTS, combo) if on}
        eng.set_state(part)
        want = {k: part.get(k, base[k]) for k in PARTS}
        want["flags"] = want["flags"] & 1
        assert_bits_equal(eng.get_state(), want, (name, combo))

        out = eng.process(silence, T, N, want_points=disp)  # the first tick shows the restored state
        assert eng.last_kernel_name().split("<")[0] == kernel, (name, eng.last_kernel_name())
        # a slot goes silent when it was, or when every channel the gate reads shows all rows below
        bits = _display_bits(want["hold_db"], dch, thr)
        gate_bits = 6 if stereo else 2
        silent = (want["flags"] == 1) | ((bits & gate_bits) == gate_bits)
        assert np.array_equal(out["silent"][:, 0].astype(bool), silent), (name, combo)
        for s in range(S):
            if silent[s]:
                assert_bits_equal(out["db"][s, 0], want["hold_db"][s, :dch], (name, combo, s))
            elif s < 5:
                ref = _oracle_tick(settings, cc, och, want, s, silence[s, :, :N + 16])
                assert not ref["silent"][0], (name, combo, s)
                rep = parity_report(out["db"][s, 0], ref["db"][0], db_min=float(eng.db_min))
                assert rep["ok"], (name, combo, s, rep)


def test_get_state_is_ordered_after_work_on_the_default_stream(monkeypatch):
    """A call enqueued on torch's default stream and still running when get_state starts: the state read is the one the
    call leaves, since the state copies wait for the legacy default stream.  N=1024 keeps the call off the N=2048
    kernels, whose implicit hold mirrors get_state writes out on the engine's own stream."""
    import torch

    from waveform_b200 import Engine

    set_knobs(monkeypatch, {})
    S, ticks, N, hop = 4096, 256, 1024, 256
    eng = Engine({"fft_size": N, "window": "hann"}, channels=1, max_streams=S)
    g = torch.Generator(device="cuda").manual_seed(0x0D5)
    x = torch.rand((S, 1, (ticks - 1) * hop + N), generator=g, device="cuda") - 0.5
    before = eng.get_state()
    with torch.cuda.stream(torch.cuda.default_stream()):
        eng.process(x, ticks, hop, want_silent=False)
        got = eng.get_state()
    torch.cuda.synchronize()
    after = eng.get_state()
    assert not np.array_equal(before["tsmooth"], after["tsmooth"])
    assert_bits_equal(got, after, "state")
