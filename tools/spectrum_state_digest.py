"""Digest of what the spectrum engine's state calls (wf_get_state / wf_set_state) leave, on every route of the GPU tests'
catalogue, to compare two builds of libwfstft.so byte for byte.

Per route, from seeded inputs: two calls on an engine, get_state, set_state of that into a fresh engine and one more call
on both; then, on an engine with the silence gate, each of the 7 non-empty combinations of tsmooth / hold_db / flags
restored over the engine's own state (hold rows with one display channel at or below floor_db - 10 and the other not),
get_state, one gated call of 4 ticks on digital silence and get_state again.  Every output and state byte goes into the route's
SHA-256, with the engine's launch count and last kernel name after each state call.  Run it once per build (the binding
reads WF_LIB_PATH at import) and compare the JSON lines; `--time` adds the wall time of get_state / set_state of 4096
slots at N=2048 (median of 20 calls, host clock around the blocking call) and the card's name and power limit.

    python tools/spectrum_state_digest.py [--time]
    WF_LIB_PATH=/path/to/other/libwfstft.so python tools/spectrum_state_digest.py [--time]
"""
from __future__ import annotations

import argparse
import hashlib
import itertools
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from gpu_common import CATALOGUE, KNOBS  # noqa: E402
from helpers import synth_pcm  # noqa: E402


def _engine(name, gate):
    from waveform_b200 import Engine

    fam, N, cc, stereo, env, disp = CATALOGUE[name]
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)
    settings = {"fft_size": N, "window": "hann", "silence_gate": gate, **({"channel_mode": "stereo"} if stereo else {})}
    return Engine(settings, channels=cc, max_streams=300 if name.endswith("-split") else 5)


def _route(name):
    fam, N, cc, stereo, env, disp = CATALOGUE[name]
    h = hashlib.sha256()

    def add(*xs):
        for x in xs:
            if isinstance(x, dict):
                add(*(x[k] for k in sorted(x) if x[k] is not None))
            elif isinstance(x, (str, int)):
                h.update(repr(x).encode())
            else:
                h.update(np.ascontiguousarray(x).tobytes())

    def state_call(eng, fn, *args):
        r = fn(*args)
        add(eng.launch_count, eng.last_kernel_name())
        return r

    a, b = _engine(name, False), _engine(name, False)
    S, hop = a.cfg.max_streams, N // 2
    x = synth_pcm(S, cc, 11 * hop + N, seed=0x5747 + N)
    part = [np.ascontiguousarray(x[:, :, 4 * i * hop:4 * i * hop + 3 * hop + N]) for i in range(3)]
    for p in part[:2]:
        add(a.process(p, 4, hop, want_points=disp))
    st = state_call(a, a.get_state)
    add(st)
    state_call(b, b.set_state, st)
    add(a.process(part[2], 4, hop, want_points=disp), b.process(part[2], 4, hop, want_points=disp))
    add(state_call(a, a.get_state), state_call(b, b.get_state))

    g = _engine(name, True)
    add(g.process(part[0], 4, hop, want_points=disp))
    base = state_call(g, g.get_state)
    dch, thr = g.display_channels, np.float32(g.cfg.floor_db - 10)
    hold = base["hold_db"].copy()
    for s in range(S):
        for d in range(dch):
            hold[s, d] = thr - (s % 2) * 7.5
            if (s % 3, d) in ((0, 1), (1, 0)) or (dch == 1 and s % 3 == 1):
                hold[s, d, (7 * s + 3 * d) % hold.shape[-1]] = thr + 0.25
    new = {"tsmooth": base["tsmooth"] * np.float32(0.5), "hold_db": hold,
           "flags": np.array([0xFE, 0x00, 0xFF] * S, np.uint8)[:S]}
    silence = np.zeros((S, cc, 4 * N + 16), np.float32)
    for combo in itertools.product((False, True), repeat=3):
        if not any(combo):
            continue
        state_call(g, g.set_state, base)
        state_call(g, g.set_state, {k: new[k] for k, on in zip(("tsmooth", "hold_db", "flags"), combo) if on})
        add(state_call(g, g.get_state), g.process(silence, 4, N, want_points=disp), state_call(g, g.get_state))
    return h.hexdigest()


def _time():
    from waveform_b200 import Engine

    for k in KNOBS:
        os.environ.pop(k, None)
    S, N = 4096, 2048
    eng = Engine({"fft_size": N, "window": "hann"}, channels=1, max_streams=S)
    eng.process(synth_pcm(S, 1, 2 * N), 2, N)
    st = eng.get_state()
    res = {}
    for what, fn in (("get_state_ms", eng.get_state), ("set_state_ms", lambda: eng.set_state(st))):
        fn()
        ts = []
        for _ in range(20):
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[what] = float(np.median(ts))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    return {**res, "slots": S, "fft_size": N, "gpu": gpu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time", action="store_true")
    args = ap.parse_args()
    from waveform_b200.engine import LIB_PATH

    digests = {name: _route(name) for name in CATALOGUE}
    out = {"lib": str(LIB_PATH), "all": hashlib.sha256(json.dumps(digests, sort_keys=True).encode()).hexdigest(),
           "routes": digests}
    if args.time:
        out["time"] = _time()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
