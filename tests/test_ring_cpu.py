"""CPU-only checks of capture-ring calls: wf_batch.capture_ring's place in the header (the previous struct's tail padding,
so sizeof(wf_batch) is unchanged), the binding's view of it, and the argument checks that need no device."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_capture_ring_layout_matches_header(tmp_path):
    from waveform_b200.engine import WfBatch

    src = tmp_path / "b.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %u\\n", sizeof(wf_batch), offsetof(wf_batch, capture_ring),'
                   ' offsetof(wf_batch, pcm_format), (unsigned)WF_CAPTURE_RING);return 0;}\n')
    exe = tmp_path / "b"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    size, ring, fmt, magic = (int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    from waveform_b200.engine import CAPTURE_RING
    assert magic == CAPTURE_RING
    assert size == C.sizeof(WfBatch) and fmt == WfBatch.pcm_format.offset
    assert ring == fmt + 4 and ring + 4 == size  # the 4 bytes after pcm_format, inside the unchanged size


def test_capture_ring_property():
    from waveform_b200.engine import WfBatch

    from waveform_b200.engine import CAPTURE_RING

    b = WfBatch()
    assert b.capture_ring == 0
    b.pcm_format = 1
    b.capture_ring = CAPTURE_RING
    raw = bytes(b)
    off = WfBatch.pcm_format.offset
    assert raw[off: off + 8] == (1).to_bytes(4, "little") + b"ring"
    assert b.pcm_format == 1 and b.capture_ring == CAPTURE_RING
    b.capture_ring = 0
    assert b.pcm_format == 1 and b.capture_ring == 0


def test_ring_entry_points_without_engine():
    from waveform_b200.engine import WF_ERR_INVALID_ARG, load_library

    L = load_library()
    buf = np.zeros(16, np.float32)
    assert L.wf_get_ring(None, 0, 1, buf.ctypes.data) == WF_ERR_INVALID_ARG
    assert L.wf_set_ring(None, 0, 1, buf.ctypes.data) == WF_ERR_INVALID_ARG



def _packets_vs_plain(N, cc, settings, calls, seed):
    """The plugin itself, fed packet by packet from the first tick on (its start-up zeros in the capture rings), against
    the plugin fed plain frames over zeros(N) ++ samples from offset hop, one run per call at the matching offsets."""
    from helpers import synth_pcm
    from oracle import refbind

    total = sum(t * h for t, h in calls)
    x = synth_pcm(1, cc, total, seed=seed)[0]
    x[:, total // 3: total // 3 + N] = 0.0  # digital silence: the gate and m_last_silent
    full = np.concatenate([np.zeros((cc, N), np.float32), x], axis=1)
    pk = refbind.RefSource(settings, channels=cc)
    plain = refbind.RefSource(settings, channels=cc)
    dch = pk.display_channels
    pos = 0
    for T_, hop in calls:
        got_db, got_sil = [], []
        for t in range(T_):
            seg = x[:, pos + t * hop: pos + (t + 1) * hop]
            pk.advance(hop / pk.sample_rate)
            pk.push(seg[0], seg[1] if cc == 2 else None)
            pk.tick(1.0 / 60.0)
            got_db.append(np.stack([pk.decibels(c) for c in range(dch)]))
            got_sil.append(1 if pk.last_silent else 0)
        want = plain.run_stft(full[:, pos + hop: pos + hop + (T_ - 1) * hop + N], T_, hop)
        assert want["frames"] == T_
        assert np.array_equal(np.stack(got_db), want["db"]), (N, T_, hop)
        assert np.array_equal(np.array(got_sil, np.uint8), want["silent"]), (N, T_, hop)
        pos += T_ * hop


@pytest.mark.parametrize("N,cc,stereo,window", [(800, 1, False, "hann"), (2048, 1, False, "hann"),
                                                 (4096, 2, True, "blackman_harris")])
def test_ring_model_is_the_plugins(N, cc, stereo, window):
    """What a capture-ring call computes (start-up zeros, then the newest N samples of ring ++ new at every tick) is what
    the compiled plugin computes when packets of `hop` samples arrive, with hops below, equal to and above N, changing
    between calls."""
    from oracle import refbind

    if not refbind.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    settings = {"fft_size": N, "window": window, "silence_gate": True}
    if stereo:
        settings["channel_mode"] = "stereo"
    _packets_vs_plain(N, cc, settings, [(3, 800), (1, 800), (2, N), (1, N + 400), (4, 512)], 0x716 + N)
