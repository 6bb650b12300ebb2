"""CPU-only checks of int16 PCM in the level-meter and waveform batches: pcm_format is the last field of wf_meter_batch and
wf_wave_batch, where the previous struct ended, the ctypes layouts are the header's, and MeterEngine.process /
WaveEngine.process refuse what pcm_format="s16" cannot read before any call reaches the library."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def _probe(tmp_path, ctype, fields):
    src = tmp_path / f"{ctype}.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   f'int main(){{printf("%zu", sizeof({ctype}));'
                   + "".join(f'printf(" %zu", offsetof({ctype}, {f}));' for f in fields)
                   + 'printf("\\n");return 0;}\n')
    exe = tmp_path / ctype
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


@pytest.mark.parametrize("ctype,cls,prev_last", [("wf_meter_batch", "WfMeterBatch", "out_min"),
                                                  ("wf_wave_batch", "WfWaveBatch", "out_min")])
def test_batch_layout_matches_header(tmp_path, ctype, cls, prev_last):
    import waveform_b200.engine as E

    T = getattr(E, cls)
    fields = [name for name, _ in T._fields_]
    assert fields[-1] == "pcm_format"
    assert _probe(tmp_path, ctype, fields) == [C.sizeof(T)] + [getattr(T, f).offset for f in fields]
    # pcm_format sits at the previous sizeof (the struct a caller of the previous header passes ends there)
    prev = getattr(T, prev_last).offset + C.sizeof(C.c_void_p)
    assert T.pcm_format.offset == prev == 88
    assert C.sizeof(T) == 96


def _engine_without_device(cls, make_cfg, **kw):
    """An engine object with a config but no handle: enough for process() to check its arguments, which it does before
    it reaches the library."""
    eng = cls.__new__(cls)
    eng.cfg = make_cfg(**kw)
    eng.display_channels = 1
    return eng


def _engines():
    from waveform_b200.engine import MeterEngine, WaveEngine, make_meter_config, make_wave_config

    return [_engine_without_device(MeterEngine, make_meter_config, settings={}, channels=1, max_streams=2),
            _engine_without_device(WaveEngine, make_wave_config, settings={}, channels=1, max_streams=2)]


def test_meter_and_wave_pcm_format_argument_errors():
    x16 = np.zeros((2, 1, 4 * 800), np.int16)
    for eng in _engines():
        for bad in ("s32", "int16", None, 1):
            with pytest.raises(ValueError):
                eng.process(x16, 4, 800, pcm_format=bad)
        for bad in (x16.astype(np.float32), x16.astype(np.int32), x16.astype(np.uint16)):
            with pytest.raises(ValueError):
                eng.process(bad, 4, 800, pcm_format="s16")
        with pytest.raises(ValueError):  # too few samples for the ticks, as for float
            eng.process(x16[:, :, :100], 4, 800, pcm_format="s16")


def test_meter_and_wave_pcm_format_errors_for_tensors():
    torch = pytest.importorskip("torch")

    x16 = torch.zeros((2, 1, 4 * 800), dtype=torch.int16)
    for eng in _engines():
        with pytest.raises(ValueError):
            eng.process(x16, 4, 800, pcm_format="s16")  # a CPU tensor
        with pytest.raises(ValueError):
            eng.process(x16.to(torch.float32), 4, 800, pcm_format="s16")
