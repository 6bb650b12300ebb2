"""CPU-only checks of the int16 PCM format: wf_batch's layout (pcm_format at the end) and wf_pcm_format as the binding
declares them are the header's, and the Python argument errors of pcm_format."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_batch_layout_matches_header(tmp_path):
    from waveform_b200.engine import PCM_F32, PCM_S16, WfBatch

    fields = [name for name, _ in WfBatch._fields_]
    assert fields[-1] == "pcm_format"
    src = tmp_path / "b.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %d %d", sizeof(wf_batch), (int)WF_PCM_F32, (int)WF_PCM_S16);'
                   + "".join(f'printf(" %zu", offsetof(wf_batch, {f}));' for f in fields)
                   + 'printf("\\n");return 0;}\n')
    exe = tmp_path / "b"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(WfBatch), PCM_F32, PCM_S16] + [getattr(WfBatch, f).offset for f in fields]
    # the previous struct ends where pcm_format begins (that is the size a caller of the previous header passes)
    assert WfBatch.pcm_format.offset == WfBatch.frame_seconds.offset + C.sizeof(C.c_void_p)


def test_pcm_format_argument_errors():
    from waveform_b200.engine import PCM_F32, PCM_S16, _Inputs, _pcm_format

    assert _pcm_format("f32") == PCM_F32 and _pcm_format("s16") == PCM_S16
    for bad in ("s32", "int16", None, 1):
        with pytest.raises(ValueError):
            _pcm_format(bad)
    x16 = np.zeros((2, 1, 64), np.int16)
    for bad in (x16.astype(np.float32), x16.astype(np.int32), x16.astype(np.uint16)):
        with pytest.raises(ValueError):
            _Inputs(bad, 1, 64, s16=True)
    assert _Inputs(x16, 1, 64, s16=True).pcm.dtype == np.int16
    # without the keyword an int16 array is converted to float32 as it is (unscaled), as before
    x = _Inputs(np.full((2, 1, 64), 7, np.int16), 1, 64)
    assert x.pcm.dtype == np.float32 and float(x.pcm.max()) == 7.0


def test_pcm_format_errors_for_tensors():
    torch = pytest.importorskip("torch")
    from waveform_b200.engine import _Inputs

    with pytest.raises(ValueError):
        _Inputs(torch.zeros((2, 1, 64), dtype=torch.int16), 1, 64, s16=True)   # a CPU tensor
