"""CPU-only checks of wf_render's C ABI: the wf_render_batch layout the binding uses is the header's, and the library
exports wf_render."""
import ctypes as C
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def test_render_batch_layout_matches_header(tmp_path):
    from waveform_b200.engine import WfRenderBatch

    fields = [name for name, _ in WfRenderBatch._fields_]
    src = tmp_path / "rb.c"
    src.write_text('#include "wfstft.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu", sizeof(wf_render_batch));'
                   + "".join(f'printf(" %zu", offsetof(wf_render_batch, {f}));' for f in fields)
                   + 'printf("\\n");return 0;}\n')
    exe = tmp_path / "rb"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(WfRenderBatch)] + [getattr(WfRenderBatch, f).offset for f in fields]


def test_wf_render_is_exported():
    from waveform_b200.engine import EXPORTS, load_library

    assert "wf_render" in EXPORTS
    L = load_library()
    assert hasattr(L, "wf_render") and L.wf_abi_version() == 2


def test_wf_render_rejects_bad_handles_without_a_device():
    """Argument errors come before any device work: a null engine or batch is WF_ERR_INVALID_ARG."""
    from waveform_b200.engine import WF_ERR_INVALID_ARG, WfRenderBatch, load_library

    L = load_library()
    rb = WfRenderBatch()
    rb.struct_size = C.sizeof(WfRenderBatch)
    assert L.wf_render(None, C.byref(rb), None) == WF_ERR_INVALID_ARG
