"""The knobs the GPU tests reset (gpu_common.KNOBS) are exactly the environment variables the library reads."""
import re
from pathlib import Path

from gpu_common import KNOBS

CSRC = Path(__file__).resolve().parents[1] / "waveform_b200" / "csrc"


def test_knobs_are_every_environment_variable_the_library_reads():
    read = set()
    for p in CSRC.rglob("*"):
        if p.suffix in (".cu", ".cuh", ".cpp", ".hpp", ".h"):
            read |= set(re.findall(r'\b(?:env_flag|env_int|getenv)\(\s*"(\w+)"', p.read_text()))
    assert read == set(KNOBS), (sorted(read - set(KNOBS)), sorted(set(KNOBS) - read))
