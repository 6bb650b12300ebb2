import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `-m gpu`)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref/libwaveform_ref.so (the compiled reference)")


@pytest.fixture(scope="session", autouse=True)
def _build_oracle():
    """The plain-C oracle is test infrastructure; build it on demand (gcc only)."""
    from oracle import oraclebind
    oraclebind.lib()
