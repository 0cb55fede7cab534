import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree shared library (built on demand on the CPU box; prebuilt on the GPU box)."""
    from controllora_b200.build import LIB, build

    if not LIB.exists():
        build()
    return LIB
