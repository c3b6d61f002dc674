import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); deselect with -m \"not gpu\" on a machine without one")


def pytest_collection_modifyitems(config, items):
    # GPU tests never silently pass on a CPU box: they are deselected by `-m "not gpu"`, and if
    # someone runs them without a device they fail loudly inside the library (B200_ERR_NO_DEVICE).
    pass


@pytest.fixture(scope="session")
def engine_lib():
    from kubeai_b200 import lib
    return lib()
