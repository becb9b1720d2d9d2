import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


@pytest.fixture(scope="session")
def models_dir():
    return os.path.join(ROOT, "tests", "golden", "models")


@pytest.fixture(scope="session")
def port_default(models_dir):
    from oracle.portbind import Port
    return Port(os.path.join(models_dir, "default.bin"))
