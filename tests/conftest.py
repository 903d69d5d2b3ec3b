import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu)")
    config.addinivalue_line("markers", "gpu_unverified: CUDA test of a component that has not had its first run on the GPU yet; "
                                       "NOT part of `-m gpu` (skips itself without CUDA) -- promote to `gpu` after the first green run (none parked at the moment)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
