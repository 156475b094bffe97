import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """The CUDA libraries, the executables and the oracle are (re)built in-tree before anything
    imports them.  `make` is incremental and every target lists its sources and headers, so an
    up-to-date tree costs a few milliseconds and an edited one can never be tested stale."""
    import __graft_entry__

    __graft_entry__.build()


def has_gpu() -> bool:
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False
