import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 GPU (select with -m gpu)")


@pytest.fixture(autouse=True, scope="session")
def _oracle_threads():
    """The torch-CPU oracle is fastest at ~16 intra-op threads (on a 128-thread host all threads are 10x slower)."""
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    yield
