import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (the project targets the H100; select with -m gpu)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with oracle/Makefile."""
    from oracle import pyoracle
    pyoracle.lib()
    # the oracle's many small OpenMP regions crawl on very wide hosts (measured: 128 threads is ~10x slower than 16)
    pyoracle.set_threads(min(16, pyoracle.use_all_cores()))
    return pyoracle


@pytest.fixture(scope="session")
def hb():
    """The product binding.  Raises (does not skip) if libhalide_b200.so is missing."""
    import halide_b200
    halide_b200.load_library()
    return halide_b200
