import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure; oracle/ is never imported by the product package)."""
    import oracle_py
    oracle_py.build()
    return oracle_py


@pytest.fixture(scope="session")
def gpu_lib():
    from tetris_mcts_b200 import _lib
    L = _lib.lib()
    if L.b200_device_count() < 1:
        pytest.fail("no CUDA device visible but a gpu-marked test was selected")
    return _lib
