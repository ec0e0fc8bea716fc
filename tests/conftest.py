import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: pytest -m gpu)')


@pytest.fixture(scope='session')
def built_library():
    """libhmcx.so built in-tree (nvcc cross-compiles without a GPU)."""
    from hamiltorch_b200 import build
    return build.build()
