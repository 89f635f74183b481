import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def cornell():
    from idkengine_b200 import scenes
    return scenes.cornell_1k(threads=1)


@pytest.fixture(scope="session")
def multi_blas():
    from idkengine_b200 import scenes
    return scenes.multi_blas(threads=1)


@pytest.fixture(scope="session")
def atrium_small():
    from idkengine_b200 import scenes
    return scenes.atrium(20000, threads=1)
