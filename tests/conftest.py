import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an sm_90 GPU (H100); run with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    import _libs
    return _libs.load_oracle()


@pytest.fixture(scope="session")
def ref():
    import _libs
    if not _libs.have_ref():
        pytest.skip("oracle/_ref/libref.so not built (needs the reference sources; run `make -C oracle ref`)")
    return _libs.load_ref()


@pytest.fixture(scope="session")
def gemm():
    import _libs
    return _libs.load_pkg()
