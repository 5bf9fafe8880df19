import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def built():
    """The product library and the oracle must exist (build() makes both); never fall back silently."""
    from shadernn_b200 import _build, _lib
    if not os.path.exists(_lib.LIB_PATH):
        _build.build()
    from oracle import oracle
    if not os.path.exists(oracle.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build_checker()
    return True


@pytest.fixture(scope="session")
def ctx(built):
    from shadernn_b200.core import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("snn_models"))
