import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle_api():
    from oracle import oracle
    return oracle.load()


@pytest.fixture(scope="session")
def cuda_api():
    import forma_b200
    return forma_b200.load()


@pytest.fixture(scope="session")
def cuda_renderer(cuda_api):
    return cuda_api.Renderer(0)


@pytest.fixture(scope="session")
def oracle_renderer(oracle_api):
    return oracle_api.Renderer(0)


@pytest.fixture()
def unsliced(cuda_api):
    """Host frames rendered as one piece (option host_slices = 1): for tests that inspect the
    stages of the last render (sorted segments, table modes, upload bytes of one renderer) -
    a sliced host frame is rendered by one renderer per slice."""
    saved = cuda_api.get_option("host_slices")
    cuda_api.set_option("host_slices", 1)
    yield
    cuda_api.set_option("host_slices", saved)
