import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle.binding import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def refshim():
    """The compiled reference (oracle/_ref). Present in the authoring container and shipped prebuilt
    to the GPU box; tests that need it skip when it is absent."""
    from oracle.binding import RefShim
    try:
        return RefShim(nocontxt=True, maxres=4096)
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"compiled reference not available: {e}")


@pytest.fixture(scope="session")
def hhg():
    import hhsuite_b200
    return hhsuite_b200


@pytest.fixture(scope="session")
def gpu_ctx(hhg):
    ctx = hhg.Context()
    yield ctx
    ctx.close()
