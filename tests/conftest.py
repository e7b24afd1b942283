import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def gs():
    import gs_b200

    return gs_b200


@pytest.fixture(scope="session")
def oracle():
    import oracle as o

    return o


@pytest.fixture(scope="session")
def ctx(gs):
    c = gs.Context(0)
    yield c
    c.close()
