import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the native pieces once per session (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_codec.npz"))


@pytest.fixture(scope="session")
def golden_names(golden):
    return sorted({k.split("/")[0] for k in golden.files if "/" in k})


@pytest.fixture
def autorelease():
    objs = []

    def _factory(obj):
        objs.append(obj)
        return obj

    yield _factory
    for o in objs:
        o.close()
