import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


def pytest_sessionstart(session):
    """Build the in-tree artefacts if they are missing or stale (nvcc cross-compiles without a GPU; gcc for the oracle)."""
    from pigo_b200 import build
    build.build()
    import oracle_lib
    oracle_lib.build()


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", "oracle_vectors.npz"))


@pytest.fixture(scope="session")
def sample_gray():
    from pigo_b200 import synth
    return synth.sample_gray()


@pytest.fixture(scope="session")
def facefinder_bytes():
    import pigo_b200
    return pigo_b200.load_cascade("facefinder")


@pytest.fixture(scope="session")
def oracle_face(facefinder_bytes):
    import oracle_lib
    return oracle_lib.OracleFace(facefinder_bytes)


@pytest.fixture(scope="session")
def gpu_face(facefinder_bytes):
    import pigo_b200
    return pigo_b200.NewPigo().Unpack(facefinder_bytes)
