import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RSC = os.path.join(ROOT, "raisimlib_b200", "rsc")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def anymal_tables():
    from oracle.urdf_tables import load_tables
    return load_tables(os.path.join(RSC, "anymal_c_like.urdf"))


@pytest.fixture(scope="session")
def atlas_tables():
    from oracle.urdf_tables import load_tables
    return load_tables(os.path.join(RSC, "atlas_like.urdf"))
