import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Native artefacts are built in-tree (nvcc cross-compiles without a GPU)."""
    from visual_odom_b200 import build
    build.build_native()
    build.build_hostcheck()
    build.build_facade()
    build.build_oracle()
    return True


@pytest.fixture(scope="session")
def ctx(built):
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=8192)
    yield c
    c.close()
