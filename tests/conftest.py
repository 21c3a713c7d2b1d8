import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built():
    """make sure every native artefact exists (no-op when up to date)"""
    from rsem_b200 import build
    build.build_all()
    return True


@pytest.fixture(scope="session")
def oracle(built):
    import oracle_binding
    return oracle_binding.Oracle()
