import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")
    if os.environ.get("LC_FAKE_NATIVE") == "1":
        # dry run of the GPU tests' Python half on a machine without a GPU: the CPU oracle stands in for liblc_gpu.so
        # (tests/fake_native.py; proves nothing about the device code)
        from tests import fake_native

        fake_native.install()


@pytest.fixture(scope="session")
def cache():
    """One HBM-resident LiquidCache on cuda:0 for the whole GPU test session."""
    from liquid_cache_b200 import LiquidCacheBuilder

    c = LiquidCacheBuilder.new().build()
    yield c
    c.close()
