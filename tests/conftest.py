import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine that has one)")
    config.addinivalue_line("markers", "slow: long-running (full-size model) test")


@pytest.fixture(scope="session")
def lib():
    from kserve_b200 import _lib
    return _lib.load()
