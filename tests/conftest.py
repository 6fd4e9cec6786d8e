import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def fixture_bytes(*parts):
    with open(os.path.join(GOLDEN, *parts), "rb") as f:
        return f.read()


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.build()
    return oracle_lib
