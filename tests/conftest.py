import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with `-m gpu`)")


@pytest.fixture(scope="session")
def lib():
    from cambrian_b200 import _lib
    return _lib.load()


def pytest_collection_modifyitems(config, items):
    """CB_TEST_FIRST="substr,substr": run the tests whose node id contains one of the substrings first (a GPU call is short:
    the cases a change touches go first, the rest of the suite follows in its usual order)."""
    first = [t for t in os.environ.get("CB_TEST_FIRST", "").split(",") if t]
    if first:
        items.sort(key=lambda it: 0 if any(t in it.nodeid for t in first) else 1)   # stable: order otherwise unchanged
