import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """The product library and the oracle, built in-tree if missing."""
    import __graft_entry__ as ge
    import hacktv_b200
    if not os.path.exists(hacktv_b200.LIB_PATH) or not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        ge.build()
    return hacktv_b200
