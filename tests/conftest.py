import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Compile the native engine and the oracle checkers once per session (no-op when up to date)."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def oracles():
    import oracle
    return {"port": oracle.Oracle("port"), "ref": oracle.reference()}     # "ref": compiled reference, or its stored outputs


@pytest.fixture(scope="session")
def ora():
    """Strongest checker available: compiled reference headers if present, else the port."""
    import oracle
    return oracle.best()
