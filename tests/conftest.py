import os, sys, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (oracle/libzkoracle.so) through its ctypes wrapper; built on demand."""
    import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "thin_chunk_proof.json")) as f:
        return json.load(f)
