import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: multi-second CPU oracle test")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (oracle/halo2_oracle.c) -- the checker, never the thing under test on the GPU path."""
    from oracle import oracle
    oracle.build()
    oracle.lib()
    return oracle


@pytest.fixture(scope="session")
def kats():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "verifier_kats.json")) as f:
        return json.load(f)
