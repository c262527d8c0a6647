import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "slow: full-size BASELINE.json configs (minutes; still part of -m gpu)")


@pytest.fixture(scope="session")
def manifest():
    return json.load(open(os.path.join(GOLDEN, "manifest.json")))


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def pkg():
    import _pkg
    p = _pkg.load()
    p.build()
    return p


@pytest.fixture(scope="session")
def ctx(pkg):
    c = pkg.Context(0)
    yield c
    c.close()


def golden_path(*parts):
    return os.path.join(GOLDEN, *parts)


def read_golden(*parts):
    with open(golden_path(*parts), "rb") as f:
        return f.read()
