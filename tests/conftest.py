import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")
    # the C-ABI library must exist before the package can be imported; build it once if it is missing
    if not os.path.exists(os.path.join(ROOT, "diffsensei_b200", "libdsengine.so")):
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))
