import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "moe-infinity_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "shims"),
          os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def lib_built():
    from moe_infinity_b200 import build
    return build.build()
