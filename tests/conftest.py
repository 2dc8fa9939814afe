import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "datafusion-comet_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o
