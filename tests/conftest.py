import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "df-vo_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100)")


@pytest.fixture(scope="session")
def hostsim_lib():
    """CPU emulation build of the library sources (tests/hostsim) -- test infrastructure only."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_hostsim_build", os.path.join(ROOT, "tests", "hostsim", "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    from b200 import native
    return native.Lib(m.build())


@pytest.fixture(scope="session")
def dev_lib():
    """The product library on a real GPU."""
    import torch
    from b200 import native
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return native.load()
