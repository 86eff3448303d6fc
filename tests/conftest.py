"""pytest configuration: `gpu` marker, package/oracle fixtures."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    import __graft_entry__ as ge
    return ge.load_package()


@pytest.fixture(scope="session")
def native(pkg):
    """The loaded native shim.  Fails loudly (no fallback) when it is not built / not loadable."""
    pkg.load()
    return pkg


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle as o
    o.build()
    return o


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test ran without a CUDA device")
    return torch.device("cuda:0")
