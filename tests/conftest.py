import os
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """CPU oracle (oracle/gnn_oracle.c via ctypes) — test infrastructure only."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle as orc
    orc.build()
    return orc


@pytest.fixture(scope="session")
def gnn():
    import gnnb200
    return gnnb200


@pytest.fixture
def cpu_abi():
    """Run the host-side mirror over tests/fake_abi.py (numpy restatement of the C-ABI contract on host memory) for one
    test.  Host logic only — says nothing about the CUDA kernels."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    with fake_abi.installed() as fake:
        yield fake


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def be(request):
    """back end: .dev (where the mirror's tensors live), .calls (entries the fake saw, None on cuda), .tol (scale)"""
    if request.param == "fake":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import fake_abi
        with fake_abi.installed() as fake:
            yield SimpleNamespace(dev=torch.device("cpu"), calls=fake.calls, tol=1.0)
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), calls=None, tol=4.0)
