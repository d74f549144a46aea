import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture()
def fp32_mode():
    """Exact-fp32 SIMT convolutions (parity at 1e-5); restored afterwards."""
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision("fp32")
    yield
    ops.set_precision(old)


@pytest.fixture()
def tf32_mode():
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision("tf32")
    yield
    ops.set_precision(old)
