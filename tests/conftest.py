import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "simple-radio-telescope-backend_b200"))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def ctx():
    """one srtb_b200 context on cuda:0, bound to torch's current stream"""
    import torch
    import srtb_b200
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    torch.cuda.set_device(0)
    c = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()
