import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref/libgstref.so (the compiled reference)")


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    from oracle import bindings
    have_ref = bindings.have_ref()
    have_gpu = _have_gpu() or os.environ.get("B200_REQUIRE_GPU") == "1"   # on the device box a missing GPU must fail loudly
    for item in items:
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device visible (gpu tests run on the H100)"))
        if "ref" in item.keywords and not have_ref:
            item.add_marker(pytest.mark.skip(reason="oracle/_ref/libgstref.so not built"))


@pytest.fixture(scope="session")
def cuda_device():
    if not _have_gpu():
        pytest.fail("test marked gpu but no CUDA device is visible")
    import torch
    torch.cuda.init()
    return torch.device("cuda:0")
