import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True)
def _iou_arithmetic_mode(request):
    """GPU tests compare the CUDA box kernels bit for bit either with the CPU oracle (mode 0: the reference's CPU build) or -- in
    tests/test_gpu_reference.py -- with the unmodified reference running on the same GPU (mode 3, the library default)."""
    if "gpu" not in request.keywords:
        yield
        return
    import torch
    if not torch.cuda.is_available():
        yield
        return
    from nerf_rpn_b200._lib import lib
    want = 3 if request.module.__name__.endswith("test_gpu_reference") else 0
    lib().nrpn_set_iou_mode(want)
    yield
    lib().nrpn_set_iou_mode(3)
