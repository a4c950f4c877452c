import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine that has one)")


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU must fail loudly rather than silently skip: the product path has
    # no CPU fallback.  `-m "not gpu"` deselects these tests before they run.
    pass


@pytest.fixture(scope="session")
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but torch.cuda.is_available() is False (no CPU fallback exists)")
    return torch.device("cuda:0")


@pytest.fixture(params=["fp32", "tf32"])
def pano_precision(request):
    """Runs a GPU test in both numerical modes of the fp32 panorama-encoder GEMMs (navillm_b200.ops.set_pano_precision):
    exact CUDA-core fp32 and the product default, wgmma tf32."""
    from navillm_b200 import ops
    prev = ops.set_pano_precision(request.param)
    yield request.param
    ops.set_pano_precision(prev)
