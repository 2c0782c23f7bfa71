import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU; run with -m gpu")


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from imagdressing_b200 import _lib

    _lib.require_b200()  # loud failure if the extension is missing or the GPU is not sm_90
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _release_gpu_memory():
    """Frozen-weight operand caches hold their source storages (whole UNets) until cleared; free them after every test
    so that one process can run the whole GPU suite on an 80 GB card."""
    yield
    torch = sys.modules.get("torch")
    if torch is None or not torch.cuda.is_initialized():
        return
    import gc

    from imagdressing_b200 import autograd

    autograd.clear_cache()
    gc.collect()
    torch.cuda.empty_cache()


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))
