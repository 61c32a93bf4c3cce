import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from parakeet_b200 import _lib
    _lib.lib()  # fail loudly if the CUDA library has not been built
    return torch.device("cuda:0")


def rel_err(a, b):
    import torch
    from _golden import NOT_STORED
    a = a.detach().double().cpu()
    b = b.detach().cpu()
    if b.dtype == torch.float32:    # a golden reference stored as a sample of its elements: compare the stored ones
        known = b.view(torch.int32) != NOT_STORED
        if not known.all():
            a, b = a.expand_as(b)[known], b[known]
    b = b.double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
