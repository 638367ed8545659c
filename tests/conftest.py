import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no GPU in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _keep_gradients_for_inspection(request):
    """The optimiser kernels clear the gradient buckets as they read them (production path).  Parity tests look at
    the gradients AFTER a step, so they run with engine.KEEP_GRADS = True (the step leaves the bucket alone and the
    next backward zeroes it); tests that exercise the clear-on-read path set it back themselves."""
    if "gpu" not in request.keywords:
        yield
        return
    from segan_pytorch_b200 import engine as E
    prev = E.KEEP_GRADS
    E.KEEP_GRADS = True
    yield
    E.KEEP_GRADS = prev
