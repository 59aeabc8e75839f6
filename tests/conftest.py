import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); select with -m gpu")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is present, so a bare `pytest tests/`
    also works on a machine without a GPU; select with -m gpu / -m 'not gpu'."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device on this machine")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _inference_mode_by_default():
    """The parity tests are forward-only: run them with autograd off (as inference callers do) so the fastest
    kernels are selected; the gradient tests re-enable it explicitly with torch.enable_grad()."""
    import torch
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    yield
    torch.set_grad_enabled(prev)
