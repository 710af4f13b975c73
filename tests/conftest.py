import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "needs_reference: needs /root/reference (build container only)")


def pytest_collection_modifyitems(config, items):
    from oracle.ref_shim import reference_available
    have_ref = reference_available()
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    for item in items:
        if "needs_reference" in item.keywords and not have_ref:
            item.add_marker(pytest.mark.skip(reason="/root/reference not present"))
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    path = os.path.join(ROOT, "tests", "golden", "lstm_golden.npz")
    return np.load(path)
