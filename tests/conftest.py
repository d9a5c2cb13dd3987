import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are skipped (not errored) on a machine without a CUDA device."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    return load


def rel_err(y, ref):
    """(max-norm, l2) error of y against ref, relative to ref -- SURVEY.md 8d parity metric."""
    y = np.asarray(y, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    den = max(float(np.max(np.abs(ref))), 1e-300)
    return float(np.max(np.abs(y - ref))) / den, float(np.linalg.norm(y - ref)) / max(float(np.linalg.norm(ref)), 1e-300)
