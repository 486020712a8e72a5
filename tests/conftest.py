import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU must fail loudly, never silently pass: no skip here.
    pass


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def ctx():
    import covins_b200
    c = covins_b200.Context(0)
    yield c
    c.close()


def golden_cases(path):
    g = np.load(path)
    names = sorted({k.split("/")[0] for k in g.files})
    return g, names
