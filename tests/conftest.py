import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


def relative_force_error(f, fref):
    """max_i |dF_i|_inf / max(1, |F_i,ref|): the reference's ASSERT_EQUAL_VEC form (AssertionUtilities.h:55-57)."""
    import numpy as np
    d = np.abs(f - fref).max(axis=1)
    n = np.maximum(1.0, np.linalg.norm(fref, axis=1))
    return float((d/n).max())


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
