import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")


def rel_errs(out, ref):
    """(max|d|/max|ref|, ||d||2/||ref||2) — the two relative errors SURVEY.md §8c names."""
    import torch
    out = out.detach().double().cpu()
    ref = ref.detach().double().cpu()
    d = (out - ref)
    den_max = max(float(ref.abs().max()), 1e-30)
    den_l2 = max(float(ref.norm()), 1e-30)
    return float(d.abs().max()) / den_max, float(d.norm()) / den_l2


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
