import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), map_location="cpu", weights_only=True)


def rel_err(a, b):
    """max |a-b| / max(|a|,|b|,1): the tolerance convention of SURVEY.md section 8c."""
    a, b = a.double(), b.double()
    both_nan = torch.isnan(a) & torch.isnan(b)
    diff = torch.where(both_nan, torch.zeros_like(a), (a - b).abs())
    scale = torch.maximum(torch.maximum(a.abs(), b.abs()), torch.ones_like(a))
    scale = torch.where(both_nan, torch.ones_like(scale), scale)
    return float((diff / scale).max()) if a.numel() else 0.0


@pytest.fixture(scope="session")
def golden():
    return load_golden


@pytest.fixture(scope="session")
def cuda_device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
