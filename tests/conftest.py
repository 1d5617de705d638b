import os
import sys

import pytest
import torch
import torch.optim  # noqa: F401  (cold import of torch._dynamo/triton can take >1 min on a fresh box: do it at collection)
import torch.amp  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 GPU")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
