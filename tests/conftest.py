import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="session")
def golden():
    return load_golden
