"""pytest configuration: markers + import path for the in-tree package and the oracle."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on the GPU box")


def load_golden(name: str):
    return np.load(os.path.join(GOLDEN_DIR, f"{name}.npz"), allow_pickle=False)


@pytest.fixture(scope="session")
def golden():
    return load_golden
