"""pytest configuration: ``gpu`` marker + import paths.

``-m "not gpu"`` runs here (no GPU): oracle vs golden vectors, host logic, C-ABI load/export checks.
``-m gpu`` runs on an H100: parity of the CUDA path (through the C ABI) against the oracle / fixtures.
Every test is self-contained: what came from the reference project is stored under ``tests/golden/``.
"""
import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "st-mgcn_b200"), os.path.join(REPO, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
