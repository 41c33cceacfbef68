import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(autouse=True)
def _fp32_unless_stated():
    """The parity tests were written against the all-fp32 (FFMA) arithmetic and state any other mode explicitly
    (``with vqvae_b200.precision("tf32")``); the package default is "tf32" (tests/test_abi_cpu.py checks that)."""
    import vqvae_b200
    vqvae_b200.set_precision("fp32")
    yield
    vqvae_b200.set_precision("fp32")


@pytest.fixture(autouse=True)
def _inference_unless_stated():
    """The forward path is the product (SURVEY section 8): tests run under ``torch.no_grad()`` like the notebook's
    ``reconstruct``; the two tests of the differentiable VectorQuantizer re-enable grad themselves."""
    import torch
    with torch.no_grad():
        yield
