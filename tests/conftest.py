"""pytest configuration: registers the ``gpu`` marker and shared fixtures.

``-m "not gpu"`` : oracle vs the reference's golden fixtures, host logic, C-ABI symbol export.
``-m gpu``       : parity of the CUDA path (through the C ABI) against the oracle.
"""
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


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def oracle():
    from oracle import ref

    ref.build()
    return ref


@pytest.fixture(scope="session")
def obed(oracle):
    return oracle.OracleBed(os.path.join(GOLDEN, "example.bed"))


@pytest.fixture(scope="session")
def obed_na(oracle):
    return oracle.OracleBed(os.path.join(GOLDEN, "example-missing.bed"))


@pytest.fixture()
def rng():
    return np.random.default_rng(20250924)
