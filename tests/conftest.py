import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); `pytest -m gpu` runs them")


@pytest.fixture(scope="session")
def pkg():
    return importlib.import_module("3dobjecttracking_b200")


@pytest.fixture(scope="session")
def synth(pkg):
    return pkg.synth


@pytest.fixture(scope="session")
def oracle():
    import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="session")
def capi(pkg):
    """The CUDA path. Tests that use it are marked gpu; there is no CPU stand-in."""
    return importlib.import_module("3dobjecttracking_b200.capi")
