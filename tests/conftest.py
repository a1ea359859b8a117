import importlib.util
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine with one)")


def load_mloam():
    """Import m-loam_b200/ (hyphenated directory) as module `mloam_b200`."""
    if "mloam_b200" in sys.modules:
        return sys.modules["mloam_b200"]
    spec = importlib.util.spec_from_file_location("mloam_b200", os.path.join(ROOT, "m-loam_b200", "__init__.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["mloam_b200"] = mod
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="session")
def mloam():
    return load_mloam()


@pytest.fixture(scope="session")
def ctx(mloam):
    """A live context on cuda:0.  No skip: on the GPU box a missing library or device is a failure."""
    c = mloam.Context(0)
    yield c
    c.close()
