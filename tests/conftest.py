import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with `pytest -m gpu`)")


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    """The CPU-side artefacts (mgsim, hostsim, oracle) are cheap to (re)build; the CUDA library comes from build()."""
    mgsim = os.path.join(REPO, "tools", "mgsim")
    if not os.path.exists(mgsim):
        subprocess.check_call(["gcc", "-O2", "-o", mgsim, mgsim + ".c", "-lm"])
    yield


@pytest.fixture(scope="session")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("mgb"))
