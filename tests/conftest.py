import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session", autouse=True)
def _build_oracle():
    """The oracle is plain C++ and builds in seconds; (re)build it so CPU and GPU suites see the same checker."""
    subprocess.run(["make"], cwd=os.path.join(ROOT, "oracle"), check=True, stdout=subprocess.DEVNULL)
    yield
