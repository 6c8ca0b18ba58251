"""pytest configuration: markers, package import (hyphenated directory), library fixtures."""
import importlib
import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

pkg = importlib.import_module("ctrl-vio_b200")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def ctvio():
    return pkg


@pytest.fixture(scope="session")
def oracle_lib():
    """CPU oracle (test infrastructure): built on demand with plain g++."""
    so = os.path.join(REPO, "oracle", "liboracle.so")
    srcs = [os.path.join(REPO, "oracle", f) for f in os.listdir(os.path.join(REPO, "oracle"))
            if f.endswith((".cpp", ".hpp"))] + [os.path.join(REPO, "include", "ctvio.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["make", "-C", os.path.join(REPO, "oracle")], check=True, capture_output=True)
    return pkg.CtvioLib(so, "ctvo_", optional=pkg.binding.DEVICE_ONLY_SYMBOLS)


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library; GPU tests fail loudly if it is missing (no fallback)."""
    return pkg.load()
