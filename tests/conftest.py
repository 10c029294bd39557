import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an NVIDIA H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """The CUDA library must exist for ABI tests (built by __graft_entry__.build() / make)."""
    from vkfft_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import subprocess
        subprocess.check_call(["make", "-C", ROOT, "-j8"], stdout=subprocess.DEVNULL)
    return _lib.load()
