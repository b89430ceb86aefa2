import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with gcc."""
    from demi_b200 import build
    build.build_oracle()
    from oracle import binding
    binding.lib()
    return binding


@pytest.fixture(scope="session")
def native():
    """The product's C-ABI library.  Built on demand with nvcc (cross-compiles without a GPU)."""
    from demi_b200 import build, _native
    build.build_engine()
    return _native
