import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `-m gpu`)")
    config.addinivalue_line("markers", "reference: needs the lhotse package itself (LHOTSE_REFERENCE_ROOT or the oracle/_ref archive); skips without it")


@pytest.fixture(scope="session", autouse=True)
def _build_library():
    """The CUDA library is built in-tree (nvcc cross-compiles without a GPU)."""
    from lhotse_b200 import build

    if build.needs_build():
        try:
            build.build()
        except Exception as e:  # no nvcc on this box: the prebuilt .so must have travelled
            if not os.path.exists(build.LIB_PATH):
                raise
            print("warning: could not rebuild libb200feat.so:", e)
    yield
