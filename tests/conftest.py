"""pytest configuration: `gpu` marker, golden fixtures, library handles."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


@pytest.fixture(scope="session")
def golden():
    """Known-answer set produced by the reference's own kernels (tests/golden/make_golden.py)."""
    from tests.util import load_golden
    return load_golden()


@pytest.fixture(scope="session")
def product():
    from surfelmeshing_b200 import _lib
    return _lib.load_product()


@pytest.fixture(scope="session")
def reference():
    """The reference's kernels rebuilt for sm_90a (oracle/_ref); skips when not built."""
    from surfelmeshing_b200 import _lib
    if not _lib.REF_LIB_PATH.exists():
        pytest.skip("oracle/_ref/libsurfel_ref.so not built (needs the reference sources at build time)")
    return _lib.load_reference_oracle()


@pytest.fixture(scope="session")
def shimref():
    """Reference host glue linked against the vis:: link shims (oracle/_ref/libsurfel_shimref.so)."""
    from surfelmeshing_b200 import _lib
    if not _lib.SHIM_LIB_PATH.exists():
        pytest.skip("oracle/_ref/libsurfel_shimref.so not built (needs the reference sources at build time)")
    return _lib.load_shim_oracle()
