import glob
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _ensure_built():
    """The shared libraries are build products (git-ignored).  If a checkout arrives without them, build them
    once (nvcc cross-compiles without a GPU) instead of failing every test at import."""
    have = (os.path.exists(os.path.join(ROOT, "pycolmap_b200", "libb200match.so"))
            and glob.glob(os.path.join(ROOT, "pycolmap_b200", "_core*.so"))
            and os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")))
    if not have:
        import __graft_entry__
        __graft_entry__.build()


_ensure_built()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90)")


@pytest.fixture(scope="session")
def ctx():
    import pycolmap_b200 as pb
    c = pb.Context(device=0, seed=0)   # the low-level context of the pybind11 host: one b2m_ctx behind the C ABI
    yield c
    c.close()
