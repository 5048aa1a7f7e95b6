import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")
    # the shared library is a build artefact (git-ignored): compile it in-tree on a fresh checkout (nvcc cross-compiles
    # sm_90a without a GPU)
    lib = os.path.join(ROOT, "tacotron-2_b200", "libt2b200.so")
    if not os.path.exists(lib):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def t2lib():
    from t2_import import t2
    return t2.lib.load()
