import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (`pytest -m gpu`)")


def pytest_sessionstart(session):
    """A fresh checkout has no built library (the .so is git-ignored): cross-compile it once when nvcc is present, so the
    ABI tests of the CPU suite do not depend on a prior `__graft_entry__.build()`."""
    import shutil

    from gtsfm_b200 import _lib

    if not _lib.LIB_PATH.exists() and shutil.which("nvcc"):
        from gtsfm_b200 import build

        build.build()


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def b200_ctx():
    """One shared C-ABI context for the GPU tests; fails loudly (no skip) when the library or GPU is missing."""
    from gtsfm_b200 import _lib

    ctx = _lib.Context(0)
    yield ctx
    ctx.close()
