import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
# the host-buffer pipeline sizes its chunks by the postings a batch references (engine.cu: chunk_postings); the test indexes are tiny, so
# without this every batch would take the single-call form and the chunked path would go untested
os.environ.setdefault("TRN_CHUNK_POSTINGS", "1")
os.environ.setdefault("TRN_CHUNK_RULE", "postings")  # (and keep it from being resized by the previous batch's tiny result)
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the kernels are built for sm_90a)")


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    # build (or reuse) the in-tree native library; no CPU fallback exists
    from trinity_b200.build import build_native
    build_native()
    yield


@pytest.fixture(scope="session")
def ref():
    """The reference oracle (oracle/_ref/libtrinity_ref.so == the reference's own code).  TEST-ONLY."""
    from refharness import load_ref
    return load_ref()
