import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _engine_library():
    """The C-ABI library is a build artefact (git-ignored): build it in-tree if a fresh checkout lacks it and nvcc is
    here (cross-compiles without a GPU).  Nothing falls back to Python when it is missing - the tests that need it fail."""
    import shutil
    from glom_pytorch_b200 import _native
    if not os.path.exists(_native.LIB_PATH) and "GLOM_B200_LIB" not in os.environ and shutil.which("nvcc"):
        from glom_pytorch_b200.build import build_library
        build_library()
    yield
