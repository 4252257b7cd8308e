import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU")


def _has_gpu() -> bool:
    if os.environ.get("CL_FORCE_NO_GPU"):
        return False
    try:
        from crowdllama_b200 import engine as eng
        return eng.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def has_gpu():
    return _has_gpu()


def pytest_collection_modifyitems(config, items):
    # GPU tests must FAIL loudly on a GPU box when the extension is missing; they are only
    # skipped when no device exists at all (the CPU container).
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
