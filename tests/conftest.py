import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _has_gpu() -> bool:
    try:
        from defer_b200 import _cabi
        return _cabi.device_count() > 0
    except Exception:
        return False


HAS_GPU = None


def pytest_collection_modifyitems(config, items):
    global HAS_GPU
    if not any("gpu" in it.keywords for it in items):
        return
    if HAS_GPU is None:
        HAS_GPU = _has_gpu()
    if not HAS_GPU:
        skip = pytest.mark.skip(reason="no CUDA device visible")
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)


@pytest.fixture(scope="session")
def resnet50():
    from defer_b200 import applications
    return applications.ResNet50()


@pytest.fixture(scope="session")
def x224():
    from defer_b200 import applications
    return applications.synthetic_input(1)
