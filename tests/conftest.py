import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _have_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def sawyer_model():
    from furniture_b200 import mjcf

    return mjcf.load_scene("Sawyer", "table_lack_0825")


@pytest.fixture(scope="session")
def swivel_model():
    """Sawyer + swivel_chair_0700 (SURVEY.md 8d config 3): cylinders, so cylinder-plane / cylinder-box / cylinder-cylinder pairs"""
    from furniture_b200 import mjcf

    return mjcf.load_scene("Sawyer", "swivel_chair_0700")
