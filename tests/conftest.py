import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU")


@pytest.fixture(scope="session")
def tiny_scene():
    from intrinsic3d_b200.scene import config_scene
    return config_scene("tiny")


@pytest.fixture(scope="session")
def small_scene():
    from intrinsic3d_b200.scene import config_scene
    return config_scene("small")
