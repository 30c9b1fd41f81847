import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def scene_a():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    arrays, names = load_scene("A")
    return load_scene_blob("A"), arrays, names


@pytest.fixture(scope="session")
def scene_b():
    from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob

    arrays, names = load_scene("B")
    return load_scene_blob("B"), arrays, names
