"""Drop-in `gym_grasper` package: same registration as the reference (gym_grasper/__init__.py:4-7), H100-backed env."""
from gym.envs.registration import register

from .version import VERSION as __version__  # noqa: F401

register(id="Grasper-v0", entry_point="gym_grasper.envs:GraspEnv")
