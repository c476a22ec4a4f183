"""Differentiable environments on the CUDA-native dflex of this package (same names as the reference's ``envs`` package)."""
from .base import DFlexEnv  # noqa: F401
from .locomotion import AntEnv, CartPoleSwingUpEnv, CheetahEnv, HopperEnv, HumanoidEnv, SNUHumanoidEnv  # noqa: F401
