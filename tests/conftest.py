import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a: pytest -m gpu)")


ENVS = ["CartPoleSwingUpEnv", "AntEnv", "HumanoidEnv", "SNUHumanoidEnv", "HopperEnv", "CheetahEnv"]


@pytest.fixture(scope="session")
def env_names():
    return ENVS
