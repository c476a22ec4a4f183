"""Drop-in ``dflex`` package: ``import dflex as df`` resolves to the H100-native implementation in
``diffrl_b200.dflex_api`` (same import surface as NVlabs/DiffRL's ``dflex``), so the reference's
``envs/*.py``, ``utils/load_utils.py`` and ``algorithms/*.py`` run on it unchanged."""
import sys as _sys

from diffrl_b200 import dflex_api as _api
from diffrl_b200.dflex_api import *  # noqa: F401,F403
from diffrl_b200.dflex_api import (Mesh, Model, ModelBuilder, ScopedTimer, SemiImplicitIntegrator, State,  # noqa: F401
                                   UsdRenderer, config, model, render, sim, util)

for _name in ("config", "model", "render", "sim", "util"):
    _sys.modules[__name__ + "." + _name] = getattr(_api, _name)
