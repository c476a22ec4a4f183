"""Error bounds of the link state (include/dfx.h dfx_link_state_*) and of the tethered rollout built on it, with the measured errors
they derive from: the tests of tests/test_link_state_emu.py (host emulation) and tests/test_gpu_link_state.py (kernels)."""


# ------------------------------------------------------------------ link state (include/dfx.h dfx_link_state_*)
# Worst error per model of the six emulated formulations of tests/test_link_state_emu.py (link_util.FORMULATIONS) on
# link_util.batch(seed 3: 75 environments, every regime row, every third environment's quaternions off the unit sphere):
#   fwd   body_X_sc / body_X_sm / body_v_s against the fp64 oracle, per environment and block (positions, quaternions, angular
#         and linear velocities), max |err| over the block's max |ref|;
#   grad  gq, gqd of standard-normal cotangents against the exact (complex-step) gradient, per environment and gradient block.
# A bound is LINK_STATE_FACTOR times it, never below LINK_STATE_FLOOR (the rule of tolerances.EXACT_GRAD_*).
LINK_STATE_MEASURED = {
    "CartPoleSwingUpEnv": dict(fwd=1.9e-7, grad=3.3e-7),
    "AntEnv": dict(fwd=3.3e-7, grad=6.7e-7),
    "HopperEnv": dict(fwd=6.6e-7, grad=8.5e-7),
    "CheetahEnv": dict(fwd=5.9e-7, grad=1.8e-6),
    "HumanoidEnv": dict(fwd=8.3e-7, grad=1.7e-6),
    "SNUHumanoidEnv": dict(fwd=9.8e-7, grad=9.3e-7),
    "twin_AntEnv": dict(fwd=6.2e-7, grad=5.6e-7),
    "twin_HumanoidEnv": dict(fwd=7.4e-7, grad=8.8e-7),
    "twin_HopperEnv": dict(fwd=3.2e-7, grad=2.8e-7),
    "twin_CheetahEnv": dict(fwd=6.0e-7, grad=6.1e-7),
    "twin_CartPoleSwingUpEnv": dict(fwd=1.9e-7, grad=1.0e-6),
    "twin_SNUHumanoidEnv": dict(fwd=6.9e-7, grad=7.6e-7),
    "gen_pair": dict(fwd=4.3e-7, grad=5.4e-7),
    "gen_mixed": dict(fwd=9.8e-7, grad=1.4e-6),
    "gen_planar": dict(fwd=7.7e-7, grad=6.3e-7),
    "gen_fixed": dict(fwd=9.0e-7, grad=9.8e-7),
    "gen_forest": dict(fwd=4.5e-7, grad=9.0e-7),
    "gen_deep24": dict(fwd=1.8e-6, grad=2.1e-6),
    "gen_wide40": dict(fwd=1.2e-6, grad=1.3e-6),
}
LINK_STATE_FACTOR = 4.0
LINK_STATE_FLOOR = 1e-6


def link_state_tol(model_name, kind):
    """bound of the link state's forward (kind "fwd") or adjoint ("grad") error of a model"""
    return max(LINK_STATE_FLOOR, LINK_STATE_FACTOR * LINK_STATE_MEASURED[model_name][kind])

# The tethered rollout of tests/test_link_state_emu.py and tests/test_gpu_link_state.py (link_util.TETHER_*: 4 env-steps of golden
# case 0 at the model's own (substeps, mm_freq), each under the wrench k (target - X_sm.p) of its start, then the link state):
# worst rel_err of gq, gqd, gact (the actions of all four env-steps) against the exact gradient, over environments 0 and 1 and
# the emulated formulations group, fused and fma.  Bound: LINK_STATE_FACTOR times it, never below LINK_STATE_FLOOR.
LINK_TETHER_MEASURED = {
    "AntEnv": dict(gq=1.6e-6, gqd=1.0e-6, gact=2.6e-6),
    "HumanoidEnv": dict(gq=1.3e-5, gqd=4.6e-6, gact=4.7e-6),
}


def link_tether_tol(model_name, block):
    return max(LINK_STATE_FLOOR, LINK_STATE_FACTOR * LINK_TETHER_MEASURED[model_name][block])
