"""Error bounds of the Jacobian state (include/dfx.h dfx_jacobian_state_*), with the measured errors they derive from: the tests of
tests/test_jacobian_state_emu.py (host emulation) and tests/test_gpu_jacobian_state.py (kernels)."""


# Worst error per model of the six emulated formulations (link_util.FORMULATIONS) on jacobian_util.batch (seed 3: 75 environments,
# every regime row, every third environment's quaternions off the unit sphere, standard-normal cotangents):
#   fwd   J and body_a_s against the fp64 oracle, per environment and block (angular and linear rows of J, angular and linear bias
#         accelerations), max |err| over the largest |ref| of the field;
#   grad  gq, gqd against the exact (complex-step) gradient, per environment and gradient block.
# A bound is JACOBIAN_STATE_FACTOR times it, never below JACOBIAN_STATE_FLOOR (the rule of link_tolerances).
JACOBIAN_STATE_MEASURED = {
    "CartPoleSwingUpEnv": dict(fwd=4.4e-06, grad=1.8e-05),
    "AntEnv": dict(fwd=3.3e-07, grad=1.0e-06),
    "HopperEnv": dict(fwd=1.4e-06, grad=2.3e-06),
    "CheetahEnv": dict(fwd=8.6e-07, grad=4.7e-06),
    "HumanoidEnv": dict(fwd=1.3e-06, grad=2.4e-06),
    "SNUHumanoidEnv": dict(fwd=8.2e-07, grad=3.1e-06),
    "twin_AntEnv": dict(fwd=8.1e-07, grad=5.6e-06),
    "twin_HumanoidEnv": dict(fwd=1.3e-06, grad=2.1e-06),
    "twin_HopperEnv": dict(fwd=3.5e-07, grad=4.2e-07),
    "twin_CheetahEnv": dict(fwd=7.3e-07, grad=9.7e-07),
    "twin_CartPoleSwingUpEnv": dict(fwd=1.2e-05, grad=5.5e-05),
    "twin_SNUHumanoidEnv": dict(fwd=8.9e-07, grad=2.0e-06),
    "gen_pair": dict(fwd=5.0e-07, grad=2.1e-06),
    "gen_mixed": dict(fwd=2.3e-06, grad=2.1e-06),
    "gen_planar": dict(fwd=8.6e-07, grad=1.1e-06),
    "gen_fixed": dict(fwd=1.9e-06, grad=1.1e-06),
    "gen_forest": dict(fwd=7.8e-07, grad=5.8e-06),
    "gen_deep24": dict(fwd=2.7e-06, grad=2.4e-06),
    "gen_wide40": dict(fwd=1.2e-06, grad=2.6e-06),
}
JACOBIAN_STATE_FACTOR = 4.0
JACOBIAN_STATE_FLOOR = 1e-6


def jacobian_state_tol(model_name, kind):
    """bound of the Jacobian state's forward (kind "fwd") or adjoint ("grad") error of a model"""
    return max(JACOBIAN_STATE_FLOOR, JACOBIAN_STATE_FACTOR * JACOBIAN_STATE_MEASURED[model_name][kind])


# The controlled rollout of tests/test_jacobian_state_emu.py and tests/test_gpu_jacobian_state.py (jacobian_util.CONTROL_*: 4 env-steps
# of golden case 0 at the model's own (substeps, mm_freq), each under act_t = u_t + J^T (W + kappa body_a_s) of its start, loss
# g_q . q_T + g_qd . qd_T): worst rel_err of gq, gqd, gu (the u of all four env-steps) against the exact gradient, over environments 0
# and 1 and the emulated formulations group, fused and fma.  Bound: JACOBIAN_STATE_FACTOR times it, never below JACOBIAN_STATE_FLOOR.
JACOBIAN_CONTROL_MEASURED = {
    "AntEnv": dict(gq=8.9e-6, gqd=1.1e-6, gu=2.3e-6),
    "HumanoidEnv": dict(gq=2.5e-5, gqd=1.4e-5, gu=6.2e-6),
}


def jacobian_control_tol(model_name, block):
    return max(JACOBIAN_STATE_FLOOR, JACOBIAN_STATE_FACTOR * JACOBIAN_CONTROL_MEASURED[model_name][block])
