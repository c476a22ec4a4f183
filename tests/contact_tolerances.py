"""Error bounds of the contact state (include/dfx.h dfx_contact_state_*) and of the rollout ending in it, with the measured errors they
derive from: the tests of tests/test_contact_state_emu.py (host emulation) and tests/test_gpu_contact_state.py (kernels)."""


# ------------------------------------------------------------------ contact state (include/dfx.h dfx_contact_state_*)
# Worst error per model of the six emulated formulations of tests/test_contact_state_emu.py (contact_util.FORMULATIONS) on
# contact_util.batch (seed 3: 75 environments, every regime row, resting contacts, height-only cotangents), ground on and off:
#   fwd   contact_f, contact_height, body_f_contact (torque, force) against the fp64 oracle, per environment and block, max |err|
#         over max(the block's max |ref|, the force floor ke |p| 2^-23 of contact_util.force_floor; heights: 1 m);
#   grad  gq, gqd of standard-normal cotangents against the exact (complex-step) gradient, per environment and gradient block
#         (contact_util.grad_errors).
# Forces are ke (up to 4e4 N/m) times depths of a few millimetres taken from metre-sized positions, so a shallow contact carries a
# relative error of |p| 2^-23 / depth: the errors here are 10-1000 times those of the link state (link_tolerances), and largest on
# the models whose batches hold the shallowest contacts (twin_HumanoidEnv: 0.1 mm; gen_planar).
# A bound is CONTACT_STATE_FACTOR times it, never below CONTACT_STATE_FLOOR (the rule of link_tolerances).  CartPole and gen_fixed
# have no contact points: their gradients are exactly zero.
CONTACT_STATE_MEASURED = {
    "CartPoleSwingUpEnv": dict(fwd=0.0, grad=0.0),
    "AntEnv": dict(fwd=1.2e-5, grad=2.8e-5),
    "HopperEnv": dict(fwd=1.6e-5, grad=1.9e-5),
    "CheetahEnv": dict(fwd=2.7e-5, grad=3.1e-5),
    "HumanoidEnv": dict(fwd=1.2e-4, grad=3.3e-4),
    "SNUHumanoidEnv": dict(fwd=1.1e-4, grad=1.4e-4),
    "twin_AntEnv": dict(fwd=6.0e-6, grad=5.9e-6),
    "twin_HumanoidEnv": dict(fwd=8.6e-4, grad=8.6e-4),
    "twin_HopperEnv": dict(fwd=5.1e-5, grad=5.0e-5),
    "twin_CheetahEnv": dict(fwd=2.6e-5, grad=3.6e-6),
    "twin_CartPoleSwingUpEnv": dict(fwd=0.0, grad=0.0),
    "twin_SNUHumanoidEnv": dict(fwd=1.8e-4, grad=1.8e-4),
    "gen_pair": dict(fwd=1.1e-5, grad=1.1e-5),
    "gen_mixed": dict(fwd=2.6e-5, grad=9.7e-6),
    "gen_planar": dict(fwd=2.3e-3, grad=2.3e-4),
    "gen_fixed": dict(fwd=0.0, grad=0.0),
    "gen_forest": dict(fwd=3.0e-5, grad=3.0e-5),
    "gen_deep24": dict(fwd=2.7e-5, grad=1.3e-4),
    "gen_wide40": dict(fwd=7.3e-5, grad=7.5e-5),
}
CONTACT_STATE_FACTOR = 4.0
CONTACT_STATE_FLOOR = 1e-6


def contact_state_tol(model_name, kind):
    """bound of the contact state's forward (kind "fwd") or adjoint ("grad") error of a model"""
    return max(CONTACT_STATE_FLOOR, CONTACT_STATE_FACTOR * CONTACT_STATE_MEASURED[model_name][kind])


# Convention check (test_contact_state_emu.convention_errors): per environment, max |qd'(ground off, f_ext = body_f_contact) -
# qd'(ground on)| of a one-substep env-step over the contact's own effect max |qd'(ground on) - qd'(ground off)|.  The two paths
# differ only in rounding: the step scatters contact wrenches through fixed-point accumulators, the external wrench enters in
# fp32 next to gravity.  Measured worst over the models with contacts and the formulations group, tile8m3 and fma: 1.7e-3
# (gen_deep24), 5.5e-4 (twin_HumanoidEnv), <= 8e-5 elsewhere.  A wrong sign gives 2, a torque about another point or a force on
# another link gives O(1).
CONVENTION_BOUND = 1e-2

# The rollout of tests/test_contact_state_emu.py and tests/test_gpu_contact_state.py (contact_util.ROLLOUT_T = 3 env-steps of
# golden case 0 at the model's own (substeps, mm_freq), then the contact state): worst rel_err of gq, gqd, gact against the exact
# gradient, over environments 0 and 1 and the emulated formulations group, fused and fma.  Bound: CONTACT_STATE_FACTOR times it,
# never below CONTACT_STATE_FLOOR.
CONTACT_ROLLOUT_MEASURED = {
    "AntEnv": dict(gq=7.4e-7, gqd=2.7e-7, gact=3.9e-6),
    "HumanoidEnv": dict(gq=8.7e-7, gqd=8.0e-7, gact=1.3e-5),
}


def contact_rollout_tol(model_name, block):
    return max(CONTACT_STATE_FLOOR, CONTACT_STATE_FACTOR * CONTACT_ROLLOUT_MEASURED[model_name][block])
