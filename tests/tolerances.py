"""Parity tolerances, stated once.

BASELINE.json (north_star): forward state trajectories match the reference within 1e-5 relative
(here: max |a - b| / max |b| over a state vector).  That bound is met for the well-conditioned
articulations (CartPole, Ant, Hopper, Cheetah: cond(H) < 1e3).  For Humanoid and SNUHumanoid the
joint-space inertia has cond(H + armature) ~ 1e4 (tests/test_emu_golden.py::
test_reference_solve_is_conditioning_limited measures it from the golden H): the REFERENCE's own
fp32 Cholesky solve of H q'' = tau deviates from an fp64 solve by up to ~2e-5 relative, so two
correct fp32 implementations (different summation order, FMA contraction on the GPU) cannot agree
better than that over 48 substeps.  Those two models are held to 3e-5.  Gradients (no tolerance is
stated by the north star) are held to 5e-5 of the largest component.
"""
FWD_RTOL = 1e-5
GRAD_RTOL = 5e-5
_ILL_CONDITIONED = {"HumanoidEnv": 3e-5, "SNUHumanoidEnv": 3e-5,
                    "gen_fixed": 3e-5}   # (tests/random_articulation.py: a 12-link chain hanging from a fixed root; the host
# emulation's forward is 1.3e-5 (8, 4) and 1.2e-5 (7, 3) off the f64 oracle in qd, relative to the largest component, on 24
# of the 75 environments beyond 1e-5)
# ON THE REFERENCE'S GOLDEN CASES themselves (tests/golden, unperturbed states) the bar is the north-star's 1e-5 for every
# model but SNU: measured Humanoid 6.8e-6, SNU 1.3e-5 on an H100.  The host-emulation A/B (tests/test_emu_golden.py::
# test_explicit_inverse_is_not_the_parity_floor) shows where SNU's excess over 1e-5 comes from: FMA contraction (8.9e-6 without,
# 1.2e-5 with), not the explicit H^-1 (8.9e-6 vs 8.0e-6 with the reference's triangular sweeps).
_GOLDEN = {"SNUHumanoidEnv": 1.5e-5}


def golden_fwd_rtol(env_name):
    return _GOLDEN.get(env_name, FWD_RTOL)


def fwd_rtol(env_name):
    return _ILL_CONDITIONED.get(env_name, FWD_RTOL)


# bf16 tape (dfx_set_tape_dtype(1), config C2 "bf16 states"): v, a, f_tot of every tape row stored as bf16, arithmetic fp32.
# The forward pass is untouched (bit-identical); gradients against the fp32 reference goldens, relative to the largest
# component (measured on the host emulation: Humanoid 2.5e-3, SNU 2.7e-2 through the muscle wrenches; actions <= 4e-4).
BF16_TAPE_STATE_GRAD_RTOL = {"SNUHumanoidEnv": 5e-2}
BF16_TAPE_STATE_GRAD_RTOL_DEFAULT = 5e-3
BF16_TAPE_ACTION_GRAD_RTOL = 1e-3


# Step adjoint against the EXACT gradient of the oracle's fp64 forward (complex step, tests/exact_util.py), per environment and
# per gradient block (each block normalised by its own largest |exact| component).  Measured on the CPU, per model and block:
#   ref   -- the reference's own stored fp32 gradients (tests/golden/<env>.npz grad_*) on its golden cases, default pattern;
#   emu   -- the host emulation of this project's adjoint (tests/host_emu) on the batch of exact_util.make_batch(name, 75,
#            EXACT_SAMPLE[name], seed=1), worst over the multi-substep patterns of exact_util.patterns(name);
#   emu1  -- the same for the one-substep pattern (1, 1).
# Worst environment over the batch, environments on a switching surface (exact_util.on_switching_surface) left out: none
# were, on any model or pattern.  Rounded up to two digits.
EXACT_GRAD_MEASURED = {
    "CartPoleSwingUpEnv": {
        "gq_joints": (1.8e-07, 6.8e-06, 9.3e-07),
        "gqd_joints": (1.1e-07, 4.5e-07, 1.0e-07),
        "gact_joints": (1.3e-06, 7.5e-06, 4.1e-06),
    },
    "AntEnv": {
        "gq_root_pos": (4.3e-05, 2.3e-04, 1.3e-04),
        "gq_root_quat": (8.9e-06, 2.4e-05, 1.2e-05),
        "gq_joints": (4.7e-06, 1.4e-05, 5.4e-06),
        "gqd_root_ang": (3.9e-06, 8.2e-06, 6.0e-06),
        "gqd_root_lin": (2.8e-06, 9.0e-06, 5.2e-06),
        "gqd_joints": (3.7e-06, 7.4e-06, 4.1e-06),
        "gact_joints": (3.5e-06, 6.5e-06, 7.5e-06),
    },
    "HopperEnv": {
        "gq_joints": (6.4e-07, 1.5e-05, 1.5e-06),
        "gqd_joints": (5.2e-07, 1.4e-06, 1.6e-07),
        "gact_joints": (8.5e-07, 1.3e-06, 1.2e-06),
    },
    "CheetahEnv": {
        "gq_joints": (7.1e-07, 9.1e-06, 1.5e-05),
        "gqd_joints": (1.4e-06, 2.7e-06, 3.1e-06),
        "gact_joints": (3.6e-07, 1.5e-06, 3.5e-06),
    },
    "HumanoidEnv": {
        "gq_root_pos": (2.5e-04, 1.1e-03, 2.8e-04),
        "gq_root_quat": (8.7e-05, 6.7e-04, 1.7e-04),
        "gq_joints": (5.1e-05, 1.1e-04, 1.1e-04),
        "gqd_root_ang": (1.2e-05, 4.3e-05, 9.9e-06),
        "gqd_root_lin": (6.4e-05, 1.1e-04, 6.2e-05),
        "gqd_joints": (8.1e-05, 1.0e-04, 5.1e-05),
        "gact_joints": (5.9e-06, 2.5e-05, 3.3e-05),
    },
    "SNUHumanoidEnv": {
        "gq_root_pos": (9.0e-05, 6.5e-04, 2.6e-05),
        "gq_root_quat": (1.3e-04, 3.0e-04, 1.2e-04),
        "gq_joints": (1.2e-04, 8.0e-05, 6.5e-05),
        "gqd_root_ang": (3.3e-05, 4.8e-05, 4.2e-06),
        "gqd_root_lin": (1.2e-04, 9.1e-05, 1.4e-05),
        "gqd_joints": (9.8e-05, 8.3e-05, 4.1e-06),
        "gact_joints": (3.4e-06, 8.1e-06, 6.0e-06),
        "gmusc": (1.6e-05, 3.9e-05, 5.5e-05),
    },
}
# environments with exact gradients per model in those batches (of 75: the first tile, the last tile and between)
EXACT_SAMPLE = {"CartPoleSwingUpEnv": 75, "AntEnv": 75, "HopperEnv": 75, "CheetahEnv": 75, "HumanoidEnv": 24, "SNUHumanoidEnv": 16}
# The bound is a multiple of the larger measured error (two fp32 adjoints with different operation order and FMA contraction
# agree with the exact gradient to the same order, not the same digits).  With one substep only the emulation's own (1, 1)
# error counts: there conditioning amplifies least, so it is the sharpest check of each phase's adjoint.  No bound is below
# EXACT_GRAD_FLOOR (8 fp32 ulps: the spread of reordering one short fp32 sum).
EXACT_GRAD_FACTOR = 4.0
EXACT_GRAD_FLOOR = 1e-6


def exact_grad_tol(env_name, substeps):
    """{block: bound} for the step adjoint against the exact gradient"""
    out = {}
    for block, (ref, emu, emu1) in EXACT_GRAD_MEASURED[env_name].items():
        measured = emu1 if substeps == 1 else max(ref, emu)
        out[block] = max(EXACT_GRAD_FLOOR, EXACT_GRAD_FACTOR * measured)
    return out


# The same, for the random articulations of tests/random_articulation.py (model seed 0, batch seed 1: make_batch(rm, 75,
# RANDOM_SAMPLE.get(name, 75), seed=1)), measured by tests/test_random_articulations_emu.py:
#   emu   -- the worst environment of the host emulation over its six formulations (group, tile32, tile8m1, tile8m3,
#            fused, fma) and the multi-substep patterns of RandomModel.patterns() (the default and (7, 3));
#   emu1  -- the same for the one-substep pattern (1, 1).
# Environments on a switching surface left out: none were.  Rounded up to two digits.
RANDOM_GRAD_MEASURED = {
    "twin_AntEnv": {
        "gq_root_pos": (1.4e-04, 1.6e-05),
        "gq_root_quat": (1.5e-04, 2.9e-05),
        "gq_joints": (2.4e-05, 8.7e-06),
        "gqd_root_ang": (4.1e-05, 9.0e-07),
        "gqd_root_lin": (6.8e-06, 3.3e-06),
        "gqd_joints": (1.2e-05, 6.9e-07),
        "gact_joints": (3.1e-05, 3.4e-05),
    },
    "twin_HumanoidEnv": {
        "gq_root_pos": (6.5e-04, 9.8e-05),
        "gq_root_quat": (1.4e-04, 1.1e-04),
        "gq_joints": (1.7e-05, 5.1e-06),
        "gqd_root_ang": (3.2e-05, 7.3e-07),
        "gqd_root_lin": (3.8e-05, 7.5e-07),
        "gqd_joints": (1.6e-05, 2.4e-06),
        "gact_joints": (1.6e-05, 3.2e-05),
    },
    "twin_HopperEnv": {
        "gq_joints": (7.8e-06, 1.2e-05),
        "gqd_joints": (3.3e-06, 3.5e-07),
        "gact_joints": (7.3e-06, 9.8e-06),
    },
    "twin_CheetahEnv": {
        "gq_joints": (3.5e-05, 4.3e-06),
        "gqd_joints": (2.2e-06, 1.6e-06),
        "gact_joints": (7.5e-06, 8.1e-06),
    },
    "twin_CartPoleSwingUpEnv": {
        "gq_joints": (2.3e-05, 2.2e-05),
        "gqd_joints": (4.8e-06, 1.1e-06),
        "gact_joints": (2.5e-05, 2.7e-05),
    },
    "twin_SNUHumanoidEnv": {
        "gq_root_pos": (1.6e-03, 1.9e-04),
        "gq_root_quat": (9.6e-05, 8.8e-05),
        "gq_joints": (2.0e-05, 2.2e-05),
        "gqd_root_ang": (1.7e-05, 4.0e-06),
        "gqd_root_lin": (7.7e-05, 4.6e-06),
        "gqd_joints": (1.8e-05, 3.0e-06),
        "gact_joints": (2.1e-05, 3.9e-05),
        "gmusc": (2.3e-05, 2.3e-05),
    },
    "gen_pair": {
        "gq_root_pos": (2.3e-05, 5.7e-06),
        "gq_root_quat": (1.2e-05, 7.9e-06),
        "gq_joints": (1.4e-05, 3.2e-06),
        "gqd_root_ang": (8.1e-07, 1.5e-07),
        "gqd_root_lin": (3.0e-06, 2.7e-07),
        "gqd_joints": (6.4e-07, 1.2e-07),
        "gact_joints": (0.0, 0.0),           # (a ball joint: no actuated dofs)
    },
    "gen_mixed": {
        "gq_root_pos": (1.7e-04, 9.3e-05),
        "gq_root_quat": (2.6e-04, 6.5e-05),
        "gq_joints": (3.7e-05, 2.7e-05),
        "gqd_root_ang": (2.7e-06, 3.6e-07),
        "gqd_root_lin": (3.7e-06, 6.1e-07),
        "gqd_joints": (1.7e-06, 3.3e-07),
        "gact_joints": (1.7e-05, 1.8e-05),
    },
    "gen_planar": {
        "gq_joints": (4.2e-05, 1.2e-05),
        "gqd_joints": (9.5e-07, 1.4e-07),
        "gact_joints": (8.0e-06, 6.8e-06),
    },
    "gen_fixed": {
        "gq_joints": (5.8e-04, 4.1e-04),
        "gqd_joints": (2.4e-05, 3.6e-06),
        "gact_joints": (1.6e-04, 2.0e-04),
    },
    "gen_forest": {
        "gq_root_pos": (5.9e-04, 1.1e-04),
        "gq_root_quat": (1.2e-04, 8.0e-05),
        "gq_joints": (1.1e-04, 3.2e-05),
        "gqd_root_ang": (2.5e-06, 2.8e-07),
        "gqd_root_lin": (5.8e-06, 1.4e-06),
        "gqd_joints": (8.1e-06, 2.0e-06),
        "gact_joints": (4.5e-05, 4.8e-05),
    },
    "gen_deep24": {
        "gq_root_pos": (6.6e-03, 1.6e-03),
        "gq_root_quat": (1.0e-03, 1.6e-03),
        "gq_joints": (3.1e-04, 3.5e-04),
        "gqd_root_ang": (9.3e-05, 3.8e-05),
        "gqd_root_lin": (2.6e-04, 8.3e-05),
        "gqd_joints": (1.2e-05, 4.2e-06),
        "gact_joints": (9.3e-05, 8.9e-05),
    },
    "gen_wide40": {
        "gq_root_pos": (4.7e-03, 1.8e-03),
        "gq_root_quat": (3.5e-04, 1.7e-04),
        "gq_joints": (3.6e-05, 1.8e-05),
        "gqd_root_ang": (8.9e-06, 2.4e-06),
        "gqd_root_lin": (2.7e-05, 2.0e-05),
        "gqd_joints": (3.9e-06, 9.7e-07),
        "gact_joints": (1.2e-05, 1.2e-05),
    },
}
# environments with exact gradients in those batches (of 75), for the models where 75 complex-step gradients per pattern
# would dominate the run time
RANDOM_SAMPLE = {"twin_HumanoidEnv": 24, "twin_SNUHumanoidEnv": 16, "gen_deep24": 24, "gen_wide40": 16}


def random_grad_tol(model_name, substeps):
    """{block: bound} for the step adjoint of a random articulation against the exact gradient"""
    return {block: max(EXACT_GRAD_FLOOR, EXACT_GRAD_FACTOR * (emu1 if substeps == 1 else emu))
            for block, (emu, emu1) in RANDOM_GRAD_MEASURED[model_name].items()}
