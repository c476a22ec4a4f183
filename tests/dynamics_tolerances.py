"""Bounds of the dynamics state (include/dfx.h dfx_dynamics_state_*), with the measured errors they come from.

The rule of tests/link_tolerances.py: a bound is DYN_FACTOR times the worst error measured, never below DYN_FLOOR, per model and
field.  MEASURED[model]: the worst per environment of
  * the host emulation, every formulation (dynamics_util.FORMULATIONS, FMA contraction included), ground on / off and wrench on /
    off (tests/test_dynamics_state_emu.py, the N = 75 environments of dynamics_util.batch), and
  * the kernels on one H100 80GB HBM3 (700 W), every kernel family, N = 1 and 75 (tests/test_gpu_dynamics_state.py),
against the fp64 oracle:
  forward : joint_qdd, joint_tau, H -- max |err| over the field's max |ref| of the environment;
  adjoint : gq, gqd, gact, gmusc, g_f_ext against the complex-step gradient (the first 4 environments) -- max |err| over the
            environment's largest exact gradient component.
Environments whose one-substep env-step is itself non-finite (two of gen_deep24's) are skipped by count.  A field a model has no
entry for (gmusc without muscles) is held to the floor.
joint_qdd carries the conditioning of H + diag(armature): the chains gen_deep24 (2e-2) and gen_fixed (5e-4) and the humanoids (1e-4)
are far above the well-conditioned models; on the two humanoids and their twins its bound is also never below the conditioning-aware
criterion of tests/tolerances.py (fwd_rtol: 3e-5 for those models, 1e-5 for every other)."""
import tolerances as T

DYN_FACTOR = 4.0
DYN_FLOOR = 1e-6

MEASURED = {
    "CartPoleSwingUpEnv": dict(joint_qdd=1.8e-05, joint_tau=4.1e-06, H=2.4e-07, gq=1.6e-05, gqd=1.3e-06, gact=1.3e-06, g_f_ext=1.3e-06),
    "AntEnv": dict(joint_qdd=5.3e-05, joint_tau=2.3e-05, H=5.1e-07, gq=1.9e-06, gqd=6.4e-08, gact=5.9e-09, g_f_ext=2.1e-09),
    "HopperEnv": dict(joint_qdd=1.6e-05, joint_tau=3.5e-05, H=1.2e-06, gq=1.2e-06, gqd=5.6e-08, gact=5.8e-09, g_f_ext=6.0e-09),
    "CheetahEnv": dict(joint_qdd=2.8e-06, joint_tau=1.4e-05, H=6.2e-07, gq=1.1e-06, gqd=1.6e-08, gact=1.1e-09, g_f_ext=1.7e-09),
    "HumanoidEnv": dict(joint_qdd=1.1e-04, joint_tau=2.1e-04, H=6.6e-07, gq=5.6e-05, gqd=1.3e-05, gact=8.8e-07, g_f_ext=1.6e-07),
    "SNUHumanoidEnv": dict(joint_qdd=1.4e-04, joint_tau=1.2e-04, H=2.5e-06, gq=9.0e-05, gqd=2.3e-07, gact=3.3e-08, gmusc=8.2e-09, g_f_ext=7.4e-08),
    "twin_CartPoleSwingUpEnv": dict(joint_qdd=2.3e-05, joint_tau=2.6e-06, H=3.8e-07, gq=1.0e-05, gqd=8.0e-06, gact=1.3e-06, g_f_ext=8.2e-07),
    "twin_AntEnv": dict(joint_qdd=1.3e-05, joint_tau=8.7e-07, H=1.6e-06, gq=1.5e-05, gqd=1.4e-07, gact=3.0e-08, g_f_ext=2.1e-08),
    "twin_HopperEnv": dict(joint_qdd=1.5e-05, joint_tau=1.7e-05, H=4.5e-07, gq=2.3e-06, gqd=1.7e-07, gact=5.9e-08, g_f_ext=3.9e-08),
    "twin_CheetahEnv": dict(joint_qdd=9.3e-06, joint_tau=8.3e-06, H=6.0e-07, gq=2.9e-06, gqd=2.6e-07, gact=1.4e-07, g_f_ext=1.1e-07),
    "twin_HumanoidEnv": dict(joint_qdd=3.9e-05, joint_tau=8.2e-06, H=2.5e-06, gq=1.4e-05, gqd=4.0e-07, gact=6.6e-08, g_f_ext=5.8e-08),
    "twin_SNUHumanoidEnv": dict(joint_qdd=1.4e-04, joint_tau=5.1e-06, H=1.8e-06, gq=2.7e-05, gqd=4.1e-07, gact=1.2e-07, gmusc=1.2e-08, g_f_ext=9.0e-08),
    "gen_pair": dict(joint_qdd=2.7e-05, joint_tau=3.1e-06, H=1.1e-06, gq=7.6e-06, gqd=4.7e-07, gact=0.0e+00, g_f_ext=3.9e-08),
    "gen_mixed": dict(joint_qdd=1.5e-04, joint_tau=4.8e-06, H=4.6e-06, gq=9.9e-06, gqd=1.0e-07, gact=1.9e-08, g_f_ext=9.9e-09),
    "gen_planar": dict(joint_qdd=4.5e-05, joint_tau=2.3e-05, H=7.8e-07, gq=5.9e-06, gqd=1.1e-07, gact=3.3e-08, g_f_ext=4.7e-08),
    "gen_fixed": dict(joint_qdd=4.6e-04, joint_tau=3.9e-06, H=4.2e-06, gq=3.3e-04, gqd=3.0e-06, gact=2.5e-07, g_f_ext=2.7e-07),
    "gen_forest": dict(joint_qdd=3.4e-05, joint_tau=5.9e-06, H=2.0e-06, gq=1.3e-04, gqd=7.2e-07, gact=1.0e-07, g_f_ext=1.2e-07),
    "gen_deep24": dict(joint_qdd=2.1e-02, joint_tau=7.8e-06, H=6.8e-06, gq=1.4e-04, gqd=8.8e-07, gact=3.5e-08, g_f_ext=4.1e-08),
    "gen_wide40": dict(joint_qdd=1.6e-04, joint_tau=5.5e-06, H=4.5e-06, gq=2.2e-05, gqd=6.9e-08, gact=1.2e-08, g_f_ext=2.6e-08),
}

ILL_CONDITIONED = ("HumanoidEnv", "SNUHumanoidEnv", "twin_HumanoidEnv", "twin_SNUHumanoidEnv")


def dynamics_tol(name, field):
    b = max(DYN_FACTOR * MEASURED[name].get(field, 0.0), DYN_FLOOR)
    if field == "joint_qdd" and name in ILL_CONDITIONED:
        base = name[len("twin_"):] if name.startswith("twin_") else name
        b = max(b, T.fwd_rtol(base))
    return b


# reference goldens (case*/first): the reference's own fp32 state of its first substep, against the emulation / kernels at the
# golden inputs: per field max |err| over max |ref| of the case; the bound is tolerances.golden_fwd_rtol per model for tau and H,
# and fwd_rtol's conditioning-aware bound for joint_qdd
def golden_tol(name, field):
    if field == "joint_qdd":
        return max(T.fwd_rtol(name), 4 * T.golden_fwd_rtol(name))
    return 4 * T.golden_fwd_rtol(name)


# the convention check: |qd_out - (qd + dt_sub qdd)| of a one-substep env-step over the fp32 rounding of that update
CONVENTION_BOUND = 1.0
# the step adjoint on a loss on qd_out against the dynamics adjoint seeded with g_qdd = dt g (+ g on gqd): max |err| over the
# environment's largest component (they differ in summation order only)
CONVENTION_GRAD_BOUND = 1e-5

# the T-step rollout ending in the dynamics state (loss 1/2 qd^T H qd + |tau|^2 + w . qdd), against the oracle's exact gradient
ROLLOUT_MEASURED = 1.2e-5     # (HumanoidEnv gq, first two environments, one H100 80GB HBM3; Ant 2e-6)


def rollout_tol():
    return max(DYN_FACTOR * ROLLOUT_MEASURED, 1e-5)
