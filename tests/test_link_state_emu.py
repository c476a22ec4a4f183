"""The link state (include/dfx.h dfx_link_state_forward / _backward) in the host emulation of every kernel formulation, against the
fp64 oracle (tests/link_oracle/link_oracle.c: the C oracle's eval_rigid_fk + eval_rigid_id).

  * the oracle's complex-step link-state gradient equals fp64 central differences of its own forward (six DiffRL models);
  * on the six DiffRL models and the random articulations (every joint type, the exact_util.regime_rows states, quaternions off
    the unit sphere), every emulated formulation (link_util.FORMULATIONS) agrees with the oracle per environment: the forward per
    block of elements, the adjoint per gradient block against the exact gradient, within link_tolerances.link_state_tol;
  * in the builds without FMA contraction the link state of (q, qd) is, bit for bit, the step's derived body_X_sc / body_X_sm /
    body_v_s of a one-substep call on the same inputs (the same kinematics code on the same inputs);
  * a tethered rollout -- env-steps under the wrench k (target - X_sm.p) of each step's start, then the link state -- chained by
    hand through the emulated step and link-state adjoints matches the oracle's exact gradient (LINK_TETHER_MEASURED)."""
import numpy as np
import pytest

import link_util as U
import random_articulation as R
from link_tolerances import LINK_TETHER_MEASURED, link_state_tol, link_tether_tol


@pytest.mark.parametrize("name", U.DIFFRL)
def test_oracle_link_gradient_matches_central_differences(name):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    for e in (0, 3):        # (environment 3 has quaternions off the unit sphere)
        gq, gqd = o.link_state_gradient(q[e], qd[e], g[0][e], g[1][e], g[2][e])
        x = np.concatenate([q[e], qd[e]]).astype(np.float64)

        def loss(v):
            out = o.link_state(v[None, :desc.Q], v[None, desc.Q:])
            return sum(float(np.dot(a.ravel(), b.ravel().astype(np.float64))) for a, b in zip(out, (g[0][e], g[1][e], g[2][e])))
        fd = np.zeros_like(x)
        for i in range(x.size):
            h = 1e-6 * (1.0 + abs(x[i]))
            xp, xm = x.copy(), x.copy()
            xp[i] += h
            xm[i] -= h
            fd[i] = (loss(xp) - loss(xm)) / (2 * h)
        ex = np.concatenate([gq, gqd])
        assert np.abs(fd).max() > 0
        assert U.rel_err(ex, fd) < 1e-6, (name, e, U.rel_err(ex, fd))


def test_batches_cover_every_joint_type_and_non_unit_quaternions():
    types, off_unit = set(), 0
    for name in U.MODELS:
        desc, q, qd, g = U.batch(name)
        types |= set(int(t) for t in desc.arrays["joint_type"][:desc.L])
        for sl in U._quat_slices(desc):
            off_unit += int((np.abs(np.linalg.norm(q[:, sl], axis=1) - 1.0) > 1e-3).sum())
    assert types == {R.PRISMATIC, R.REVOLUTE, R.BALL, R.FIXED, R.FREE}, types
    assert off_unit > 0


@pytest.mark.parametrize("name", U.MODELS)
def test_emulated_link_state_matches_oracle(name):
    model, ne = U.model_of(name)
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    egq, egqd = U.exact_link_gradients(name, o, q, qd, g)
    tf, tg = link_state_tol(name, "fwd"), link_state_tol(name, "grad")
    for form, flags in U.FORMULATIONS.items():
        emu = U.LinkEmuSim(model, ne, **flags)
        emu.N = q.shape[0]
        for block, err in U.forward_errors(emu.link_state(q, qd), ref).items():
            assert err.max() <= tf, (name, form, block, int(err.argmax()), float(err.max()), tf)
        gq, gqd = emu.link_state_backward(q, qd, *g)
        for block, err in U.grad_errors(desc, gq, gqd, egq, egqd).items():
            assert err.max() <= tg, (name, form, block, int(err.argmax()), float(err.max()), tg)


@pytest.mark.parametrize("name", U.MODELS)
def test_link_state_is_the_one_substep_derived_dumps_bit_for_bit(name):
    model, ne = U.model_of(name)
    desc, q, qd, g = U.batch(name)
    act = np.zeros((q.shape[0], desc.D), np.float32)
    musc = np.zeros((q.shape[0], desc.M), np.float32) if desc.M else None
    for form, flags in U.FORMULATIONS.items():
        if form == "fma":
            continue
        emu = U.LinkEmuSim(model, ne, **flags)
        emu.N = q.shape[0]
        got = emu.link_state(q, qd)
        _, _, _, dumps = emu.forward(q, qd, act, musc, 1, 1, 1.0 / 960.0, tape=False, derived=True)
        for k, key in enumerate(("body_X_sc", "body_X_sm", "body_v_s")):
            assert np.array_equal(got[k].ravel(), dumps[key].ravel()), (name, form, key)


@pytest.mark.parametrize("name", sorted(LINK_TETHER_MEASURED))
def test_emulated_tethered_rollout_matches_oracle(name):
    import wrench_util as W
    model, meta, q0, qd0, acts = U.tether_case(name, 8)
    o = U.oracle_of(name)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    for form in ("group", "fused", "fma"):
        flags = U.FORMULATIONS[form]
        link = U.LinkEmuSim(model, meta["num_envs"], **flags)
        step = W.WrenchEmuSim(model, meta["num_envs"], **flags)
        link.N = step.N = q0.shape[0]
        target = U.tether_target(link.link_state(q0, qd0)[1])
        rng = np.random.default_rng(9)
        g = tuple(rng.standard_normal((q0.shape[0], desc_L, w)).astype(np.float32)
                  for desc_L, w in ((link.desc.L, 7), (link.desc.L, 7), (link.desc.L, 6)))
        out, gq, gqd, gact = U.emu_tether_rollout(link, step, q0, qd0, acts, target, g, S, mm, dt)
        ref = o.tether_rollout(q0[0], qd0[0], acts[:, 0], None, target[0], U.TETHER_K, S, mm, dt)
        assert max(U.rel_err(a[0], b) for a, b in zip(out, ref)) < 1e-4, (name, form)
        err = U.tether_errors(o, q0, qd0, acts, target, g, gq, gqd, gact, S, mm, dt, envs=range(2))
        print(name, form, {k: "%.1e" % v for k, v in err.items()})
        for k, v in err.items():
            assert v <= link_tether_tol(name, k), (name, form, k, v, link_tether_tol(name, k))
