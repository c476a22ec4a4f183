"""The contact state (include/dfx.h dfx_contact_state_forward / _backward) in the host emulation of every kernel formulation, against
the fp64 oracle (tests/contact_oracle/contact_oracle.c: eval_rigid_contacts restated per point).

  * the oracle's complex-step contact-state gradient equals fp64 central differences of its own forward, away from the contact
    switching surfaces;
  * the batches cover penetrating and clear points, resting contacts (|v_t| = 0), height-only cotangents, and at least one model
    whose contacts the pack regroups (not sorted by body), so the Model-order permutation is exercised;
  * on the six DiffRL models and the random articulations (exact_util.regime_rows included), every emulated formulation
    (contact_util.FORMULATIONS) agrees with the oracle per environment -- the forward per block of elements, the adjoint per
    gradient block against the exact gradient -- within contact_tolerances.contact_state_tol, with the ground on and off;
  * convention: with the ground off, a one-substep env-step under f_ext = body_f_contact equals the same env-step with the ground
    on, up to the fixed-point rounding of the step's contact scatter (CONVENTION_BOUND): the sign, the torque's reference point and
    the link sums in one check;
  * a T = 3 rollout of env-steps ending in the contact state, chained by hand through the emulated step and contact-state
    adjoints, matches the oracle's exact gradient (CONTACT_ROLLOUT_MEASURED)."""
import numpy as np
import pytest

import contact_util as U
from contact_tolerances import CONTACT_ROLLOUT_MEASURED, CONVENTION_BOUND, contact_rollout_tol, contact_state_tol

CONTACT_MODELS = [m for m in U.MODELS if U.oracle_of(m).desc.C > 0]


def _penetrating_envs(name, o, q, qd, count):
    """the first `count` environments with a penetrating point, moving (not at rest) and not on a switching surface"""
    h = U.reference(name, o, q, qd)[1]
    out = []
    for e in range(q.shape[0]):
        if (h[e] < -1e-4).any() and qd[e].any() and not U.one_ulp_sensitive(o, q, qd, e):
            out.append(e)
        if len(out) == count:
            break
    return out


@pytest.mark.parametrize("name", ["AntEnv", "HopperEnv", "HumanoidEnv", "twin_AntEnv", "gen_mixed"])
def test_oracle_contact_gradient_matches_central_differences(name):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    envs = _penetrating_envs(name, o, q, qd, 2)
    assert envs, name
    for e in envs:
        gq, gqd = o.contact_state_gradient(q[e], qd[e], g[0][e], g[1][e], g[2][e])
        x = np.concatenate([q[e], qd[e]]).astype(np.float64)

        def loss(v):
            out = o.contact_state(v[None, :desc.Q], v[None, desc.Q:])
            return sum(float(np.dot(a.ravel(), b.ravel().astype(np.float64))) for a, b in zip(out, (g[0][e], g[1][e], g[2][e])))
        fd = np.zeros_like(x)
        for i in range(x.size):
            h = 1e-7 * (1.0 + abs(x[i]))
            xp, xm = x.copy(), x.copy()
            xp[i] += h
            xm[i] -= h
            fd[i] = (loss(xp) - loss(xm)) / (2 * h)
        ex = np.concatenate([gq, gqd])
        assert np.abs(fd).max() > 0
        assert U.rel_err(ex, fd) < 1e-5, (name, e, U.rel_err(ex, fd))


def test_batches_cover_the_contact_regimes_and_an_unsorted_model():
    pen = clear = resting = height_only = 0
    unsorted = []
    for name in CONTACT_MODELS:
        o = U.oracle_of(name)
        desc, q, qd, g = U.batch(name)
        h = U.reference(name, o, q, qd)[1]
        pen += int((h < 0).sum())
        clear += int((h >= 0).sum())
        resting += int(((h < 0).any(axis=1) & ~qd.any(axis=1)).sum())
        height_only += int((~g[0].any(axis=(1, 2)) & ~g[2].any(axis=(1, 2)) & g[1].any(axis=1)).sum())
        if not U.contacts_sorted(desc):
            unsorted.append(name)
    assert pen > 0 and clear > 0 and resting > 0 and height_only > 0, (pen, clear, resting, height_only)
    assert unsorted, "no model in the run has contacts the pack regroups"
    print("models whose contacts are not sorted by body:", unsorted)


@pytest.mark.parametrize("ground", [True, False], ids=["ground", "no_ground"])
@pytest.mark.parametrize("name", U.MODELS)
def test_emulated_contact_state_matches_oracle(name, ground):
    model, ne = U.model_of(name)
    o = U.oracle_of(name)
    o.set_ground(ground)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    if not ground:
        assert not ref[0].any() and not ref[2].any()
    egq, egqd = U.exact_contact_gradients(name, o, q, qd, g)
    tf, tg = contact_state_tol(name, "fwd"), contact_state_tol(name, "grad")
    for form, flags in U.FORMULATIONS.items():
        emu = U.ContactEmuSim(model, ne, **flags)
        emu.N = q.shape[0]
        emu.set_ground(ground)
        out = emu.contact_state(q, qd)
        if not ground:
            assert not out[0].any(), (name, form)
        for block, err in U.forward_errors(desc, out, ref).items():
            assert err.max() <= tf, (name, form, block, int(err.argmax()), float(err.max()), tf)
        gq, gqd = emu.contact_state_backward(q, qd, *g)
        for block, err in U.grad_errors(desc, gq, gqd, egq, egqd).items():
            assert err.max() <= tg, (name, form, block, int(err.argmax()), float(err.max()), tg)


def convention_errors(emu, q, qd, musc=None, dt=1.0 / 960.0):
    """[n]: contact_util.convention_errors of the host emulation's one-substep env-steps"""
    n, D = q.shape[0], emu.desc.D
    act = np.zeros((n, D), np.float32)
    emu.set_ground(True)
    w = emu.contact_state(q, qd)[2]
    _, qd_on, _, _ = emu.forward(q, qd, act, musc, 1, 1, dt)
    emu.set_ground(False)
    _, qd_ext, _, _ = emu.forward(q, qd, act, musc, 1, 1, dt, f_ext=w)
    _, qd_off, _, _ = emu.forward(q, qd, act, musc, 1, 1, dt)
    emu.set_ground(True)
    return U.convention_errors(qd_on, qd_ext, qd_off)


@pytest.mark.parametrize("name", CONTACT_MODELS)
def test_ground_off_with_body_f_contact_as_f_ext_is_the_ground(name):
    model, ne = U.model_of(name)
    desc, q, qd, _ = U.batch(name)
    musc = np.zeros((q.shape[0], desc.M), np.float32) if desc.M else None
    for form in ("group", "tile8m3", "fma"):
        emu = U.ContactEmuSim(model, ne, **U.FORMULATIONS[form])
        emu.N = q.shape[0]
        err = convention_errors(emu, q, qd, musc)
        assert (err > 0).any(), (name, form, "no environment with a contact")
        assert err.max() <= CONVENTION_BOUND, (name, form, int(err.argmax()), float(err.max()))


def emu_contact_rollout(emu, q, qd, acts, g, S, mm, dt):
    """the rollout and its adjoint in the host emulation, chained by hand: (final contact state, gq, gqd, gact [T, n, D])"""
    tapes = []
    for t in range(acts.shape[0]):
        q2, qd2, tape, _ = emu.forward(q, qd, acts[t], None, S, mm, dt)
        tapes.append(tape)
        q, qd = q2, qd2
    out = emu.contact_state(q, qd)
    gq, gqd = emu.contact_state_backward(q, qd, *g)
    gact = np.zeros_like(acts)
    for t in reversed(range(acts.shape[0])):
        gq, gqd, ga, _ = emu.backward(acts[t], None, tapes[t], gq, gqd, S, mm, dt)
        gact[t] = ga.reshape(acts[t].shape)
    return out, gq.reshape(q.shape), gqd.reshape(qd.shape), gact


def rollout_cotangents(desc, n, seed=9):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, desc.C, 3)).astype(np.float32), rng.standard_normal((n, desc.C)).astype(np.float32),
            rng.standard_normal((n, desc.L, 6)).astype(np.float32))


@pytest.mark.parametrize("name", sorted(CONTACT_ROLLOUT_MEASURED))
def test_emulated_contact_rollout_matches_oracle(name):
    model, meta, q0, qd0, acts = U.rollout_case(name, 8)
    o = U.oracle_of(name)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    for form in ("group", "fused", "fma"):
        emu = U.ContactEmuSim(model, meta["num_envs"], **U.FORMULATIONS[form])
        emu.N = q0.shape[0]
        g = rollout_cotangents(emu.desc, q0.shape[0])
        out, gq, gqd, gact = emu_contact_rollout(emu, q0, qd0, acts, g, S, mm, dt)
        ref = o.rollout(q0[0], qd0[0], acts[:, 0], None, S, mm, dt)
        assert U.rel_err(out[1][0], ref[1]) < 1e-4, (name, form)
        err = U.rollout_errors(o, q0, qd0, acts, g, gq, gqd, gact, S, mm, dt, envs=range(2))
        print(name, form, {k: "%.1e" % v for k, v in err.items()})
        for k, v in err.items():
            assert v <= contact_rollout_tol(name, k), (name, form, k, v, contact_rollout_tol(name, k))
