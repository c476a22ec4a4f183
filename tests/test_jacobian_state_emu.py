"""The Jacobian state (include/dfx.h dfx_jacobian_state_forward / _backward) in the host emulation of every kernel formulation,
against the fp64 oracle (tests/jacobian_oracle/jacobian_oracle.c: eval_rigid_fk + eval_rigid_id, then the spatial_jacobian loop).

  * the oracle's complex-step gradient equals fp64 central differences of its own forward (six DiffRL models);
  * on the six DiffRL models and the random articulations (every joint type, the regime rows, quaternions off the unit sphere),
    every emulated formulation (link_util.FORMULATIONS) agrees with the oracle per environment: the forward per block, the adjoint
    per gradient block against the exact gradient, within jacobian_tolerances.jacobian_state_tol; J is exactly 0 where no dof
    moves the link, and a free root's columns are exactly the identity;
  * in the builds without FMA contraction, J is bit for bit the spatial.h rule applied to the step's derived joint_S_s of a
    one-substep call on the same inputs, and body_a_s its derived body_a_s;
  * the reference goldens: J assembled (numpy, here) from case*/first/joint_S_s and case*/first/body_a_s, at case*/{q0, qd0};
  * the point bias acceleration stated in include/dfx.h, b = a_v + a_w x p + w x (v_o + w x p), against fp64 second differences of
    a body-fixed point along q(t) = q0 + t qd (q'' = 0) on the articulations whose joints all have dq/dt = qd;
  * a controlled rollout -- env-steps under act_t = u_t + J^T (W + kappa body_a_s) of each step's start -- chained by hand through
    the emulated step and Jacobian-state adjoints matches the oracle's exact gradient (JACOBIAN_CONTROL_MEASURED)."""
import numpy as np
import pytest

import jacobian_util as U
import random_articulation as R
from emu_util import load_golden
from jacobian_tolerances import JACOBIAN_CONTROL_MEASURED, jacobian_control_tol, jacobian_state_tol


@pytest.mark.parametrize("name", U.DIFFRL)
def test_oracle_jacobian_gradient_matches_central_differences(name):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    for e in (0, 3):        # (environment 3 has quaternions off the unit sphere)
        gq, gqd = o.jacobian_state_gradient(q[e], qd[e], g[0][e], g[1][e])
        x = np.concatenate([q[e], qd[e]]).astype(np.float64)

        def loss(v):
            J, a = o.jacobian_state(v[None, :desc.Q], v[None, desc.Q:])
            return float(np.dot(J.ravel(), g[0][e].ravel().astype(np.float64)) + np.dot(a.ravel(), g[1][e].ravel().astype(np.float64)))
        fd = np.zeros_like(x)
        for i in range(x.size):
            h = 1e-6 * (1.0 + abs(x[i]))
            xp, xm = x.copy(), x.copy()
            xp[i] += h
            xm[i] -= h
            fd[i] = (loss(xp) - loss(xm)) / (2 * h)
        ex = np.concatenate([gq, gqd])
        assert np.abs(fd).max() > 0
        assert U.U.rel_err(ex, fd) < 1e-6, (name, e, U.U.rel_err(ex, fd))


def _free_root_columns(desc):
    """[(link, dof start)] of the free joints"""
    a = desc.arrays
    q0 = int(a["joint_qd_start"][0])
    return [(i, int(a["joint_qd_start"][i]) - q0) for i in range(desc.L) if int(a["joint_type"][i]) == R.FREE]


@pytest.mark.parametrize("name", U.MODELS)
def test_emulated_jacobian_state_matches_oracle(name):
    model, ne = U.U.model_of(name)
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    egq, egqd = U.exact_gradients(name, o, q, qd, g)
    tf, tg = jacobian_state_tol(name, "fwd"), jacobian_state_tol(name, "grad")
    mask = U.ancestor_mask(desc)
    for form, flags in U.FORMULATIONS.items():
        emu = U.JacobianEmuSim(model, ne, **flags)
        emu.N = q.shape[0]
        out = emu.jacobian_state(q, qd)
        assert not out[0].transpose(0, 2, 1, 3)[:, :, ~mask].any(), (name, form)
        for i0, d0 in _free_root_columns(desc):
            sub = np.nonzero(mask[:, d0])[0]
            assert np.array_equal(out[0][:, sub][:, :, :, d0:d0 + 6], np.broadcast_to(np.eye(6, dtype=np.float32), (q.shape[0], len(sub), 6, 6)))
        for block, err in U.forward_errors(out, ref).items():
            assert err.max() <= tf, (name, form, block, int(err.argmax()), float(err.max()), tf)
        gq, gqd = emu.jacobian_state_backward(q, qd, *g)
        for block, err in U.grad_errors(desc, gq, gqd, egq, egqd).items():
            assert err.max() <= tg, (name, form, block, int(err.argmax()), float(err.max()), tg)


@pytest.mark.parametrize("name", U.MODELS)
def test_jacobian_state_is_the_one_substep_derived_dumps_bit_for_bit(name):
    model, ne = U.U.model_of(name)
    desc, q, qd, g = U.batch(name)
    act = np.zeros((q.shape[0], desc.D), np.float32)
    musc = np.zeros((q.shape[0], desc.M), np.float32) if desc.M else None
    for form, flags in U.FORMULATIONS.items():
        if form == "fma":
            continue
        emu = U.JacobianEmuSim(model, ne, **flags)
        emu.N = q.shape[0]
        J, a = emu.jacobian_state(q, qd)
        _, _, _, dumps = emu.forward(q, qd, act, musc, 1, 1, 1.0 / 960.0, tape=False, derived=True)
        assert np.array_equal(J, U.assemble_J(desc, dumps["joint_S_s"])), (name, form)
        assert np.array_equal(a.ravel(), dumps["body_a_s"].ravel()), (name, form)


@pytest.mark.parametrize("name", U.DIFFRL)
def test_jacobian_state_matches_reference_goldens(name):
    d, model = load_golden(name)
    ne = int(d["meta/num_envs"])
    cases = sorted({k.split("/")[0] for k in d if k.startswith("case") and k.endswith("/first/joint_S_s")})
    assert cases, name
    emu = U.JacobianEmuSim(model, ne)
    tf = jacobian_state_tol(name, "fwd")
    for c in cases:
        q, qd = d[c + "/q0"].reshape(ne, -1), d[c + "/qd0"].reshape(ne, -1)
        J, a = emu.jacobian_state(q, qd)
        ref = (U.assemble_J(emu.desc, d[c + "/first/joint_S_s"].reshape(ne, -1, 6)), d[c + "/first/body_a_s"].reshape(ne, -1, 6))
        for block, err in U.forward_errors((J, a), ref).items():
            assert err.max() <= tf, (name, c, block, float(err.max()), tf)


def _linear_dq(desc):
    """every joint's dq/dt is qd (no ball or free joints)"""
    return all(int(t) not in (R.BALL, R.FREE) for t in desc.arrays["joint_type"][:desc.L])


@pytest.mark.parametrize("name", [n for n in U.MODELS if _linear_dq(U.batch(n, n=12)[0])])
def test_point_bias_acceleration_of_the_documented_formula(name):
    o = U.oracle_of(name)
    desc, q, qd, _ = U.batch(name, n=12)
    q, qd = q.astype(np.float64), qd.astype(np.float64)
    rng = np.random.default_rng(4)
    h = 1e-4
    for e in range(q.shape[0]):
        J, a = o.jacobian_state(q[e:e + 1], qd[e:e + 1])
        X_sc, _, v = o.link_state(q[e:e + 1], qd[e:e + 1])
        for i in range(desc.L):
            pb = rng.standard_normal(3) * 0.3          # a point fixed to link i, in its frame

            def world(t):
                Xs = o.link_state(q[e:e + 1] + t * qd[e:e + 1], qd[e:e + 1])[0][0, i]
                x, y, z, w = Xs[3:]
                R3 = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                               [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                               [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
                return Xs[:3] + R3 @ pb
            p = world(0.0)
            fd = (world(h) - 2 * p + world(-h)) / (h * h)
            w_, vo = v[0, i, :3], v[0, i, 3:]
            aw, av = a[0, i, :3], a[0, i, 3:]
            b = av + np.cross(aw, p) + np.cross(w_, vo + np.cross(w_, p))
            assert np.abs(b - fd).max() <= 1e-4 * (1.0 + np.abs(fd).max()), (name, e, i, b, fd)
            # and the point Jacobian J_v - [p]x J_w gives the point's velocity
            Jp = J[0, i, 3:] - np.cross(p[None, :], J[0, i, :3].T).T
            dp = (world(h) - world(-h)) / (2 * h)
            assert np.abs(Jp @ qd[e] - dp).max() <= 1e-6 * (1.0 + np.abs(dp).max()), (name, e, i)


@pytest.mark.parametrize("name", sorted(JACOBIAN_CONTROL_MEASURED))
def test_emulated_controlled_rollout_matches_oracle(name):
    model, meta, q0, qd0, u, W = U.control_case(name, 8)
    o = U.oracle_of(name)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    rng = np.random.default_rng(9)
    g_q, g_qd = rng.standard_normal(q0.shape).astype(np.float32), rng.standard_normal(qd0.shape).astype(np.float32)
    for form in ("group", "fused", "fma"):
        emu = U.JacobianEmuSim(model, meta["num_envs"], **U.FORMULATIONS[form])
        emu.N = q0.shape[0]
        qT, qdT, gq, gqd, gu = U.emu_control_rollout(emu, q0, qd0, u, W, g_q, g_qd, S, mm, dt)
        rq, rqd = o.controlled_rollout(q0[0], qd0[0], u[:, 0], None, W, U.CONTROL_KAPPA, S, mm, dt)
        assert max(U.U.rel_err(qT[0], rq), U.U.rel_err(qdT[0], rqd)) < 1e-4, (name, form)
        err = U.control_errors(o, q0, qd0, u, W, g_q, g_qd, gq, gqd, gu, S, mm, dt, envs=range(2))
        print(name, form, {k: "%.1e" % v for k, v in err.items()})
        for k, v in err.items():
            assert v <= jacobian_control_tol(name, k), (name, form, k, v, jacobian_control_tol(name, k))
