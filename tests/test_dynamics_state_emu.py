"""The dynamics state (include/dfx.h dfx_dynamics_state_forward / _backward) in the host emulation of every kernel formulation,
against the fp64 oracle (tests/dynamics_oracle/dynamics_oracle.c) and the reference's own goldens.

  * the oracle's complex-step gradient equals fp64 central differences of its own forward;
  * on the six DiffRL models and the random articulations, with the ground on and off and with and without an external wrench,
    the emulated forward and adjoint agree with the oracle per environment and block (dynamics_tolerances.dynamics_tol), the
    adjoint with a NON-symmetric cotangent of H;
  * joint_qdd, joint_tau and H equal the reference's goldens case*/first/{joint_qdd, joint_tau, H} at case*/{q0, qd0, act[, musc]};
  * they are the derived dumps of a one-substep emulated env-step under the same wrench, bit for bit;
  * convention: a one-substep env-step gives qd_out = qd + dt qdd within the fp32 rounding of that update, and for a loss on qd_out
    alone the step adjoint equals the dynamics adjoint seeded with g_qdd = dt g, plus g on gqd."""
import numpy as np
import pytest

import dynamics_util as U
from dynamics_tolerances import CONVENTION_BOUND, CONVENTION_GRAD_BOUND, dynamics_tol, golden_tol
from emu_util import load_golden

EXACT_ENVS = range(4)       # environments per batch whose adjoint is checked against the complex-step gradient


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv", "SNUHumanoidEnv", "gen_mixed"])
def test_oracle_dynamics_gradient_matches_central_differences(name):
    o = U.oracle_of(name)
    desc, inp, g = U.batch(name)
    D, Q, M, L = desc.D, desc.Q, desc.M, desc.L
    e = 1
    parts = [inp["q"][e], inp["qd"][e], inp["act"][e]] + ([inp["musc"][e]] if M else []) + [inp["f_ext"][e].ravel()]
    x = np.concatenate(parts).astype(np.float64)
    sizes = [Q, D, D] + ([M] if M else []) + [L * 6]
    cut = np.cumsum(sizes)[:-1]

    def loss(v):
        p = np.split(v, cut)
        musc = p[3][None] if M else None
        out = o.dynamics_state(p[0][None], p[1][None], p[2][None], musc, p[-1][None])
        return sum(float(np.dot(a.ravel(), b.ravel().astype(np.float64))) for a, b in zip(out, (g[0][e], g[1][e], g[2][e])))
    ex = o.dynamics_state_gradient(inp["q"][e], inp["qd"][e], inp["act"][e], None if not M else inp["musc"][e], inp["f_ext"][e],
                                   g[0][e], g[1][e], g[2][e])
    exact = np.concatenate([ex[0], ex[1], ex[2]] + ([ex[3]] if M else []) + [ex[4].ravel()])
    fd = np.zeros_like(x)
    for i in range(x.size):
        h = 1e-6 * (1.0 + abs(x[i]))
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        fd[i] = (loss(xp) - loss(xm)) / (2 * h)
    assert np.abs(fd).max() > 0
    assert U.rel_err(exact, fd) < 1e-5, (name, U.rel_err(exact, fd))


def _check_against_oracle(name, ground, wrench, forms):
    model, ne = U.model_of(name)
    o = U.oracle_of(name)
    o.set_ground(ground)
    desc, inp, g = U.batch(name, wrench=wrench)
    ref = U.reference(name, o, inp)
    envs = list(EXACT_ENVS)
    exact = U.exact_gradients(name, o, inp, g, envs)
    worst, skipped = {}, 0
    for form in forms:
        emu = U.DynamicsEmuSim(model, ne, **U.FORMULATIONS[form])
        emu.N = inp["q"].shape[0]
        emu.set_ground(ground)
        # environments whose one-substep env-step is itself non-finite (gen_deep24 has one) are skipped by count
        _, qd_out, _, _ = emu.forward(inp["q"], inp["qd"], inp["act"], inp["musc"], 1, 1, 1.0 / 960.0, f_ext=inp["f_ext"])
        ok = U.finite_rows(np.asarray(qd_out).reshape(emu.N, -1))
        skipped = max(skipped, int((~ok).sum()))
        out = emu.dynamics_state(inp["q"], inp["qd"], inp["act"], inp["musc"], inp["f_ext"])
        for field, err in U.forward_errors(out, ref).items():
            err = err[ok]
            worst[field] = max(worst.get(field, 0.0), float(err.max()))
            assert err.max() <= dynamics_tol(name, field), (name, form, field, int(err.argmax()), float(err.max()))
        grads = emu.dynamics_state_backward(inp["q"], inp["qd"], inp["act"], inp["musc"], inp["f_ext"], *g)
        got = [None if x is None else x[envs] for x in grads]
        for field, err in U.grad_errors(got, exact).items():
            err = err[ok[envs]]
            worst[field] = max(worst.get(field, 0.0), float(err.max(initial=0.0)))
            assert err.max(initial=0.0) <= dynamics_tol(name, field), (name, form, field, int(err.argmax()), float(err.max()))
    print("measured", name, ground, wrench, {k: "%.1e" % v for k, v in worst.items()}, "non-finite env-steps skipped", skipped)


@pytest.mark.parametrize("name", U.MODELS)
def test_emulated_dynamics_state_matches_oracle_every_formulation(name):
    _check_against_oracle(name, True, True, list(U.FORMULATIONS))


@pytest.mark.parametrize("wrench", [True, False], ids=["f_ext", "no_f_ext"])
@pytest.mark.parametrize("ground", [True, False], ids=["ground", "no_ground"])
@pytest.mark.parametrize("name", U.MODELS)
def test_emulated_dynamics_state_matches_oracle_ground_and_wrench(name, ground, wrench):
    if ground and wrench:
        pytest.skip("covered by every formulation above")
    _check_against_oracle(name, ground, wrench, ["group", "tile8m3"])


def golden_inputs(name, case):
    d, model = load_golden(name)
    ne = int(d["meta/num_envs"])
    p = "case%d/" % case
    D, M = int(d["meta/joint_dof_count"]) // ne, int(d["meta/muscle_count"]) // ne
    f = lambda k: np.asarray(d[p + k], np.float32)
    inp = dict(q=f("q0").reshape(ne, -1), qd=f("qd0").reshape(ne, D), act=f("act").reshape(ne, D),
               musc=f("musc").reshape(ne, M) if M else None, f_ext=None)
    ref = (f("first/joint_qdd").reshape(ne, D), f("first/joint_tau").reshape(ne, D), f("first/H").reshape(ne, D, D))
    return d, model, ne, inp, ref


@pytest.mark.parametrize("name", U.DIFFRL)
def test_emulated_dynamics_state_matches_reference_goldens(name):
    d, _, _, _, _ = golden_inputs(name, 0)
    cases = sorted({int(k.split("/")[0][4:]) for k in d.files if k.startswith("case") and k.endswith("/first/H")})
    assert cases
    for case in cases:
        _, model, ne, inp, ref = golden_inputs(name, case)
        for form in ("group", "tile8m3", "fma"):
            emu = U.DynamicsEmuSim(model, ne, **U.FORMULATIONS[form])
            out = emu.dynamics_state(**inp)
            for field, got, r in zip(U.FIELDS, out, ref):
                err = U.rel_err(got, r)
                assert err <= golden_tol(name, field), (name, case, form, field, err)


@pytest.mark.parametrize("wrench", [True, False], ids=["f_ext", "no_f_ext"])
@pytest.mark.parametrize("name", U.MODELS)
def test_dynamics_state_is_the_one_substep_derived_dumps_bit_for_bit(name, wrench):
    from diffrl_b200.modelpack import DfxDerived
    from emu_util import fptr
    model, ne = U.model_of(name)
    desc, inp, _ = U.batch(name, wrench=wrench)
    n, D = inp["q"].shape[0], desc.D
    for form in ("group", "tile8m3", "fused"):
        emu = U.DynamicsEmuSim(model, ne, **U.FORMULATIONS[form])
        emu.N = n
        out = emu.dynamics_state(**inp)
        dumps = dict(joint_qdd=np.zeros((n, D), np.float32), joint_tau=np.zeros((n, D), np.float32), H=np.zeros((n, D, D), np.float32))
        dv = DfxDerived()
        for k, v in dumps.items():
            setattr(dv, k, v.ctypes.data)
        c = lambda x: None if x is None else np.ascontiguousarray(x, np.float32)
        q_out, qd_out = np.empty_like(inp["q"]), np.empty_like(inp["qd"])
        tape = np.zeros(emu.lib.emu_tape_floats(emu.pack, n, 1, 1), np.float32)
        f_ext = inp["f_ext"] if wrench else np.zeros((n, desc.L, 6), np.float32)
        emu.lib.emu_step_forward_ext(emu.pack, n, 1, 1, 1.0 / 960.0, fptr(c(inp["q"])), fptr(c(inp["qd"])), fptr(c(inp["act"])),
                                     fptr(c(inp["musc"])), fptr(q_out), fptr(qd_out), fptr(tape), __import__("ctypes").byref(dv),
                                     fptr(c(f_ext)))
        for field, got in zip(U.FIELDS, out):
            ok = U.finite_rows(got)
            assert np.array_equal(got[ok], dumps[field][ok]), (name, form, field)


@pytest.mark.parametrize("name", U.MODELS)
def test_convention_one_substep_env_step(name):
    model, ne = U.model_of(name)
    desc, inp, _ = U.batch(name)
    n, D = inp["q"].shape[0], desc.D
    dt = 1.0 / 960.0
    rng = np.random.default_rng(23)
    g = rng.standard_normal((n, D)).astype(np.float32)
    for form in ("group", "tile8m3"):
        emu = U.DynamicsEmuSim(model, ne, **U.FORMULATIONS[form])
        emu.N = n
        qdd = emu.dynamics_state(**inp)[0]
        _, qd_out, tape, _ = emu.forward(inp["q"], inp["qd"], inp["act"], inp["musc"], 1, 1, dt, f_ext=inp["f_ext"])
        qd_out = qd_out.reshape(n, D)
        ok = U.finite_rows(qdd, qd_out)
        assert ok.sum() >= n // 2, (name, int(ok.sum()))
        err = U.convention_error(inp["qd"][ok], qdd[ok], qd_out[ok], dt)
        assert err.max() <= CONVENTION_BOUND, (name, form, float(err.max()))
        # adjoint: a loss on qd_out alone
        sg = emu.backward(inp["act"], inp["musc"], tape, np.zeros_like(inp["q"]), g, 1, 1, dt, f_ext=inp["f_ext"])
        dgq, dgqd, dgact, dgmusc, dgf = emu.dynamics_state_backward(inp["q"], inp["qd"], inp["act"], inp["musc"], inp["f_ext"],
                                                                    g * np.float32(dt), None, None)
        dyn = [dgq, dgqd + g, dgact, dgmusc, dgf]
        step = [np.asarray(x).reshape(n, -1) if x is not None else None for x in sg]
        ok &= U.finite_rows(*[x for x in step if x is not None])
        pairs = [(k, np.asarray(a, np.float64).reshape(n, -1)[ok], np.asarray(b, np.float64).reshape(n, -1)[ok])
                 for k, (a, b) in enumerate(zip(step, dyn)) if a is not None and b is not None]
        scale = np.maximum(np.max([np.abs(a).max(axis=1, initial=0.0) for _, a, _ in pairs], axis=0), 1e-30)
        for k, a, b in pairs:
            err = (np.abs(a - b).max(axis=1, initial=0.0) / scale).max(initial=0.0)
            assert err <= CONVENTION_GRAD_BOUND, (name, form, U.GRAD_NAMES[k], err)
