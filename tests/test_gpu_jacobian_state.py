"""The Jacobian state (include/dfx.h dfx_jacobian_state_forward / _backward) on the kernels.

* the six DiffRL articulations and the random articulations on every kernel family that exists for them -- auto, tile8/16/32,
  group8/16/32 and the generic lane-group instantiation (flag 4) -- at N = 1 and N = 75: the forward per environment and block
  against the fp64 oracle, the adjoint per environment and gradient block against the exact gradient, within
  jacobian_tolerances.jacobian_state_tol;
* on the same family: J equals the spatial.h rule applied to the one-substep derived joint_S_s dump and body_a_s the body_a_s dump
  (within that bound; whether bit for bit is printed); J[n, i, r, :] is gqd of link_state_backward seeded with the one-hot g_v_s[i, r]
  (an independent code path); einsum(J, qd) is link_state's body_v_s; through the C ABI nothing past environment N - 1 of
  over-allocated buffers is written, all-NULL outputs launch nothing, each direction is one launch, and two calls are bitwise equal;
* composition: 4 env-steps of SimStepFunction under act_t = u_t + J(q_t)^T (W + kappa body_a_s(q_t, qd_t)) (JacobianStateFunction), so
  both cotangents feed back through the step; gradients of (u, q0, qd0) against the oracle's exact gradient of the same rollout
  (jacobian_tolerances.jacobian_control_tol), tape and recompute adjoint modes bitwise equal;
* env.jacobian_state() after fused env-steps of the Ant and Humanoid envs, and the refusals (ValueError) of bad inputs."""
import contextlib
import ctypes

import numpy as np
import pytest

import jacobian_util as U
from jacobian_tolerances import jacobian_control_tol, jacobian_state_tol
from link_tolerances import link_state_tol
from test_gpu_link_state import CASES

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _selected(variant):
    """the kernel family `variant` for packs created and launches made inside: the tile width is read when a pack is created, the
    group width and flag 4 (generic instantiation) at every launch, so the selection is held around the launches too"""
    from test_gpu_golden import _select as select
    from diffrl_b200 import _capi
    try:
        if variant == "generic":
            select("auto")
            _capi.lib().dfx_set_flags(9 | 32 | 4)
        else:
            select(variant)
        yield
    finally:
        select("auto")


def _engine(name, variant, n):
    """an engine of the model for n environments, created inside _selected(variant): its pack is on the selected family (tile
    width, or lane groups of the forced width)"""
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    model, ne = U.U.model_of(name)
    desc, _ = U.U.articulation_from_model(model, ne)
    eng = ArticulationEngine(desc, n, "cuda:0")
    tile = int(_capi.lib().dfx_pack_query(eng.pack, 9))
    if variant.startswith("tile"):
        assert tile == int(variant[4:]), (name, variant, tile)
    elif variant != "auto":
        assert tile == 0, (name, variant, tile)
    if variant.startswith("group"):          # the launches run the forced group width
        plan = (ctypes.c_int * 6)()
        for bwd in (0, 1):
            assert eng.lib.dfx_launch_plan(eng.pack, bwd, plan) == 0
            assert plan[0] == int(variant[5:]), (name, variant, bwd, list(plan))
    return eng


def _t(a):
    import torch
    return None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda:0")


def _run(eng, q, qd, g):
    out = eng.jacobian_state(_t(q), _t(qd))
    gq, gqd = eng.jacobian_state_backward(_t(q), _t(qd), *(_t(x) for x in g))
    return [o.cpu().numpy() for o in out], gq.view(q.shape).cpu().numpy(), gqd.view(qd.shape).cpu().numpy()


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_jacobian_state_matches_oracle(name, variant):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    egq, egqd = U.exact_gradients(name, o, q, qd, g)
    tf, tg = jacobian_state_tol(name, "fwd"), jacobian_state_tol(name, "grad")
    mask = U.ancestor_mask(desc)
    worst = {}
    with _selected(variant):
        for n in (1, 75):
            eng = _engine(name, variant, n)
            out, gq, gqd = _run(eng, q[:n], qd[:n], tuple(x[:n] for x in g))
            assert not out[0].transpose(0, 2, 1, 3)[:, :, ~mask].any(), (name, variant, "J is not exactly 0 where no dof moves the link")
            for block, err in U.forward_errors(out, tuple(r[:n] for r in ref)).items():
                assert err.max() <= tf, (name, variant, n, block, int(err.argmax()), float(err.max()), tf)
                worst["fwd"] = max(worst.get("fwd", 0.0), float(err.max()) / tf)
            for block, err in U.grad_errors(desc, gq, gqd, egq[:n], egqd[:n]).items():
                assert err.max() <= tg, (name, variant, n, block, int(err.argmax()), float(err.max()), tg)
                worst["grad"] = max(worst.get("grad", 0.0), float(err.max()) / tg)
    print(name, variant, "worst error / bound", {k: "%.2f" % v for k, v in worst.items()})


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_jacobian_state_dumps_link_state_and_abi(name, variant):
    with _selected(variant):     # (every launch below, the step's and the link state's included, runs on the selected family)
        _dumps_link_state_and_abi(name, variant)


def _dumps_link_state_and_abi(name, variant):
    import torch
    from diffrl_b200 import _capi
    desc, q, qd, g = U.batch(name)
    n, L, Q, D = q.shape[0], desc.L, desc.Q, desc.D
    eng = _engine(name, variant, n)
    out, gq, gqd = _run(eng, q, qd, g)
    tf = jacobian_state_tol(name, "fwd")
    # the step's derived dumps of a one-substep call on the same family
    act = torch.zeros((n, D), device="cuda:0")
    musc = torch.zeros((n, desc.M), device="cuda:0") if desc.M else None
    _, _, _, dumps = eng.forward(_t(q), _t(qd), act, musc, 1, 1, 1.0 / 960.0, want_tape=False, derived=["joint_S_s", "body_a_s"])
    dumped = (U.assemble_J(desc, dumps["joint_S_s"].cpu().numpy()), dumps["body_a_s"].view(n, L, 6).cpu().numpy())
    for block, err in U.forward_errors(out, dumped).items():
        assert err.max() <= tf, (name, variant, block, float(err.max()), tf)
    print(name, variant, "Jacobian state == one-substep derived dumps bit for bit:",
          all(np.array_equal(a, b) for a, b in zip(out, dumped)))
    # J qd is the link state's body_v_s; row (i, r) of J is the gradient of body_v_s[i, r] with respect to qd (per environment, within
    # the two ops' bounds: J's scaled by sum |qd|, the link state's forward or adjoint one)
    Jd = out[0].astype(np.float64)
    scale_J = np.abs(Jd).reshape(n, -1).max(axis=1)
    v_s = eng.link_state(_t(q), _t(qd), want=("body_v_s",))[2].cpu().numpy()
    err = np.abs(np.einsum("nird,nd->nir", Jd, qd) - v_s).reshape(n, -1).max(axis=1)
    bound = tf * scale_J * np.abs(qd).sum(axis=1) + link_state_tol(name, "fwd") * np.abs(v_s).reshape(n, -1).max(axis=1)
    assert (err <= bound).all(), (name, variant, int((err / bound).argmax()), float((err / bound).max()))
    gv = np.zeros((n, L, 6), np.float32)
    tg = tf + link_state_tol(name, "grad")
    for i in range(L):
        for r in range(6):
            gv[:] = 0.0
            gv[:, i, r] = 1.0
            _, col = eng.link_state_backward(_t(q), _t(qd), None, None, _t(gv), need=(False, True))
            err = np.abs(col.view(n, D).cpu().numpy() - Jd[:, i, r, :]).max(axis=1)
            assert (err <= tg * scale_J).all(), (name, variant, i, r, float((err / scale_J).max()), tg)
    # two calls: bitwise equal
    out2, gq2, gqd2 = _run(eng, q, qd, g)
    assert all(np.array_equal(a, b) for a, b in zip(out, out2)) and np.array_equal(gq, gq2) and np.array_equal(gqd, gqd2)
    # the C ABI with buffers of n + 5 environments, pre-filled: nothing past environment n - 1 is written; one launch each way;
    # all-NULL outputs launch nothing
    extra, fill = 5, 12345.0
    bufs = [torch.full(((n + extra) * L * w,), fill, device="cuda:0") for w in (6 * D, 6)]
    grads = [torch.full(((n + extra) * w,), fill, device="cuda:0") for w in (Q, D)]
    qt, qdt = _t(q), _t(qd)
    gt = [_t(x) for x in g]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    lib = _capi.lib()
    c0 = lib.dfx_launch_count()
    assert eng.lib.dfx_jacobian_state_forward(eng.pack, n, p(qt), p(qdt), *(p(b) for b in bufs), stream) == 0
    c1 = lib.dfx_launch_count()
    assert eng.lib.dfx_jacobian_state_backward(eng.pack, n, p(qt), p(qdt), *(p(x) for x in gt), *(p(x) for x in grads), stream) == 0
    c2 = lib.dfx_launch_count()
    assert eng.lib.dfx_jacobian_state_forward(eng.pack, n, p(qt), p(qdt), None, None, stream) == 0
    assert eng.lib.dfx_jacobian_state_backward(eng.pack, n, p(qt), p(qdt), p(gt[0]), p(gt[1]), None, None, stream) == 0
    assert (c1 - c0, c2 - c1, lib.dfx_launch_count() - c2) == (1, 1, 0), (name, variant)
    torch.cuda.synchronize()
    for b, w, ref in zip(bufs, (6 * D, 6), out):
        assert bool((b[n * L * w:] == fill).all()), (name, variant)
        assert np.array_equal(b[:n * L * w].cpu().numpy(), ref.ravel())
    for b, w, ref in zip(grads, (Q, D), (gq, gqd)):
        assert bool((b[n * w:] == fill).all()), (name, variant)
        assert np.array_equal(b[:n * w].cpu().numpy(), ref.ravel())


# ------------------------------------------------------------------ composition with the step
def _control_grads(eng, q0, qd0, u, W, g_q, g_qd, S, mm, dt):
    import torch
    from diffrl_b200.engine import JacobianStateFunction, SimStepFunction
    q = _t(q0).requires_grad_(True)
    qd = _t(qd0).requires_grad_(True)
    us = [_t(x).requires_grad_(True) for x in u]
    Wt = _t(W)
    qi, qdi = q, qd
    for t in range(len(us)):
        J, a = JacobianStateFunction.apply(eng, qi, qdi)
        act = us[t] + torch.einsum("nlrd,nlr->nd", J, Wt[None] + U.CONTROL_KAPPA * a)
        qi, qdi = SimStepFunction.apply(eng, S, mm, dt, qi, qdi, act, None)
    loss = (qi.view(q.shape) * _t(g_q)).sum() + (qdi.view(qd.shape) * _t(g_qd)).sum()
    loss.backward()
    return q.grad, qd.grad, torch.stack([x.grad for x in us])


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv"])
def test_controlled_rollout_gradient_matches_oracle_in_both_adjoint_modes(name):
    import torch
    import diffrl_b200
    from diffrl_b200.engine import ArticulationEngine
    model, meta, q0, qd0, u, W = U.control_case(name, 8)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    desc, _ = U.U.articulation_from_model(model, meta["num_envs"])
    eng = ArticulationEngine(desc, q0.shape[0], "cuda:0")
    rng = np.random.default_rng(9)
    g_q, g_qd = rng.standard_normal(q0.shape).astype(np.float32), rng.standard_normal(qd0.shape).astype(np.float32)
    tape = _control_grads(eng, q0, qd0, u, W, g_q, g_qd, S, mm, dt)
    diffrl_b200.set_adjoint_mode("recompute")
    try:
        rec = _control_grads(eng, q0, qd0, u, W, g_q, g_qd, S, mm, dt)
    finally:
        diffrl_b200.set_adjoint_mode("tape")
    for a, b in zip(tape, rec):
        assert torch.equal(a, b), name
    o = U.oracle_of(name)
    gq, gqd, gu = (x.cpu().numpy() for x in tape)
    err = U.control_errors(o, q0, qd0, u, W, g_q, g_qd, gq, gqd, gu, S, mm, dt, envs=range(2))
    print(name, "controlled rollout error / bound", {k: "%.2f" % (v / jacobian_control_tol(name, k)) for k, v in err.items()})
    for k, v in err.items():
        assert v <= jacobian_control_tol(name, k), (name, k, v, jacobian_control_tol(name, k))


# ------------------------------------------------------------------ the envs and the refusals
@pytest.mark.parametrize("env_name", ["AntEnv", "HumanoidEnv"])
def test_env_jacobian_state_after_fused_steps(env_name):
    import torch
    import diffrl_b200
    from diffrl_b200 import envs
    env = getattr(envs, env_name)(num_envs=8, device="cuda:0", no_grad=False)
    env.reset()
    acts = [torch.full((env.num_envs, env.num_actions), 0.3 * (k + 1), device="cuda:0", requires_grad=True) for k in range(3)]
    for a in acts:
        env.step(a)
    J, a_s = env.jacobian_state()
    q, qd = env.state.joint_q, env.state.joint_qd
    ref = diffrl_b200.jacobian_state(env.model, q, qd)
    assert torch.equal(J, ref.J) and torch.equal(a_s, ref.body_a_s)
    v_s = env.link_state().body_v_s
    N, L, _, D = J.shape
    assert (N, L) == (env.num_envs, v_s.shape[1])
    assert float((torch.einsum("nird,nd->nir", J.double(), qd.view(N, D).double()) - v_s.double()).abs().max()) <= \
        1e-5 * (1.0 + float(v_s.abs().max()))
    # a loss on J and body_a_s reaches the actions through the steps that produced the state
    (J.square().sum() + a_s.square().sum()).backward()
    for a in acts:
        assert a.grad is not None and bool(torch.isfinite(a.grad).all()) and float(a.grad.abs().max()) > 0, env_name


def test_jacobian_state_refuses_bad_inputs():
    import torch
    from diffrl_b200.engine import JacobianStateFunction
    eng = _engine("AntEnv", "auto", 4)
    q = torch.zeros((4, eng.Q), device="cuda:0")
    q[:, 6] = 1.0
    qd = torch.zeros((4, eng.D), device="cuda:0")
    for bad_q, bad_qd in ((q[:, :-1], qd), (q.double(), qd), (q.cpu(), qd), (q, qd[:3]), (q, "x")):
        with pytest.raises(ValueError):
            eng.jacobian_state(bad_q, bad_qd)
        with pytest.raises(ValueError):
            JacobianStateFunction.apply(eng, bad_q, bad_qd)
    gJ = torch.zeros((4, eng.L, 6, eng.D), device="cuda:0")
    for bad in (gJ[:, :, :5], gJ.double(), gJ.cpu()):
        with pytest.raises(ValueError):
            eng.jacobian_state_backward(q, qd, bad, None)
    for ok in (gJ, gJ.view(4, 6 * eng.L, eng.D), gJ.view(-1)):
        eng.jacobian_state_backward(q, qd, ok, None)
