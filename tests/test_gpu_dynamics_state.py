"""The dynamics state (include/dfx.h dfx_dynamics_state_forward / _backward) on the kernels.

* the six DiffRL articulations and the random articulations on every kernel family that exists for them -- auto, tile8/16/32,
  group8/16/32 and the generic lane-group instantiation (flag 4) -- at N = 1 and N = 75: the forward per environment and field
  against the fp64 oracle, the adjoint (non-symmetric g_H) against the exact gradient, within dynamics_tolerances.dynamics_tol;
  the worst error over its bound is printed per case;
* on the same family: the outputs are the derived dumps of dfx_step_forward_ex with substeps = 1 under the same wrench, bit for
  bit; the convention check (qd_out = qd + dt qdd of that env-step, and the step adjoint of a loss on qd_out against the seeded
  dynamics adjoint); nothing past environment N - 1 of over-allocated buffers is written; two calls are bitwise equal; a
  non-finite q in one environment leaves every other environment unchanged.  Environments whose one-substep env-step is itself
  non-finite are skipped by count, and the count is printed;
* the reference's goldens case*/first/{joint_qdd, joint_tau, H};
* composition: T = 3 env-steps of SimStepFunction, loss 1/2 qd^T H qd + |tau|^2 + w . qdd on the end state, against the oracle's
  exact gradient, tape and recompute adjoint modes bitwise equal;
* env.dynamics_state(actions) on the Ant, Humanoid and SNU envs, and the refusals."""
import contextlib
import ctypes

import numpy as np
import pytest

import dynamics_util as U
from dynamics_tolerances import CONVENTION_BOUND, CONVENTION_GRAD_BOUND, dynamics_tol, golden_tol, rollout_tol
from test_dynamics_state_emu import EXACT_ENVS, golden_inputs

pytestmark = pytest.mark.gpu

TILES = {"CartPoleSwingUpEnv": (32,), "AntEnv": (8, 16, 32), "HopperEnv": (32,), "CheetahEnv": (32,), "HumanoidEnv": (8, 16),
         "SNUHumanoidEnv": (8, 16)}
NB = 75


def _tiles(name):
    return TILES.get(name[len("twin_"):] if name.startswith("twin_") else name, ())


CASES = [(name, v) for name in U.MODELS
         for v in ["auto"] + ["tile%d" % e for e in _tiles(name)] + ["group8", "group16", "group32", "generic"]]


@contextlib.contextmanager
def _selected(variant):
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
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    model, ne = U.model_of(name)
    desc, _ = U.articulation_from_model(model, ne)
    eng = ArticulationEngine(desc, n, "cuda:0")
    tile = int(_capi.lib().dfx_pack_query(eng.pack, 9))
    if variant.startswith("tile"):
        assert tile == int(variant[4:]), (name, variant, tile)
    elif variant != "auto":
        assert tile == 0, (name, variant, tile)
    return eng


def _t(a):
    import torch
    return None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda:0")


def _sub(inp, n):
    return {k: None if v is None else v[:n] for k, v in inp.items()}


def _run(eng, inp, g):
    ti = [_t(inp[k]) for k in ("q", "qd", "act", "musc", "f_ext")]
    out = eng.dynamics_state(*ti)
    grads = eng.dynamics_state_backward(*ti, *(_t(x) for x in g))
    n = inp["q"].shape[0]
    return [o.cpu().numpy() for o in out], [None if x is None else x.cpu().numpy().reshape(n, -1) for x in grads]


def _step_ok(eng, inp):
    """[n] bool: environments whose one-substep env-step (dfx_step_forward_ex) is finite"""
    import torch
    _, qd_out, _, _ = eng.forward(_t(inp["q"]), _t(inp["qd"]), _t(inp["act"]), _t(inp["musc"]), 1, 1, 1.0 / 960.0, want_tape=False,
                                  f_ext=_t(inp["f_ext"]))
    return torch.isfinite(qd_out.view(inp["q"].shape[0], -1)).all(dim=1).cpu().numpy()


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_dynamics_state_matches_oracle(name, variant):
    o = U.oracle_of(name)
    desc, inp, g = U.batch(name, NB)
    ref = U.reference(name, o, inp)
    envs = list(EXACT_ENVS)
    exact = U.exact_gradients(name, o, inp, g, envs)
    worst, absolute, skipped = {}, {}, 0
    with _selected(variant):
        for n in (1, NB):
            eng = _engine(name, variant, n)
            sub = _sub(inp, n)
            ok = _step_ok(eng, sub)
            skipped += int((~ok).sum())
            out, grads = _run(eng, sub, tuple(x[:n] for x in g))
            for field, err in U.forward_errors(out, tuple(r[:n] for r in ref)).items():
                err = err[ok]
                b = dynamics_tol(name, field)
                assert (err <= b).all(), (name, variant, n, field, float(err.max()), b)
                worst[field] = max(worst.get(field, 0.0), float(err.max(initial=0.0)) / b)
                absolute[field] = max(absolute.get(field, 0.0), float(err.max(initial=0.0)))
            m = min(n, len(envs))
            got = [None if x is None else x[:m] for x in grads]
            ex = [None if x is None else x[:m] for x in exact]
            for field, err in U.grad_errors(got, ex).items():
                err = err[ok[:m]]
                b = dynamics_tol(name, field)
                assert (err <= b).all(), (name, variant, n, field, float(err.max()), b)
                worst[field] = max(worst.get(field, 0.0), float(err.max(initial=0.0)) / b)
                absolute[field] = max(absolute.get(field, 0.0), float(err.max(initial=0.0)))
    print(name, variant, "worst error / bound", {k: "%.2f" % v for k, v in worst.items()}, "non-finite env-steps skipped", skipped)
    print("measured", name, variant, {k: "%.1e" % v for k, v in absolute.items()})


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_dynamics_state_dumps_convention_abi_and_determinism(name, variant):
    import torch
    desc, inp, g = U.batch(name, NB)
    n, L, Q, D, M = NB, desc.L, desc.Q, desc.D, desc.M
    dt = 1.0 / 960.0
    with _selected(variant):
        eng = _engine(name, variant, n)
        ok = _step_ok(eng, inp)
        out, grads = _run(eng, inp, g)
        out2, grads2 = _run(eng, inp, g)
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(out, out2))
        assert all(a is None or np.array_equal(a, b, equal_nan=True) for a, b in zip(grads, grads2))
        # the derived dumps of a one-substep env-step under the same wrench, bit for bit
        ti = [_t(inp[k]) for k in ("q", "qd", "act", "musc", "f_ext")]
        _, qd_out, tape, dumps = eng.forward(ti[0], ti[1], ti[2], ti[3], 1, 1, dt, derived=("joint_qdd", "joint_tau", "H"), f_ext=ti[4])
        for field, got in zip(U.FIELDS, out):
            d = dumps[field].view(got.shape).cpu().numpy()
            assert np.array_equal(got[ok], d[ok]), (name, variant, field)
        # convention: qd_out = qd + dt qdd; the step adjoint of a loss on qd_out is the seeded dynamics adjoint
        qd_out = qd_out.view(n, D).cpu().numpy()
        err = U.convention_error(inp["qd"][ok], out[0][ok], qd_out[ok], dt)
        assert err.max(initial=0.0) <= CONVENTION_BOUND, (name, variant, float(err.max()))
        gout = np.random.default_rng(29).standard_normal((n, D)).astype(np.float32)
        sg = eng.backward(ti[2], ti[3], tape, None, _t(gout), 1, 1, dt, f_ext=ti[4])
        dg = eng.dynamics_state_backward(*ti, _t(gout * np.float32(dt)), None, None)
        dyn = [dg[0], dg[1] + _t(gout).view(-1), dg[2], dg[3], dg[4]]
        cerr = 0.0
        pairs = [(a.view(n, -1).cpu().double().numpy()[ok], b.view(n, -1).cpu().double().numpy()[ok])
                 for a, b in zip(sg, dyn) if a is not None and b is not None]
        scale = np.maximum(np.max([np.abs(a).max(axis=1, initial=0.0) for a, _ in pairs], axis=0), 1e-30)
        for a, b in pairs:
            cerr = max(cerr, float((np.abs(a - b).max(axis=1, initial=0.0) / scale).max(initial=0.0)))
        assert cerr <= CONVENTION_GRAD_BOUND, (name, variant, cerr)
        print(name, variant, "convention error / bound %.2f, adjoint %.2f" % (err.max(initial=0.0) / CONVENTION_BOUND,
                                                                              cerr / CONVENTION_GRAD_BOUND),
              "non-finite env-steps skipped", int((~ok).sum()))
        # the C ABI with buffers of n + 5 environments, pre-filled: nothing past environment n - 1 is written
        extra, fill = 5, 12345.0
        widths = (D, D, D * D)
        bufs = [torch.full(((n + extra) * w,), fill, device="cuda:0") for w in widths]
        gw = (Q, D, D, M, L * 6)
        gbufs = [torch.full(((n + extra) * w + 1,), fill, device="cuda:0") for w in gw]
        ws = eng.dynamics_workspace()
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        gt = [_t(x) for x in g]
        assert eng.lib.dfx_dynamics_state_forward(eng.pack, n, *(p(x) for x in ti), *(p(b) for b in bufs), stream) == 0
        assert eng.lib.dfx_dynamics_state_backward(eng.pack, n, *(p(x) for x in ti), p(ws), *(p(x) for x in gt),
                                                   *(p(b) if w else None for b, w in zip(gbufs, gw)), stream) == 0
        torch.cuda.synchronize()
        for b, w, r in zip(bufs, widths, out):
            assert bool((b[n * w:] == fill).all()), (name, variant)
            assert np.array_equal(b[:n * w].cpu().numpy(), r.ravel(), equal_nan=True)
        for b, w, r in zip(gbufs, gw, grads):
            if not w:
                continue
            assert bool((b[n * w:] == fill).all()), (name, variant)
            if r is not None:
                assert np.array_equal(b[:n * w].cpu().numpy(), r.ravel(), equal_nan=True)
        # a non-finite q in one environment leaves the others (of its tile and every other) as they were
        bad = 3
        badinp = dict(inp)
        badinp["q"] = inp["q"].copy()
        badinp["q"][bad, 0] = np.nan
        outb, gradsb = _run(eng, badinp, g)
        keep = np.arange(n) != bad
        for a, b in zip(out, outb):
            assert np.array_equal(a[keep], b[keep], equal_nan=True), (name, variant)
        for a, b in zip(grads, gradsb):
            assert a is None or np.array_equal(a[keep], b[keep], equal_nan=True), (name, variant)


@pytest.mark.parametrize("name", U.DIFFRL)
def test_cuda_dynamics_state_matches_reference_goldens(name):
    from diffrl_b200.engine import ArticulationEngine
    d, _, _, _, _ = golden_inputs(name, 0)
    cases = sorted({int(k.split("/")[0][4:]) for k in d.files if k.startswith("case") and k.endswith("/first/H")})
    worst = 0.0
    for case in cases:
        _, model, ne, inp, ref = golden_inputs(name, case)
        eng = ArticulationEngine.from_model(model, "cuda:0", ne)
        out = eng.dynamics_state(*(_t(inp[k]) for k in ("q", "qd", "act", "musc", "f_ext")))
        for field, got, r in zip(U.FIELDS, out, ref):
            err = U.rel_err(got.cpu().numpy(), r)
            assert err <= golden_tol(name, field), (name, case, field, err)
            worst = max(worst, err / golden_tol(name, field))
    print(name, "golden worst error / bound %.2f" % worst)


# ------------------------------------------------------------------ composition with the step
ROLLOUT_W = 0.1


def _rollout_loss_grads(eng, q0, qd0, acts, S, mm, dt):
    import torch
    from diffrl_b200.engine import DynamicsStateFunction, SimStepFunction
    q = _t(q0).requires_grad_(True)
    qd = _t(qd0).requires_grad_(True)
    a = [_t(x).requires_grad_(True) for x in acts]
    qi, qdi = q, qd
    for t in range(len(a) - 1):
        qi, qdi = SimStepFunction.apply(eng, S, mm, dt, qi, qdi, a[t], None)
    qdd, tau, H = DynamicsStateFunction.apply(eng, qi, qdi, a[-1], None, None)
    v = qdi.view(qdd.shape)
    loss = 0.5 * torch.einsum("ni,nij,nj->", v, H, v) + (tau ** 2).sum() + ROLLOUT_W * qdd.sum()
    loss.backward()
    return q.grad, qd.grad, torch.stack([x.grad for x in a])


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv"])
def test_dynamics_rollout_gradient_matches_oracle_in_both_adjoint_modes(name):
    import torch
    import diffrl_b200
    import wrench_util as W
    from diffrl_b200.engine import ArticulationEngine
    model, meta, inp = W.golden_batch(name, 8)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    rng = np.random.default_rng(5)
    acts = np.stack([(inp["act"] * rng.uniform(0.5, 1.5, inp["act"].shape)).astype(np.float32) for _ in range(4)])   # T = 3, + 1
    desc, _ = U.articulation_from_model(model, meta["num_envs"])
    eng = ArticulationEngine(desc, 8, "cuda:0")
    tape = _rollout_loss_grads(eng, inp["q0"], inp["qd0"], acts, S, mm, dt)
    diffrl_b200.set_adjoint_mode("recompute")
    try:
        rec = _rollout_loss_grads(eng, inp["q0"], inp["qd0"], acts, S, mm, dt)
    finally:
        diffrl_b200.set_adjoint_mode("tape")
    for a, b in zip(tape, rec):
        assert torch.equal(a, b), name
    o = U.oracle_of(name)
    gq, gqd, gact = (x.cpu().numpy() for x in tape)
    D = desc.D
    err = dict(gq=0.0, gqd=0.0, gact=0.0)
    for e in range(2):
        qdd, tau, H, qT, qdT = o.rollout(inp["q0"][e], inp["qd0"][e], acts[:, e], S, mm, dt)
        # the cotangent of the rollout's outputs at the exact end state: the loss is linear in none of them
        g = (np.full(D, ROLLOUT_W), 2.0 * tau, 0.5 * np.outer(qdT, qdT), np.zeros_like(qT), (H + H.T) @ qdT * 0.5)
        ex = o.rollout_gradient(inp["q0"][e], inp["qd0"][e], acts[:, e], g, S, mm, dt)
        for k, got, x in zip(("gq", "gqd", "gact"), (gq[e], gqd[e], gact[:, e]), ex):
            err[k] = max(err[k], U.rel_err(got, x))
    print(name, "dynamics rollout error / bound", {k: "%.2f" % (v / rollout_tol()) for k, v in err.items()})
    for k, v in err.items():
        assert v <= rollout_tol(), (name, k, v, rollout_tol())


# ------------------------------------------------------------------ envs
@pytest.mark.parametrize("env_name", ["AntEnv", "HumanoidEnv", "SNUHumanoidEnv"])
def test_env_dynamics_state(env_name):
    import torch
    import diffrl_b200
    from diffrl_b200 import envs
    env = getattr(envs, env_name)(num_envs=8, device="cuda:0", no_grad=False)
    env.reset()
    a0 = torch.full((env.num_envs, env.num_actions), 0.3, device="cuda:0", requires_grad=True)
    env.step(a0)
    a1 = torch.full((env.num_envs, env.num_actions), -0.2, device="cuda:0", requires_grad=True)
    ds = env.dynamics_state(a1)
    D = env.model.joint_dof_count // env.num_envs
    assert ds.joint_qdd.shape == (env.num_envs, D) and ds.H.shape == (env.num_envs, D, D)
    # the same as the public function under the actuation the action map forms
    from diffrl_b200.env_ops import ActionMapFunction
    width, offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = env._action_map()
    _, drive = ActionMapFunction.apply(env.num_envs, width, offset, pre_scale, pre_bias, drive_scale, strength, a1.detach())
    ref = diffrl_b200.dynamics_state(env.model, env.state.joint_q.detach(), env.state.joint_qd.detach(),
                                     None if is_muscle else drive, drive if is_muscle else None)
    for a, b in zip(ds, ref):
        assert torch.equal(a.detach(), b), env_name
    loss = (ds.joint_tau ** 2).sum() + ds.joint_qdd.abs().sum() + ds.H.diagonal(dim1=1, dim2=2).sum()
    loss.backward()
    for a in (a0, a1):
        assert a.grad is not None and bool(torch.isfinite(a.grad).all()) and float(a.grad.abs().max()) > 0, env_name


def test_bad_dynamics_state_inputs_are_refused():
    import torch
    from diffrl_b200.engine import DynamicsStateFunction
    eng = _engine("AntEnv", "auto", 4)
    Q, D, L = eng.Q, eng.D, eng.L
    q = torch.zeros((4, Q), device="cuda:0")
    q[:, 6] = 1.0
    qd = torch.zeros((4, D), device="cuda:0")
    act = torch.zeros((4, D), device="cuda:0")
    for bad in ((torch.zeros((4, Q + 1), device="cuda:0"), qd, act), (q, torch.zeros((5, D), device="cuda:0"), act),
                (q.double(), qd, act), (q, qd.half(), act), (q.cpu(), qd, act), (q, qd, act.cpu()), (q, qd, None),
                (q, qd, torch.zeros((4, D + 1), device="cuda:0"))):
        with pytest.raises(ValueError):
            eng.dynamics_state(*bad)
        with pytest.raises(ValueError):
            DynamicsStateFunction.apply(eng, *bad, None, None)
    with pytest.raises(ValueError):
        eng.dynamics_state(q, qd, act, None, torch.zeros((4, L, 5), device="cuda:0"))
    with pytest.raises(ValueError):
        eng.dynamics_state_backward(q, qd, act, None, None, torch.zeros((4, D + 1), device="cuda:0"), None, None)
    with pytest.raises(ValueError):
        eng.dynamics_state_backward(q, qd, act, None, None, None, None, torch.zeros((4, D, D), device="cuda:0", dtype=torch.float64))
    snu = _engine("SNUHumanoidEnv", "auto", 2)
    with pytest.raises(ValueError):
        snu.dynamics_state(torch.zeros((2, snu.Q), device="cuda:0"), torch.zeros((2, snu.D), device="cuda:0"),
                           torch.zeros((2, snu.D), device="cuda:0"), None)
    # the ABI: NULL q / qd / act / workspace, NULL musc with muscles, n <= 0 and a NULL pack are cudaErrorInvalidValue (1) without a
    # launch; nothing to compute is 0 without a launch
    lib, P = eng.lib, eng.pack
    out = torch.zeros(4 * D, device="cuda:0")
    gq = torch.zeros(4 * Q, device="cuda:0")
    ws = eng.dynamics_workspace()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    before = lib.dfx_launch_count()
    fwd = (P, 4, p(q), p(qd), p(act), None, None, p(out), None, None, s)
    for k in (0, 2, 3, 4):
        args = list(fwd)
        if k == 0:
            args[0] = None
        else:
            args[k] = None
        assert lib.dfx_dynamics_state_forward(*args) == 1
    for nn in (0, -1):
        assert lib.dfx_dynamics_state_forward(P, nn, *fwd[2:]) == 1
    bwd = (P, 4, p(q), p(qd), p(act), None, None, p(ws), p(out), None, None, p(gq), None, None, None, None, s)
    for k in (0, 2, 3, 4, 7):
        args = list(bwd)
        if k == 0:
            args[0] = None
        else:
            args[k] = None
        assert lib.dfx_dynamics_state_backward(*args) == 1
    sq = torch.zeros(2 * snu.Q, device="cuda:0")
    sd = torch.zeros(2 * snu.D, device="cuda:0")
    assert snu.lib.dfx_dynamics_state_forward(snu.pack, 2, p(sq), p(sd), p(sd), None, None, p(sd), None, None, s) == 1
    assert lib.dfx_dynamics_state_forward(P, 4, p(q), p(qd), p(act), None, None, None, None, None, s) == 0
    assert lib.dfx_dynamics_state_backward(P, 4, p(q), p(qd), p(act), None, None, p(ws), p(out), None, None,
                                           None, None, None, None, None, s) == 0
    assert lib.dfx_launch_count() == before
    assert lib.dfx_dynamics_state_forward(*fwd) == 0
    assert lib.dfx_launch_count() == before + 1
    assert lib.dfx_dynamics_state_backward(*bwd) == 0
    assert lib.dfx_launch_count() == before + 2       # (the tile kernels: one launch)
