"""The link state (include/dfx.h dfx_link_state_forward / _backward) on the kernels.

* the six DiffRL articulations and the random articulations (size twins included) on every kernel family that exists for them
  -- auto, tile8/16/32, group8/16/32 and the generic lane-group instantiation (flag 4) -- at N = 1 and N = 75 (neither a whole
  tile): the forward per environment and block against the fp64 oracle, the adjoint per environment and gradient block against
  the exact gradient, within link_tolerances.link_state_tol (4x the host emulation's error, never below 1e-6);
* on the same family, the one-substep derived dumps of the step agree within that bound (whether bit for bit is printed);
  through the C ABI nothing past environment N - 1 of over-allocated buffers is written; two calls are bitwise equal;
* composition: 4 env-steps of SimStepFunction under the tether wrench k (target - X_sm.p) of each step's input state (from the
  link state), loss on the final link state: gradients of the actions and the start state against the oracle's exact gradient
  of the same rollout (link_tolerances.link_tether_tol), tape and recompute adjoint modes bitwise equal;
* env.link_state() after fused env-steps of the Ant and Humanoid envs, and the refusals (ValueError) of bad inputs."""
import ctypes

import numpy as np
import pytest

import link_util as U
from link_tolerances import link_state_tol, link_tether_tol

pytestmark = pytest.mark.gpu

# tile widths with a kernel for the articulation's sizes (dfx_tile.cu DFX_TILE_MODELS; the twins have their original's sizes)
TILES = {"CartPoleSwingUpEnv": (32,), "AntEnv": (8, 16, 32), "HopperEnv": (32,), "CheetahEnv": (32,), "HumanoidEnv": (8, 16),
         "SNUHumanoidEnv": (8, 16)}


def _tiles(name):
    return TILES.get(name[len("twin_"):] if name.startswith("twin_") else name, ())


CASES = [(name, v) for name in U.MODELS
         for v in ["auto"] + ["tile%d" % e for e in _tiles(name)] + ["group8", "group16", "group32", "generic"]]


def _select(variant):
    """test_gpu_golden._select, plus 'generic': the lane-group kernels of the automatic width on the generic instantiation (flag 4)"""
    from test_gpu_golden import _select as select
    from diffrl_b200 import _capi
    if variant == "generic":
        select("auto")
        _capi.lib().dfx_set_flags(9 | 32 | 4)
    else:
        select(variant)


def _engine(name, variant, n):
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    model, ne = U.model_of(name)
    desc, _ = U.articulation_from_model(model, ne)
    _select(variant)
    try:
        eng = ArticulationEngine(desc, n, "cuda:0")
    finally:
        _select("auto")
    tile = int(_capi.lib().dfx_pack_query(eng.pack, 9))
    if variant.startswith("tile"):
        assert tile == int(variant[4:]), (name, variant, tile)
    elif variant != "auto":
        assert tile == 0, (name, variant, tile)
    return eng


def _t(a):
    import torch
    return None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda:0")


def _run(eng, q, qd, g):
    out = eng.link_state(_t(q), _t(qd))
    gq, gqd = eng.link_state_backward(_t(q), _t(qd), *(_t(x) for x in g))
    return [o.cpu().numpy() for o in out], gq.view(q.shape).cpu().numpy(), gqd.view(qd.shape).cpu().numpy()


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_link_state_matches_oracle(name, variant):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    egq, egqd = U.exact_link_gradients(name, o, q, qd, g)
    tf, tg = link_state_tol(name, "fwd"), link_state_tol(name, "grad")
    worst = {}
    for n in (1, 75):
        eng = _engine(name, variant, n)
        out, gq, gqd = _run(eng, q[:n], qd[:n], tuple(x[:n] for x in g))
        for block, err in U.forward_errors(out, tuple(r[:n] for r in ref)).items():
            assert err.max() <= tf, (name, variant, n, block, int(err.argmax()), float(err.max()), tf)
            worst["fwd"] = max(worst.get("fwd", 0.0), float(err.max()) / tf)
        for block, err in U.grad_errors(desc, gq, gqd, egq[:n], egqd[:n]).items():
            assert err.max() <= tg, (name, variant, n, block, int(err.argmax()), float(err.max()), tg)
            worst["grad"] = max(worst.get("grad", 0.0), float(err.max()) / tg)
    print(name, variant, "worst error / bound", {k: "%.2f" % v for k, v in worst.items()})


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_link_state_dumps_abi_and_determinism(name, variant):
    import torch
    desc, q, qd, g = U.batch(name)
    n = q.shape[0]
    eng = _engine(name, variant, n)
    out, gq, gqd = _run(eng, q, qd, g)
    # the step's derived dumps of a one-substep call on the same family
    act = torch.zeros((n, desc.D), device="cuda:0")
    musc = torch.zeros((n, desc.M), device="cuda:0") if desc.M else None
    _, _, _, dumps = eng.forward(_t(q), _t(qd), act, musc, 1, 1, 1.0 / 960.0, want_tape=False,
                                 derived=["body_X_sc", "body_X_sm", "body_v_s"])
    dumped = [dumps[k].view(n, desc.L, -1).cpu().numpy() for k in ("body_X_sc", "body_X_sm", "body_v_s")]
    tf = link_state_tol(name, "fwd")
    for block, err in U.forward_errors(out, dumped).items():
        assert err.max() <= tf, (name, variant, block, float(err.max()), tf)
    print(name, variant, "link state == one-substep derived dumps bit for bit:", all(np.array_equal(a, b) for a, b in zip(out, dumped)))
    # two calls: bitwise equal
    out2, gq2, gqd2 = _run(eng, q, qd, g)
    assert all(np.array_equal(a, b) for a, b in zip(out, out2)) and np.array_equal(gq, gq2) and np.array_equal(gqd, gqd2)
    # the C ABI with buffers of n + 5 environments, pre-filled: nothing past environment n - 1 is written
    L, Q, D, extra = desc.L, desc.Q, desc.D, 5
    fill = 12345.0
    bufs = [torch.full(((n + extra) * L * w,), fill, device="cuda:0") for w in (7, 7, 6)]
    grads = [torch.full(((n + extra) * w,), fill, device="cuda:0") for w in (Q, D)]
    qt, qdt = _t(q), _t(qd)
    gt = [_t(x) for x in g]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    assert eng.lib.dfx_link_state_forward(eng.pack, n, p(qt), p(qdt), *(p(b) for b in bufs), stream) == 0
    assert eng.lib.dfx_link_state_backward(eng.pack, n, p(qt), p(qdt), *(p(x) for x in gt), *(p(x) for x in grads), stream) == 0
    torch.cuda.synchronize()
    for b, w, ref in zip(bufs, (7, 7, 6), out):
        assert bool((b[n * L * w:] == fill).all()), (name, variant)
        assert np.array_equal(b[:n * L * w].cpu().numpy(), ref.ravel())
    for b, w, ref in zip(grads, (Q, D), (gq, gqd)):
        assert bool((b[n * w:] == fill).all()), (name, variant)
        assert np.array_equal(b[:n * w].cpu().numpy(), ref.ravel())


# ------------------------------------------------------------------ composition with the step
def _tether_grads(eng, q0, qd0, acts, target, g, S, mm, dt):
    import torch
    from diffrl_b200.engine import LinkStateFunction, SimStepFunction
    q = _t(q0).requires_grad_(True)
    qd = _t(qd0).requires_grad_(True)
    a = [_t(x).requires_grad_(True) for x in acts]
    tgt = _t(target)
    qi, qdi = q, qd
    for t in range(len(a)):
        X_sm = LinkStateFunction.apply(eng, qi, qdi)[1]
        f = torch.cat([torch.zeros_like(X_sm[:, :, :3]), U.TETHER_K * (tgt - X_sm[:, :, :3])], dim=2)
        qi, qdi = SimStepFunction.apply(eng, S, mm, dt, qi, qdi, a[t], None, f)
    out = LinkStateFunction.apply(eng, qi, qdi)
    loss = sum((o * _t(x)).sum() for o, x in zip(out, g))
    loss.backward()
    return q.grad, qd.grad, torch.stack([x.grad for x in a])


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv"])
def test_tethered_rollout_gradient_matches_oracle_in_both_adjoint_modes(name):
    import torch
    import diffrl_b200
    from diffrl_b200.engine import ArticulationEngine
    model, meta, q0, qd0, acts = U.tether_case(name, 8)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    desc, _ = U.articulation_from_model(model, meta["num_envs"])
    eng = ArticulationEngine(desc, q0.shape[0], "cuda:0")
    target = U.tether_target(eng.link_state(_t(q0), _t(qd0))[1].cpu().numpy())
    rng = np.random.default_rng(9)
    g = tuple(rng.standard_normal((q0.shape[0], desc.L, w)).astype(np.float32) for w in (7, 7, 6))
    tape = _tether_grads(eng, q0, qd0, acts, target, g, S, mm, dt)
    diffrl_b200.set_adjoint_mode("recompute")
    try:
        rec = _tether_grads(eng, q0, qd0, acts, target, g, S, mm, dt)
    finally:
        diffrl_b200.set_adjoint_mode("tape")
    for a, b in zip(tape, rec):
        assert torch.equal(a, b), name
    o = U.oracle_of(name)
    gq, gqd, gact = (x.cpu().numpy() for x in tape)
    err = U.tether_errors(o, q0, qd0, acts, target, g, gq, gqd, gact, S, mm, dt, envs=range(2))
    print(name, "tethered rollout error / bound", {k: "%.2f" % (v / link_tether_tol(name, k)) for k, v in err.items()})
    for k, v in err.items():
        assert v <= link_tether_tol(name, k), (name, k, v, link_tether_tol(name, k))


# ------------------------------------------------------------------ envs
@pytest.mark.parametrize("env_name", ["AntEnv", "HumanoidEnv"])
def test_env_link_state_after_fused_env_steps(env_name):
    import torch
    import diffrl_b200
    from diffrl_b200 import envs
    env = getattr(envs, env_name)(num_envs=8, device="cuda:0", no_grad=False)
    env.reset()
    acts = [torch.full((env.num_envs, env.num_actions), 0.3 * (k + 1), device="cuda:0", requires_grad=True) for k in range(3)]
    for a in acts:
        env.step(a)
    ls = env.link_state()
    ref = diffrl_b200.link_state(env.model, env.state.joint_q, env.state.joint_qd)
    L = env.model.link_count // env.num_envs
    assert ls.body_X_sc.shape == (env.num_envs, L, 7) and ls.body_v_s.shape == (env.num_envs, L, 6)
    for a, b in zip(ls, ref):
        assert torch.equal(a, b)
    v_com = ls.body_v_s[:, :, 3:] + torch.cross(ls.body_v_s[:, :, :3], ls.body_X_sm[:, :, :3], dim=2)
    loss = ls.body_X_sm[:, :, 1].sum() + (v_com ** 2).sum()
    loss.backward()
    for a in acts:
        assert a.grad is not None and bool(torch.isfinite(a.grad).all()) and float(a.grad.abs().max()) > 0, env_name


def test_bad_link_state_inputs_are_refused():
    import torch
    from diffrl_b200.engine import LinkStateFunction
    eng = _engine("AntEnv", "auto", 4)
    Q, D, L = eng.Q, eng.D, eng.L
    q = torch.zeros((4, Q), device="cuda:0")
    q[:, 6] = 1.0
    qd = torch.zeros((4, D), device="cuda:0")
    for bad_q, bad_qd in ((torch.zeros((4, Q + 1), device="cuda:0"), qd), (q, torch.zeros((5, D), device="cuda:0")),
                          (q.double(), qd), (q, qd.half()), (q.cpu(), qd), (q, qd.cpu()), (q.view(2, 2, Q), qd)):
        with pytest.raises(ValueError):
            eng.link_state(bad_q, bad_qd)
        with pytest.raises(ValueError):
            LinkStateFunction.apply(eng, bad_q, bad_qd)
    with pytest.raises(ValueError):
        eng.link_state_backward(q, qd, torch.zeros((4, L, 6), device="cuda:0"), None, None)
    with pytest.raises(ValueError):
        eng.link_state_backward(q, qd, None, None, torch.zeros((4, L, 6), device="cuda:0", dtype=torch.float64))
    # flat and [N, Q] / [N, D] are both accepted and agree
    a = eng.link_state(q, qd)
    b = eng.link_state(q.view(-1), qd.view(-1))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
