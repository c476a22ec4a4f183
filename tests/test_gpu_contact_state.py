"""The contact state (include/dfx.h dfx_contact_state_forward / _backward) on the kernels.

* the six DiffRL articulations and the random articulations on every kernel family that exists for them -- auto, tile8/16/32,
  group8/16/32 and the generic lane-group instantiation (flag 4), selected for the whole test -- at N = 1 and N = 75 (neither a
  whole tile): the forward per environment and block against the fp64 oracle, the adjoint per environment and gradient block
  against the exact gradient, within contact_tolerances.contact_state_tol.  An environment over its bound is admissible only
  when its oracle result moves comparably under a one-ulp input perturbation (a contact switching surface); such exclusions are
  printed per case;
* on the same family, through the C ABI: the convention check (ground off via dfx_pack_set_gravity, a one-substep env-step under
  f_ext = body_f_contact equals the same env-step with the ground on, contact_tolerances.CONVENTION_BOUND); nothing past
  environment N - 1 of over-allocated buffers is written; two calls are bitwise equal; an environment with a non-finite q leaves
  every other environment's outputs unchanged;
* composition: T = 3 env-steps of SimStepFunction, loss on the final contact state: gradients of the actions and the start state
  against the oracle's exact gradient of the same rollout (contact_tolerances.contact_rollout_tol), tape and recompute adjoint
  modes bitwise equal;
* env.contact_state() after fused env-steps of the Ant and Humanoid envs, and the refusals (ValueError in Python,
  cudaErrorInvalidValue at the ABI)."""
import contextlib
import ctypes

import numpy as np
import pytest

import contact_util as U
from contact_tolerances import CONVENTION_BOUND, contact_rollout_tol, contact_state_tol
from test_contact_state_emu import rollout_cotangents

pytestmark = pytest.mark.gpu

# tile widths with a kernel for the articulation's sizes (dfx_tile.cu DFX_TILE_MODELS; the twins have their original's sizes)
TILES = {"CartPoleSwingUpEnv": (32,), "AntEnv": (8, 16, 32), "HopperEnv": (32,), "CheetahEnv": (32,), "HumanoidEnv": (8, 16),
         "SNUHumanoidEnv": (8, 16)}


def _tiles(name):
    return TILES.get(name[len("twin_"):] if name.startswith("twin_") else name, ())


CASES = [(name, v) for name in U.MODELS
         for v in ["auto"] + ["tile%d" % e for e in _tiles(name)] + ["group8", "group16", "group32", "generic"]]


@contextlib.contextmanager
def _selected(variant):
    """the kernel family `variant` for packs created and launches made inside (the group width and flag 4 are read at launch)"""
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


def _run(eng, q, qd, g):
    out = eng.contact_state(_t(q), _t(qd))
    gq, gqd = eng.contact_state_backward(_t(q), _t(qd), *(_t(x) for x in g))
    return [o.cpu().numpy() for o in out], gq.view(q.shape).cpu().numpy(), gqd.view(qd.shape).cpu().numpy()


def _check(name, variant, o, q, qd, errors, bound, worst, kind, excluded):
    """every environment within `bound`, or on a switching surface (recorded in `excluded`)"""
    for block, err in errors.items():
        for e in np.nonzero(err > bound)[0]:
            assert U.one_ulp_sensitive(o, q, qd, int(e)), (name, variant, kind, block, int(e), float(err[e]), bound)
            excluded.add(int(e))
        ok = np.array([e not in excluded for e in range(len(err))])
        if ok.any():
            worst[kind] = max(worst.get(kind, 0.0), float(err[ok].max()) / bound)


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_contact_state_matches_oracle(name, variant):
    o = U.oracle_of(name)
    desc, q, qd, g = U.batch(name)
    ref = U.reference(name, o, q, qd)
    egq, egqd = U.exact_contact_gradients(name, o, q, qd, g)
    tf, tg = contact_state_tol(name, "fwd"), contact_state_tol(name, "grad")
    worst, excluded = {}, set()
    with _selected(variant):
        for n in (1, 75):
            eng = _engine(name, variant, n)
            out, gq, gqd = _run(eng, q[:n], qd[:n], tuple(x[:n] for x in g))
            _check(name, variant, o, q, qd, U.forward_errors(desc, out, tuple(r[:n] for r in ref)), tf, worst, "fwd", excluded)
            _check(name, variant, o, q, qd, U.grad_errors(desc, gq, gqd, egq[:n], egqd[:n]), tg, worst, "grad", excluded)
    print(name, variant, "worst error / bound", {k: "%.2f" % v for k, v in worst.items()}, "excluded", sorted(excluded))


@pytest.mark.parametrize("name,variant", CASES)
def test_cuda_contact_state_convention_abi_and_determinism(name, variant):
    import torch
    desc, q, qd, g = U.batch(name)
    n, L, C, Q, D = q.shape[0], desc.L, desc.C, desc.Q, desc.D
    with _selected(variant):
        eng = _engine(name, variant, n)
        out, gq, gqd = _run(eng, q, qd, g)
        # two calls: bitwise equal
        out2, gq2, gqd2 = _run(eng, q, qd, g)
        assert all(np.array_equal(a, b) for a, b in zip(out, out2)) and np.array_equal(gq, gq2) and np.array_equal(gqd, gqd2)
        # convention: ground off + f_ext = body_f_contact is the ground (one substep), through dfx_pack_set_gravity and the step
        if C:
            gx, gy, gz = (float(x) for x in desc.gravity)
            act = torch.zeros((n, D), device="cuda:0")
            musc = torch.zeros((n, desc.M), device="cuda:0") if desc.M else None
            dt = 1.0 / 960.0
            _, qd_on, _, _ = eng.forward(_t(q), _t(qd), act, musc, 1, 1, dt, want_tape=False)
            assert eng.lib.dfx_pack_set_gravity(eng.pack, gx, gy, gz, 0) == 0
            try:
                _, qd_ext, _, _ = eng.forward(_t(q), _t(qd), act, musc, 1, 1, dt, want_tape=False, f_ext=_t(out[2]))
                _, qd_off, _, _ = eng.forward(_t(q), _t(qd), act, musc, 1, 1, dt, want_tape=False)
                off = eng.contact_state(_t(q), _t(qd))
            finally:
                eng.lib.dfx_pack_set_gravity(eng.pack, gx, gy, gz, 1)
            assert not off[0].any() and not off[2].any() and torch.equal(off[1].cpu(), torch.tensor(out[1]))
            qd_on, qd_ext, qd_off = (x.view(n, D).cpu().numpy() for x in (qd_on, qd_ext, qd_off))
            err = U.convention_errors(qd_on, qd_ext, qd_off)
            assert (err > 0).any() and err.max() <= CONVENTION_BOUND, (name, variant, int(err.argmax()), float(err.max()))
            print(name, variant, "convention error / bound %.2f" % (err.max() / CONVENTION_BOUND),
                  "non-finite env-steps", int((~np.isfinite(qd_on).all(axis=1)).sum()))
        # the C ABI with buffers of n + 5 environments, pre-filled: nothing past environment n - 1 is written
        extra, fill = 5, 12345.0
        widths = (C * 3, C, L * 6)
        bufs = [torch.full(((n + extra) * w + 1,), fill, device="cuda:0") for w in widths]
        grads = [torch.full(((n + extra) * w,), fill, device="cuda:0") for w in (Q, D)]
        qt, qdt = _t(q), _t(qd)
        gt = [_t(x) for x in g]
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        assert eng.lib.dfx_contact_state_forward(eng.pack, n, p(qt), p(qdt), *(p(b) for b in bufs), stream) == 0
        assert eng.lib.dfx_contact_state_backward(eng.pack, n, p(qt), p(qdt), *(p(x) for x in gt), *(p(x) for x in grads), stream) == 0
        torch.cuda.synchronize()
        for b, w, r in zip(bufs, widths, out):
            assert bool((b[n * w:] == fill).all()), (name, variant)
            assert np.array_equal(b[:n * w].cpu().numpy(), r.ravel())
        for b, w, r in zip(grads, (Q, D), (gq, gqd)):
            assert bool((b[n * w:] == fill).all()), (name, variant)
            assert np.array_equal(b[:n * w].cpu().numpy(), r.ravel())
        # a non-finite q in one environment leaves the others (of its tile and every other) as they were
        bad = 3
        qb = q.copy()
        qb[bad, 0] = np.nan
        outb, gqb, gqdb = _run(eng, qb, qd, g)
        keep = np.arange(n) != bad
        for a, b in zip(out, outb):
            assert np.array_equal(a[keep], b[keep]), (name, variant)
        assert np.array_equal(gq[keep], gqb[keep]) and np.array_equal(gqd[keep], gqdb[keep]), (name, variant)


def test_no_contacts_give_zero_wrenches_and_gradients():
    import torch
    for name in ("CartPoleSwingUpEnv", "gen_fixed"):
        desc, q, qd, g = U.batch(name)
        eng = _engine(name, "auto", q.shape[0])
        f, h, w = eng.contact_state(_t(q), _t(qd))
        assert f.shape == (q.shape[0], 0, 3) and h.shape == (q.shape[0], 0) and not bool(w.any())
        gq, gqd = eng.contact_state_backward(_t(q), _t(qd), None, None, torch.ones_like(w))
        assert not bool(gq.any()) and not bool(gqd.any())


# ------------------------------------------------------------------ composition with the step
def _rollout_grads(eng, q0, qd0, acts, g, S, mm, dt):
    import torch
    from diffrl_b200.engine import ContactStateFunction, SimStepFunction
    q = _t(q0).requires_grad_(True)
    qd = _t(qd0).requires_grad_(True)
    a = [_t(x).requires_grad_(True) for x in acts]
    qi, qdi = q, qd
    for t in range(len(a)):
        qi, qdi = SimStepFunction.apply(eng, S, mm, dt, qi, qdi, a[t], None)
    out = ContactStateFunction.apply(eng, qi, qdi)
    loss = sum((o * _t(x)).sum() for o, x in zip(out, g))
    loss.backward()
    return q.grad, qd.grad, torch.stack([x.grad for x in a])


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv"])
def test_contact_rollout_gradient_matches_oracle_in_both_adjoint_modes(name):
    import torch
    import diffrl_b200
    from diffrl_b200.engine import ArticulationEngine
    model, meta, q0, qd0, acts = U.rollout_case(name, 8)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    desc, _ = U.articulation_from_model(model, meta["num_envs"])
    eng = ArticulationEngine(desc, q0.shape[0], "cuda:0")
    g = rollout_cotangents(desc, q0.shape[0])
    tape = _rollout_grads(eng, q0, qd0, acts, g, S, mm, dt)
    diffrl_b200.set_adjoint_mode("recompute")
    try:
        rec = _rollout_grads(eng, q0, qd0, acts, g, S, mm, dt)
    finally:
        diffrl_b200.set_adjoint_mode("tape")
    for a, b in zip(tape, rec):
        assert torch.equal(a, b), name
    o = U.oracle_of(name)
    gq, gqd, gact = (x.cpu().numpy() for x in tape)
    err = U.rollout_errors(o, q0, qd0, acts, g, gq, gqd, gact, S, mm, dt, envs=range(2))
    print(name, "contact rollout error / bound", {k: "%.2f" % (v / contact_rollout_tol(name, k)) for k, v in err.items()})
    for k, v in err.items():
        assert v <= contact_rollout_tol(name, k), (name, k, v, contact_rollout_tol(name, k))


# ------------------------------------------------------------------ envs
@pytest.mark.parametrize("env_name", ["AntEnv", "HumanoidEnv"])
def test_env_contact_state_after_fused_env_steps(env_name):
    import torch
    import diffrl_b200
    from diffrl_b200 import envs
    env = getattr(envs, env_name)(num_envs=8, device="cuda:0", no_grad=False)
    env.reset()
    acts = [torch.full((env.num_envs, env.num_actions), 0.3 * (k + 1), device="cuda:0", requires_grad=True) for k in range(3)]
    for a in acts:
        env.step(a)
    cs = env.contact_state()
    ref = diffrl_b200.contact_state(env.model, env.state.joint_q, env.state.joint_qd)
    L = env.model.link_count // env.num_envs
    C = env.model.contact_count // env.num_envs
    assert cs.contact_f.shape == (env.num_envs, C, 3) and cs.contact_height.shape == (env.num_envs, C)
    assert cs.body_f_contact.shape == (env.num_envs, L, 6)
    for a, b in zip(cs, ref):
        assert torch.equal(a, b)
    # the force is upward where a point penetrates, and zero where it does not
    pen = cs.contact_height < 0
    assert bool((cs.contact_f[..., 1][pen] >= 0).all()) and not bool(cs.contact_f[~pen].any())
    loss = cs.body_f_contact[:, :, 4].sum() + (cs.contact_height ** 2).sum()
    loss.backward()
    for a in acts:
        assert a.grad is not None and bool(torch.isfinite(a.grad).all()) and float(a.grad.abs().max()) > 0, env_name


def test_bad_contact_state_inputs_are_refused():
    import torch
    from diffrl_b200.engine import ContactStateFunction
    eng = _engine("AntEnv", "auto", 4)
    Q, D, L, C = eng.Q, eng.D, eng.L, eng.C
    q = torch.zeros((4, Q), device="cuda:0")
    q[:, 6] = 1.0
    qd = torch.zeros((4, D), device="cuda:0")
    for bad_q, bad_qd in ((torch.zeros((4, Q + 1), device="cuda:0"), qd), (q, torch.zeros((5, D), device="cuda:0")),
                          (q.double(), qd), (q, qd.half()), (q.cpu(), qd), (q, qd.cpu()), (q.view(2, 2, Q), qd)):
        with pytest.raises(ValueError):
            eng.contact_state(bad_q, bad_qd)
        with pytest.raises(ValueError):
            ContactStateFunction.apply(eng, bad_q, bad_qd)
    with pytest.raises(ValueError):
        eng.contact_state_backward(q, qd, torch.zeros((4, C, 2), device="cuda:0"), None, None)
    with pytest.raises(ValueError):
        eng.contact_state_backward(q, qd, None, torch.zeros((4, C), device="cuda:0", dtype=torch.float64), None)
    with pytest.raises(ValueError):
        eng.contact_state_backward(q, qd, None, None, torch.zeros((4, L, 7), device="cuda:0"))
    # flat and [N, Q] / [N, D] are both accepted and agree
    a = eng.contact_state(q, qd)
    b = eng.contact_state(q.view(-1), qd.view(-1))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # the ABI: NULL q / qd, n <= 0 and a NULL pack are cudaErrorInvalidValue (1), without a launch; nothing to compute is 0
    lib, P = eng.lib, eng.pack
    out = torch.zeros(4 * L * 6, device="cuda:0")
    gq = torch.zeros(4 * Q, device="cuda:0")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    before = lib.dfx_launch_count()
    for args in ((P, 4, None, p(qd), None, None, p(out), s), (P, 4, p(q), None, None, None, p(out), s), (P, 0, p(q), p(qd), None, None, p(out), s),
                 (P, -1, p(q), p(qd), None, None, p(out), s), (None, 4, p(q), p(qd), None, None, p(out), s)):
        assert lib.dfx_contact_state_forward(*args) == 1
    for args in ((P, 4, None, p(qd), None, None, None, p(gq), None, s), (P, 0, p(q), p(qd), None, None, None, p(gq), None, s),
                 (None, 4, p(q), p(qd), None, None, None, p(gq), None, s)):
        assert lib.dfx_contact_state_backward(*args) == 1
    assert lib.dfx_contact_state_forward(P, 4, p(q), p(qd), None, None, None, s) == 0
    assert lib.dfx_contact_state_backward(P, 4, p(q), p(qd), None, None, None, None, None, s) == 0
    assert lib.dfx_launch_count() == before
    assert lib.dfx_contact_state_forward(P, 4, p(q), p(qd), None, None, p(out), s) == 0
    assert lib.dfx_launch_count() == before + 1
