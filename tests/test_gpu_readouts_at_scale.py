"""The four state readouts -- link, contact, dynamics and Jacobian state (include/dfx.h dfx_*_state_forward / _backward) -- where a
training run uses them: at the batch sizes of BASELINE.json, on packs with a bf16 tape, on buffers that hold garbage, and on
side streams and inside CUDA graphs.  Every comparison below is bit for bit, except the one against the fp64 oracles.

* at size: Ant 65536 + 37, Humanoid 8192 + 5 and SNU 4096 + 11 environments (the last tile partial; lane groups of 32 for Ant
  at 8192 + 37) that repeat a 64-environment pattern give every environment the outputs and gradients of its pattern
  environment in a 64-environment run.  64 environments fill whole tiles of 8, 16 and 32, so every lane repeats its computation;
* at size with independent per-environment inputs: a spread sample of about 48 environments (the first and last of the batch
  and of several tiles, the whole partial tile) against the fp64 oracles and exact gradients, within each op's bounds.  An
  environment over a bound is admitted only when the oracle's own result moves comparably under 1-4 ulp input perturbations
  (parity_util's conditioning rule); the worst error over its bound and every admitted environment are printed;
* a pack created after set_tape_dtype("bf16") gives the outputs and gradients of one created after "fp32", on every tile
  width of every DiffRL articulation (the dynamics backward re-runs an env-step into its workspace with fp32 rows whatever the
  tape dtype), and so does DFlexEnv.dynamics_state(actions);
* through the C ABI, results do not depend on what the output, gradient and workspace buffers held before (0, NaN, 1e30), and
  NaN inputs and cotangents of one environment -- first, middle or last of a CTA, or in the partial CTA -- leave every other
  environment's outputs and gradients unchanged;
* the autograd Functions on a side stream whose inputs a kernel of that stream has just written equal the default-stream run,
  and a CUDA graph of one SimStepFunction env-step, a loss on all four readouts of its end state and backward() (the dynamics
  backward allocating its workspace during capture) replays to the eager results on two input sets."""
import ctypes

import numpy as np
import pytest

import contact_util as CU
import dynamics_util as DU
import jacobian_util as JU
import link_util as LU
from contact_tolerances import contact_state_tol
from dynamics_tolerances import dynamics_tol
from jacobian_tolerances import jacobian_state_tol
from link_tolerances import link_state_tol
from parity_util import _probes
from test_gpu_dynamics_state import _step_ok
from test_gpu_jacobian_state import _engine, _selected
from test_gpu_link_state import TILES

pytestmark = pytest.mark.gpu

AT_SIZE = {"AntEnv": 65536 + 37, "HumanoidEnv": 8192 + 5, "SNUHumanoidEnv": 4096 + 11}
PATTERN = 64


# ------------------------------------------------------------------ inputs and the runner
def _inputs(name, n, seed=3):
    """(desc, numpy inputs of the four readouts for n environments): contact_util.batch's states (link_util.batch's -- every regime
    row, quaternions off the unit sphere -- with every fifth environment at rest), dynamics_util.batch's actuation, muscle
    activations and wrench, and each op's cotangents from its own batch builder"""
    desc, q, qd, g_contact = CU.batch(name, n, seed)
    _, dyn, g_dyn = DU.batch(name, n, seed)
    return desc, dict(q=q, qd=qd, act=dyn["act"], musc=dyn["musc"], f_ext=dyn["f_ext"], g_link=LU.batch(name, n, seed)[3],
                      g_contact=g_contact, g_jac=JU.batch(name, n, seed)[3], g_dyn=g_dyn)


def _map(x, f):
    return {k: tuple(f(a) for a in v) if isinstance(v, tuple) else f(v) for k, v in x.items()}


def _gpu(x):
    import torch
    return _map(x, lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda:0"))


def _tiled(x, n):
    """the environments of x repeated to n"""
    def rep(a):
        if a is None:
            return None
        return a.repeat((-(-n // a.shape[0]),) + (1,) * (a.dim() - 1))[:n].contiguous()
    return _map(x, rep)


def _run(eng, x, fill=None):
    """{name: [n, w] tensor}: every output and every gradient of the four readouts (the dynamics state with the wrench, "dyn", and
    without, "dyn0") through the C ABI on the current stream.  The output, gradient and workspace buffers are filled with `fill`
    first (None: as the caching allocator hands them out)."""
    import torch
    n, L, C, Q, D, M = eng.N, eng.L, eng.C, eng.Q, eng.D, eng.M
    lib, P = eng.lib, eng.pack
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())

    def buf(w, rows=n):
        t = torch.empty((rows, w), dtype=torch.float32, device="cuda:0")
        return t if fill is None else t.fill_(fill)

    def call(what, code):
        assert code == 0, (what, code)

    q, qd = x["q"], x["qd"]
    res = {}
    out, g = [buf(L * 7), buf(L * 7), buf(L * 6)], [buf(Q), buf(D)]
    call("link fwd", lib.dfx_link_state_forward(P, n, p(q), p(qd), *map(p, out), s))
    call("link bwd", lib.dfx_link_state_backward(P, n, p(q), p(qd), *map(p, x["g_link"]), *map(p, g), s))
    res.update(zip(("link.X_sc", "link.X_sm", "link.v_s", "link.gq", "link.gqd"), out + g))
    out, g = [buf(C * 3), buf(C), buf(L * 6)], [buf(Q), buf(D)]
    call("contact fwd", lib.dfx_contact_state_forward(P, n, p(q), p(qd), *map(p, out), s))
    call("contact bwd", lib.dfx_contact_state_backward(P, n, p(q), p(qd), *map(p, x["g_contact"]), *map(p, g), s))
    res.update(zip(("contact.f", "contact.height", "contact.body", "contact.gq", "contact.gqd"), out + g))
    out, g = [buf(L * 6 * D), buf(L * 6)], [buf(Q), buf(D)]
    call("jacobian fwd", lib.dfx_jacobian_state_forward(P, n, p(q), p(qd), *map(p, out), s))
    call("jacobian bwd", lib.dfx_jacobian_state_backward(P, n, p(q), p(qd), *map(p, x["g_jac"]), *map(p, g), s))
    res.update(zip(("jac.J", "jac.a_s", "jac.gq", "jac.gqd"), out + g))
    for tag, f_ext in (("dyn", x["f_ext"]), ("dyn0", None)):
        ins = (q, qd, x["act"], x["musc"], f_ext)
        out = [buf(D), buf(D), buf(D * D)]
        call(tag + " fwd", lib.dfx_dynamics_state_forward(P, n, *map(p, ins), *map(p, out), s))
        ws = buf(int(lib.dfx_dynamics_workspace_floats(P, n)), rows=1)
        g = [buf(Q), buf(D), buf(D), buf(M) if M else None, buf(L * 6) if f_ext is not None else None]
        call(tag + " bwd", lib.dfx_dynamics_state_backward(P, n, *map(p, ins), p(ws), *map(p, x["g_dyn"]), *map(p, g), s))
        res.update((tag + "." + k, v) for k, v in zip(("qdd", "tau", "H", "gq", "gqd", "gact", "gmusc", "g_f_ext"), out + g)
                   if v is not None)
    return res


def _differing(a, b):
    """the rows (environments) of two [n, w] tensors that differ in any bit"""
    import torch
    return (a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).any(dim=1).nonzero().flatten().tolist()


def _assert_same(got, ref, what, skip=None):
    """bitwise equality of two _run results, per environment; `skip`: an environment exempt"""
    assert got.keys() == ref.keys(), (what, sorted(got), sorted(ref))
    for k in ref:
        bad = [e for e in _differing(got[k], ref[k]) if e != skip]
        assert not bad, (what, k, "environments", bad[:8], len(bad))


# ------------------------------------------------------------------ 1. every environment at size, through repeated patterns
@pytest.mark.parametrize("name,variant,n", [(name, "auto", n) for name, n in AT_SIZE.items()] + [("AntEnv", "group32", 8192 + 37)])
def test_every_environment_at_size_equals_its_pattern_environment(name, variant, n):
    import torch
    _, x = _inputs(name, PATTERN, seed=11)
    x = _gpu(x)
    with _selected(variant):
        ref = _run(_engine(name, variant, PATTERN), x)
        got = _run(_engine(name, variant, n), _tiled(x, n))
    torch.cuda.synchronize()
    pattern = torch.arange(n, device="cuda:0") % PATTERN
    assert got.keys() == ref.keys()
    for k in ref:
        bad = _differing(got[k], ref[k][pattern])
        assert not bad, (name, variant, n, k, "environments", bad[:8], len(bad))
    print(name, variant, n, "environments: every output and gradient of the four readouts equals its pattern environment's")


# ------------------------------------------------------------------ 2. a sample against the fp64 oracles at size
def _sample(n, E, k=48):
    """the first and last environment of the batch and of its first, second, middle and last whole tile of E, every environment
    of the partial tile, and a spread over the rest: about k environments"""
    full = n // E
    picked = [t * E + o for t in (0, 1, full // 2, full - 1) for o in (0, E - 1)] + list(range(full * E, n)) + [n - 1]
    spread = np.linspace(0, n - 1, max(2, k - len(set(picked)))).round().astype(np.int64)
    return np.unique(np.concatenate([picked, spread]).astype(np.int64))


def _ops(name, desc, x):
    """per readout: (oracle forward of (q, qd, env), forward error measure, bound of a forward block, oracle exact gradient of
    (q, qd, env), gradient error measure, bound of a gradient block, output keys, gradient keys) -- the measures and bounds of
    tests/test_gpu_{link,contact,dynamics,jacobian}_state.py"""
    ol, oc, oj, od = LU.oracle_of(name), CU.oracle_of(name), JU.oracle_of(name), DU.oracle_of(name)
    gl, gc, gj, gd = x["g_link"], x["g_contact"], x["g_jac"], x["g_dyn"]
    row = lambda a, e: None if a is None else a[e]
    dyn_in = lambda e: (x["act"][e:e + 1], row(x["musc"], slice(e, e + 1)), row(x["f_ext"], slice(e, e + 1)))
    return {
        "link": (lambda q, qd, e: ol.link_state(q, qd), LU.forward_errors, lambda b: link_state_tol(name, "fwd"),
                 lambda q, qd, e: ol.link_state_gradient(q, qd, gl[0][e], gl[1][e], gl[2][e]),
                 lambda got, ex: LU.grad_errors(desc, *got, *ex), lambda b: link_state_tol(name, "grad"),
                 ("link.X_sc", "link.X_sm", "link.v_s"), ("link.gq", "link.gqd")),
        "contact": (lambda q, qd, e: oc.contact_state(q, qd), lambda got, ref: CU.forward_errors(desc, got, ref),
                    lambda b: contact_state_tol(name, "fwd"),
                    lambda q, qd, e: oc.contact_state_gradient(q, qd, gc[0][e], gc[1][e], gc[2][e]),
                    lambda got, ex: CU.grad_errors(desc, *got, *ex), lambda b: contact_state_tol(name, "grad"),
                    ("contact.f", "contact.height", "contact.body"), ("contact.gq", "contact.gqd")),
        "jacobian": (lambda q, qd, e: oj.jacobian_state(q, qd), JU.forward_errors, lambda b: jacobian_state_tol(name, "fwd"),
                     lambda q, qd, e: oj.jacobian_state_gradient(q, qd, gj[0][e], gj[1][e]),
                     lambda got, ex: JU.grad_errors(desc, *got, *ex), lambda b: jacobian_state_tol(name, "grad"),
                     ("jac.J", "jac.a_s"), ("jac.gq", "jac.gqd")),
        "dynamics": (lambda q, qd, e: od.dynamics_state(q, qd, *dyn_in(e)), DU.forward_errors, lambda b: dynamics_tol(name, b),
                     lambda q, qd, e: od.dynamics_state_gradient(q, qd, x["act"][e], row(x["musc"], e), row(x["f_ext"], e),
                                                                 gd[0][e], gd[1][e], gd[2][e]),
                     DU.grad_errors, lambda b: dynamics_tol(name, b),
                     ("dyn.qdd", "dyn.tau", "dyn.H"), ("dyn.gq", "dyn.gqd", "dyn.gact", "dyn.gmusc", "dyn.g_f_ext")),
    }


def _stack(rows):
    return [None if rows[0][k] is None else np.stack([np.asarray(r[k]) for r in rows]) for k in range(len(rows[0]))]


def _movement(kind, oracle, measure, base, q_row, qd_row, e):
    """the largest change, in the error measure, of the oracle's result for environment e under parity_util's 1-4 ulp
    perturbations of its (q, qd)"""
    moved = 0.0
    for pq, pqd in _probes(q_row, qd_row):
        if kind == "fwd":
            probe = list(oracle(pq[None], pqd[None], e))
        else:
            probe = [None if a is None else np.asarray(a)[None] for a in oracle(pq, pqd, e)]
        moved = max(moved, max(float(v.max()) for v in measure(probe, base).values()))
    return moved


@pytest.mark.parametrize("name", list(AT_SIZE))
def test_sampled_environments_at_size_match_the_fp64_oracles(name):
    import torch
    n = AT_SIZE[name]
    desc, x = _inputs(name, n, seed=7)
    eng = _engine(name, "auto", n)
    E = int(eng.lib.dfx_pack_query(eng.pack, 9))
    assert E, (name, "the default family of the named sizes is a tile kernel")
    idx = _sample(n, E)
    got = _run(eng, _gpu(x))
    ok = _step_ok(eng, {k: x[k] for k in ("q", "qd", "act", "musc", "f_ext")})[idx]
    at = torch.tensor(idx, device="cuda:0")
    got = {k: v[at].cpu().numpy() for k, v in got.items()}
    shapes = {"link.X_sc": (desc.L, 7), "link.X_sm": (desc.L, 7), "link.v_s": (desc.L, 6), "contact.f": (desc.C, 3),
              "contact.height": (desc.C,), "contact.body": (desc.L, 6), "jac.J": (desc.L, 6, desc.D), "jac.a_s": (desc.L, 6),
              "dyn.H": (desc.D, desc.D)}
    got = {k: v.reshape((len(idx),) + shapes.get(k, (-1,))) for k, v in got.items()}
    worst, admitted = _check_sample(name, desc, x, idx, got, ok)
    print(name, "auto", n, "environments,", len(idx), "sampled: worst error / bound", {k: "%.2f" % v for k, v in worst.items()},
          "non-finite env-steps skipped", int((~ok).sum()))
    print(name, "admitted by the conditioning rule:", admitted or "none")


def _check_sample(name, desc, x, idx, got, ok):
    """got: {key: [len(idx), ...]} results of the sampled environments idx of the inputs x; ok: [len(idx)] whether their one-substep
    env-step is finite (the dynamics state skips the others).  Asserts every sampled environment within each op's bound or admitted
    by the conditioning rule; returns ({op.kind: worst error / bound of the environments within}, [admitted, with the reason])."""
    q, qd = x["q"], x["qd"]
    worst, admitted = {}, []
    for op, (fwd, fwd_err, fwd_tol, grad, grad_err, grad_tol, out_keys, grad_keys) in _ops(name, desc, x).items():
        keep = ok if op == "dynamics" else np.ones(len(idx), bool)       # (environments whose one-substep env-step is non-finite)
        refs = [fwd(q[e:e + 1], qd[e:e + 1], e) for e in idx]
        ref = [np.concatenate([r[k] for r in refs]) for k in range(len(out_keys))]
        exact = _stack([grad(q[e], qd[e], e) for e in idx])
        if op == "contact":
            pen = float((ref[1] < 0).mean())
            assert pen >= 0.05, (name, "share of sampled contact points that penetrate", pen)
            print(name, "sampled contact points in penetration: %.1f %%" % (100 * pen))
        checks = (("fwd", fwd_err([got[k] for k in out_keys], ref), fwd_tol, fwd, fwd_err, ref),
                  ("grad", grad_err([got.get(k) for k in grad_keys], exact), grad_tol, grad, grad_err, exact))
        for kind, errors, tol, oracle, measure, expected in checks:
            for block, err in errors.items():
                b = tol(block)
                for j in np.nonzero(keep & (err > b))[0]:
                    # the conditioning rule: the oracle's own result moves comparably under rounding-sized input changes
                    e = int(idx[j])
                    base = [None if r is None else r[j:j + 1] for r in expected]
                    moved = _movement(kind, oracle, measure, base, q[e], qd[e], e)
                    assert err[j] <= max(b, 8.0 * moved), (name, op, kind, block, "env %d: error %.2e, bound %.2e, one-ulp movement of "
                                                           "the oracle %.2e" % (e, err[j], b, moved))
                    admitted.append("%s %s %s env %d: error / bound %.2f, oracle moves %.1e under 1-4 ulp" % (op, kind, block, e,
                                                                                                          err[j] / b, moved))
                within = keep & (err <= b)
                if within.any():
                    worst[op + "." + kind] = max(worst.get(op + "." + kind, 0.0), float(err[within].max()) / b)
    return worst, admitted


# ------------------------------------------------------------------ 3. bf16-tape packs
@pytest.mark.parametrize("name,variant", [(name, "tile%d" % e) for name in LU.DIFFRL for e in TILES[name]])
def test_readouts_are_bitwise_equal_on_bf16_and_fp32_tape_packs(name, variant):
    import diffrl_b200
    _, x = _inputs(name, 75)
    x = _gpu(x)
    engs = {}
    with _selected(variant):
        try:
            for dtype in ("bf16", "fp32"):
                diffrl_b200.set_tape_dtype(dtype)
                engs[dtype] = _engine(name, variant, 75)
        finally:
            diffrl_b200.set_tape_dtype("fp32")
        assert engs["bf16"].tape_bf16 and not engs["fp32"].tape_bf16, (name, variant)
        _assert_same(_run(engs["bf16"], x), _run(engs["fp32"], x), (name, variant, "bf16 tape vs fp32 tape"))


@pytest.mark.parametrize("env_name", ["AntEnv", "HumanoidEnv", "SNUHumanoidEnv"])
def test_env_dynamics_state_is_bitwise_equal_on_bf16_and_fp32_tape_packs(env_name):
    import torch
    import diffrl_b200
    from diffrl_b200 import envs
    from diffrl_b200.dflex_api.sim import _engine_for
    res, start = {}, None
    for dtype in ("bf16", "fp32"):
        diffrl_b200.set_tape_dtype(dtype)
        try:
            env = getattr(envs, env_name)(num_envs=8, device="cuda:0", no_grad=False)
            env.reset()
            if start is None:           # (both packs start from the same state, cut from the graph of the first env)
                start = tuple(t.detach() for t in env.get_state())
            env.reset_with_state(*start)
            gen = torch.Generator().manual_seed(5)
            a = (1.5 * torch.randn((env.num_envs, env.num_actions), generator=gen)).to("cuda:0").requires_grad_(True)
            ds = env.dynamics_state(a)
            w = [torch.randn(t.shape, generator=gen).to("cuda:0") for t in ds]
            sum((t * wt).sum() for t, wt in zip(ds, w)).backward()
            assert _engine_for(env.model).tape_bf16 == (dtype == "bf16"), (env_name, dtype)
            res[dtype] = [t.detach().clone() for t in ds] + [a.grad.clone()]
        finally:
            diffrl_b200.set_tape_dtype("fp32")
    for name, u, v in zip(("joint_qdd", "joint_tau", "H", "actions.grad"), res["bf16"], res["fp32"]):
        assert not _differing(u.view(u.shape[0], -1), v.view(v.shape[0], -1)), (env_name, name)


# ------------------------------------------------------------------ 4. poisoned buffers and environment isolation
def _cta_envs(eng, n):
    """environments to poison: for the forward's and the backward's CTA size E, the first, a middle and the last environment of
    the second CTA (of the first when there is no second), and one in the partial CTA"""
    ks = set()
    for bwd in (0, 1):
        plan = (ctypes.c_int * 6)()
        assert eng.lib.dfx_launch_plan(eng.pack, bwd, plan) == 0
        E = int(plan[1])
        c = E if n >= 2 * E else 0
        ks |= {c, c + E // 2, c + E - 1}
        if n % E:
            ks.add(n - (n % E) // 2 - 1)
    return sorted(k for k in ks if k < n)


def _poisoned(x, k):
    """x with environment k's state, actuation, muscle activations, wrench and every cotangent NaN"""
    def nan_row(a):
        if a is None:
            return None
        a = a.clone()
        a[k] = float("nan")
        return a
    return _map(x, nan_row)


@pytest.mark.parametrize("variant", ["auto", "group16"])
@pytest.mark.parametrize("name,n", [("AntEnv", 75), ("HumanoidEnv", 75), ("SNUHumanoidEnv", 75), ("HumanoidEnv", AT_SIZE["HumanoidEnv"])])
def test_readouts_ignore_prior_buffer_contents_and_keep_environments_apart(name, n, variant):
    _, x = _inputs(name, n)
    x = _gpu(x)
    with _selected(variant):
        eng = _engine(name, variant, n)
        ref = _run(eng, x, fill=0.0)
        for fill in (float("nan"), 1e30):
            _assert_same(_run(eng, x, fill=fill), ref, (name, variant, n, "buffers pre-filled with", fill))
        ks = _cta_envs(eng, n)
        for k in ks:
            got = _run(eng, _poisoned(x, k))
            assert bool(got["link.X_sc"][k].isnan().any()), (name, variant, k, "the poisoned environment's pose is not NaN")
            _assert_same(got, ref, (name, variant, n, "NaN inputs and cotangents in environment", k), skip=k)
    print(name, variant, n, "environments: results independent of prior buffer contents; NaN environments", ks, "stay isolated")


# ------------------------------------------------------------------ 5. streams and CUDA graphs
def _autograd(eng, x):
    """{name: [n, w]}: the outputs of the four readouts' autograd Functions and the gradients torch.autograd.grad takes through
    them under x's cotangents (the dynamics state with the wrench)"""
    import torch
    from diffrl_b200.engine import ContactStateFunction, DynamicsStateFunction, JacobianStateFunction, LinkStateFunction
    n = eng.N
    ins = {k: x[k].detach().clone().requires_grad_(True) for k in ("q", "qd", "act", "musc", "f_ext") if x[k] is not None}
    q, qd = ins["q"], ins["qd"]
    res = {}
    calls = (("link", LinkStateFunction.apply(eng, q, qd), x["g_link"], (q, qd)),
             ("contact", ContactStateFunction.apply(eng, q, qd), x["g_contact"], (q, qd)),
             ("jac", JacobianStateFunction.apply(eng, q, qd), x["g_jac"], (q, qd)),
             ("dyn", DynamicsStateFunction.apply(eng, q, qd, ins["act"], ins.get("musc"), ins["f_ext"]), x["g_dyn"],
              tuple(ins.values())))
    for tag, outs, cot, wrt in calls:
        used = [(o, g) for o, g in zip(outs, cot) if o.numel()]
        grads = torch.autograd.grad([o for o, _ in used], wrt, [g.view(o.shape) for o, g in used])
        res.update(("%s.out%d" % (tag, i), o.detach().reshape(n, -1)) for i, o in enumerate(outs))
        res.update(("%s.grad%d" % (tag, i), g.reshape(n, -1)) for i, g in enumerate(grads))
    return res


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv", "SNUHumanoidEnv"])
def test_autograd_functions_on_a_side_stream_equal_the_default_stream(name):
    import torch
    _, x = _inputs(name, 75)
    x = _gpu(x)
    eng = _engine(name, "auto", 75)
    ref = _autograd(eng, x)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)         # holds the side stream: work misplaced on another stream would run before its inputs
        xs = _map(x, lambda a: None if a is None else torch.full_like(a, float("nan")).copy_(a))
        got = _autograd(eng, xs)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    _assert_same(got, ref, (name, "side stream vs default stream"))


def _graph_case(name, seed):
    """(engine, (S, mm, dt), inputs): golden states of the model, actions scaled per environment, weights of the loss"""
    import wrench_util as W
    model, meta, inp = W.golden_batch(name, 16)
    rng = np.random.default_rng(seed)
    desc, _ = LU.articulation_from_model(model, meta["num_envs"])
    n = inp["q0"].shape[0]
    qd = (inp["qd0"] * rng.uniform(0.8, 1.2, (n, 1))).astype(np.float32)
    act = (inp["act"] * rng.uniform(0.5, 1.5, inp["act"].shape)).astype(np.float32)
    return desc, (meta["S"], meta["mm"], meta["dt"]), dict(q=inp["q0"], qd=qd, act=act)


def _graph_loss(eng, cfg, q, qd, act, w):
    """one env-step, then sum(w . output) over every output of the four readouts of its end state; returns (loss, outputs)"""
    from diffrl_b200.engine import ContactStateFunction, DynamicsStateFunction, JacobianStateFunction, LinkStateFunction, SimStepFunction
    S, mm, dt = cfg
    q1, qd1 = SimStepFunction.apply(eng, S, mm, dt, q, qd, act, None)
    outs = (LinkStateFunction.apply(eng, q1, qd1) + ContactStateFunction.apply(eng, q1, qd1) + JacobianStateFunction.apply(eng, q1, qd1)
            + DynamicsStateFunction.apply(eng, q1, qd1, act, None, None))
    return sum((o * wo).sum() for o, wo in zip(outs, w)), outs


@pytest.mark.parametrize("name", ["AntEnv", "HumanoidEnv"])
def test_cuda_graph_of_a_step_and_readout_loss_replays_the_eager_results(name):
    import torch
    from diffrl_b200.engine import ArticulationEngine
    desc, cfg, x0 = _graph_case(name, 1)
    _, _, x1 = _graph_case(name, 2)
    n = x0["q"].shape[0]
    eng = ArticulationEngine(desc, n, "cuda:0")
    gen = torch.Generator().manual_seed(3)
    shapes = [(n, desc.L, 7), (n, desc.L, 7), (n, desc.L, 6), (n, desc.C, 3), (n, desc.C), (n, desc.L, 6), (n, desc.L, 6, desc.D),
              (n, desc.L, 6), (n, desc.D), (n, desc.D), (n, desc.D, desc.D)]
    w = [torch.randn(s, generator=gen).to("cuda:0") for s in shapes]
    t = lambda a: torch.tensor(a, device="cuda:0")

    def eager(xi):
        leaves = [t(xi[k]).requires_grad_(True) for k in ("q", "qd", "act")]
        loss, outs = _graph_loss(eng, cfg, *leaves, w)
        loss.backward()
        return [loss.detach().view(1)] + [o.detach() for o in outs] + [v.grad for v in leaves]

    static = [t(x0[k]).requires_grad_(True) for k in ("q", "qd", "act")]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):             # warm-up off the default stream, as torch.cuda.graphs asks
        for _ in range(2):
            for v in static:
                v.grad = None
            _graph_loss(eng, cfg, *static, w)[0].backward()
    torch.cuda.current_stream().wait_stream(side)
    for v in static:
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):             # the dynamics backward allocates its workspace here, from the graph's pool
        loss, outs = _graph_loss(eng, cfg, *static, w)
        loss.backward()
    for xi in (x1, x0):
        with torch.no_grad():
            for v, k in zip(static, ("q", "qd", "act")):
                v.copy_(t(xi[k]))
        graph.replay()
        torch.cuda.synchronize()
        replayed = [loss.detach().view(1)] + [o.detach() for o in outs] + [v.grad for v in static]
        replayed = [r.clone() for r in replayed]
        ref = eager(xi)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(ref[0]).all()), name
        for i, (a, b) in enumerate(zip(replayed, ref)):
            assert not _differing(a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)), (name, "graph replay vs eager, result", i)
    print(name, "graph of env-step + four-readout loss + backward: two replays equal eager bit for bit")
