"""External link wrenches (include/dfx.h DfxExternalWrench, the _ex entries) on the kernels.

* every kernel family of the six DiffRL articulations (auto, tile8/16/32, group8/16/32), N = 75:
  - at the model's own (substeps, mm_freq), fp32 tape: q', qd' and gq, gqd, gact, g_f_ext against the fp64 oracle within
    wrench_util.wrench_tol (4x the host emulation's error);
  - at (1, 1), (7, 3) and the model's own, both tape dtypes: a zero wrench steps bit for bit as the entries without one
    (states, tape, cotangents), and the recompute adjoint equals tape mode bit for bit, g_f_ext included;
* physics independent of the oracle: a free body under a force at its centre of mass, a pure torque, Ant held up by
  F_i = -m_i g on every link;
* the three env step paths (op-by-op, mapped, single launch) give the same wrench gradient;
* refusals: shape / dtype / device of f_ext, GraphedRollout with a wrench set, an articulation whose wrench kernels do not fit."""
import numpy as np
import pytest

import random_articulation as R
import wrench_util as W
from wrench_util import WrenchOracle, wrench_tol
from test_gpu_golden import _select

pytestmark = pytest.mark.gpu

N = 75
VARIANTS = ["auto", "tile8", "tile16", "tile32", "group8", "group16", "group32"]


def _t(a):
    import torch
    return None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda:0")


def _engine(model, meta, variant, bf16=False):
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    _select(variant)
    _capi.lib().dfx_set_tape_dtype(int(bf16))
    try:
        desc, _ = articulation_from_model(model, meta["num_envs"])
        return ArticulationEngine(desc, N, "cuda:0")
    finally:
        _capi.lib().dfx_set_tape_dtype(0)
        _select("auto")


def _step(eng, inp, f, S, mm, dt, recompute=False):
    """forward with a tape, then the tape (or recompute) adjoint; f None: the entries without a wrench"""
    q0, qd0, act, musc = _t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"])
    ft = _t(f)
    q, qd, tape, _ = eng.forward(q0, qd0, act, musc, S, mm, dt, f_ext=ft)
    if recompute:
        g = eng.backward_recompute(q0, qd0, act, musc, _t(inp["gq_out"]), _t(inp["gqd_out"]), S, mm, dt, f_ext=ft)
    else:
        g = eng.backward(act, musc, tape, _t(inp["gq_out"]), _t(inp["gqd_out"]), S, mm, dt, f_ext=ft)
    return q, qd, tape, g


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", W.ENVS)
def test_cuda_wrench_matches_oracle(name, variant):
    model, meta, inp = W.golden_batch(name, N)
    eng = _engine(model, meta, variant)
    f = W.random_wrench(model, meta["num_envs"], N, 7)
    q, qd, _, g = _step(eng, inp, f, meta["S"], meta["mm"], meta["dt"])
    o = WrenchOracle.from_model(model, meta["num_envs"])
    err = W.oracle_errors(o, inp, f.astype(np.float64), q.cpu().numpy(), qd.cpu().numpy(),
                          [x.cpu().numpy() for x in (g[0], g[1], g[2], g[4])], meta)
    print(name, variant, "tile", int(eng.lib.dfx_pack_query(eng.pack, 9)), {k: "%.2f" % (v / wrench_tol(name, k)) for k, v in err.items()})
    for block, v in err.items():
        assert v <= wrench_tol(name, block), (name, variant, block, v, wrench_tol(name, block))


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", W.ENVS)
def test_zero_wrench_and_recompute_are_bitwise(name, variant, bf16):
    import torch
    model, meta, inp = W.golden_batch(name, N)
    eng = _engine(model, meta, variant, bf16)
    f = W.random_wrench(model, meta["num_envs"], N, 7)
    for S, mm in ((1, 1), (7, 3), (meta["S"], meta["mm"])):
        dt = meta["dt"] * S / meta["S"]
        plain = _step(eng, inp, None, S, mm, dt)
        zero = _step(eng, inp, np.zeros_like(f), S, mm, dt)
        for a, b in zip(plain[:3], zero[:3]):
            assert torch.equal(a, b), (name, variant, bf16, S, mm)
        for a, b in zip(plain[3], zero[3][:4]):
            assert (a is None and b is None) or torch.equal(a, b), (name, variant, bf16, S, mm)
        tape = _step(eng, inp, f, S, mm, dt)
        rec = _step(eng, inp, f, S, mm, dt, recompute=True)
        for a, b in zip(tape[3], rec[3]):
            assert (a is None and b is None) or torch.equal(a, b), (name, variant, bf16, S, mm)
        assert torch.isfinite(tape[3][4]).all() and tape[3][4].abs().max() > 0


# ------------------------------------------------------------------ physics
def _free_body(mass=2.0, inertia=(0.3, 0.5, 0.7)):
    m = R._build(np.random.default_rng(0), [R.FREE], [-1], [])
    I = np.zeros((1, 6, 6))
    I[0, :3, :3] = np.diag(inertia)
    I[0, 3:, 3:] = np.eye(3) * mass
    m["body_I_m"] = I
    m["ground"] = False
    m["joint_X_cm"] = np.array([[0.1, -0.2, 0.05, 0, 0, 0, 1]])   # centre of mass off the joint frame
    return m


def test_force_at_centre_of_mass_accelerates_without_rotation():
    import torch
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    mass = 2.0
    desc, _ = articulation_from_model(_free_body(mass), 1)
    eng = ArticulationEngine(desc, 1, "cuda:0")
    eng.set_gravity([0.0, 0.0, 0.0], False)
    q = torch.tensor([0, 1, 0, 0, 0, 0, 1], dtype=torch.float32, device="cuda:0")
    qd = torch.zeros(6, device="cuda:0")
    F = np.array([3.0, -1.5, 2.0])
    f = torch.tensor(np.concatenate([np.zeros(3), F])[None, None], dtype=torch.float32, device="cuda:0")
    S, dt = 16, 1.0 / 60.0
    for _ in range(10):
        q, qd, _, _ = eng.forward(q, qd, torch.zeros(6, device="cuda:0"), None, S, 1, dt, want_tape=False, f_ext=f)
    w, v = qd[:3].cpu().numpy(), qd[3:].cpu().numpy()
    c = q[:3].cpu().numpy() + np.array([0.1, -0.2, 0.05])      # (unrotated body: the COM offset stays as it was)
    v_com = v + np.cross(w, c)
    assert np.abs(w).max() < 1e-6, w
    assert np.allclose(v_com, F * 10 * dt / mass, rtol=1e-5, atol=1e-6), (v_com, F * 10 * dt / mass)


def test_pure_torque_spins_the_body():
    import torch
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    inertia = np.array([0.3, 0.5, 0.7])
    desc, _ = articulation_from_model(_free_body(2.0, inertia), 1)
    eng = ArticulationEngine(desc, 1, "cuda:0")
    eng.set_gravity([0.0, 0.0, 0.0], False)
    q = torch.tensor([0, 1, 0, 0, 0, 0, 1], dtype=torch.float32, device="cuda:0")
    tau = np.array([0.2, -0.4, 0.3])
    f = torch.tensor(np.concatenate([tau, np.zeros(3)])[None, None], dtype=torch.float32, device="cuda:0")
    dt = 1.0 / 960.0
    _, qd, _, _ = eng.forward(q, torch.zeros(6, device="cuda:0"), torch.zeros(6, device="cuda:0"), None, 1, 1, dt,
                              want_tape=False, f_ext=f)
    w = qd[:3].cpu().numpy()
    assert np.allclose(w, tau / inertia * dt, rtol=1e-5, atol=1e-9), (w, tau / inertia * dt)


def test_ant_held_up_by_its_weight_stays_at_rest():
    import torch
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    model, meta, inp = W.golden_batch("AntEnv", 4)
    desc, _ = articulation_from_model(model, meta["num_envs"])
    eng = ArticulationEngine(desc, 4, "cuda:0")
    L = eng.L
    Q = eng.Q
    q = inp["q0"].copy()
    target = np.asarray(model["joint_target"], np.float32)[:Q]
    q[:, 7:] = target[7:]
    q[:, 1] += 1.0                      # clear of the ground
    m = W.link_masses(model)[:L]
    f = np.zeros((4, L, 6), np.float32)
    f[:, :, 4] = 9.81 * m               # F_i = -m_i g, g = (0, -9.81, 0)
    qt, qdt = _t(q), torch.zeros((4, eng.D), device="cuda:0")
    act = torch.zeros((4, eng.D), device="cuda:0")
    for _ in range(100):
        qt, qdt, _, _ = eng.forward(qt, qdt, act, None, meta["S"], meta["mm"], meta["dt"], want_tape=False, f_ext=_t(f))
    assert float((qt.cpu() - torch.tensor(q)).abs().max()) < 1e-6
    assert float(qdt.abs().max()) < 1e-6


# ------------------------------------------------------------------ the env paths
def _env_wrench_grad(single_launch, fused_map, steps=3):
    import torch
    from diffrl_b200.envs.locomotion import AntEnv
    env = AntEnv(num_envs=16, no_grad=False, device="cuda:0")
    env.single_launch_step, env.fused_action_map = single_launch, fused_map
    env.reset()
    L = env.model.link_count // env.num_envs
    w = torch.tensor(W.random_wrench({"body_I_m": env.model.body_I_m.cpu().numpy()}, env.num_envs, env.num_envs, 3),
                     device="cuda:0", requires_grad=True)
    env.set_external_wrench(w)
    a = torch.full((env.num_envs, env.num_actions), 0.3, device="cuda:0")
    loss = 0.0
    for _ in range(steps):
        obs, rew, done, _ = env.step(a)
        loss = loss + rew.sum()
    loss.backward()
    assert w.grad is not None and w.grad.shape == (env.num_envs, L, 6)
    return w.grad.clone()


def test_env_paths_give_the_same_wrench_gradient():
    import torch
    g1 = _env_wrench_grad(True, True)
    g2 = _env_wrench_grad(False, True)
    g3 = _env_wrench_grad(False, False)
    assert float(g1.abs().max()) > 0
    # (the transition is compiled twice -- epilogue and own kernel -- so observations and rewards may differ by a few ulp)
    for g in (g2, g3):
        assert torch.allclose(g1, g, rtol=1e-5, atol=1e-6 * float(g1.abs().max())), float((g1 - g).abs().max())


def test_dflex_integrator_reads_state_wrench():
    import torch
    import diffrl_b200.dflex_api as df
    from diffrl_b200.envs.locomotion import AntEnv
    env = AntEnv(num_envs=2, no_grad=False, device="cuda:0")
    f = torch.tensor(W.random_wrench({"body_I_m": env.model.body_I_m.cpu().numpy()}, 2, 2, 5), device="cuda:0",
                     requires_grad=True)
    st = env.model.state()
    st.joint_q, st.joint_qd = env.state.joint_q.detach().clone(), env.state.joint_qd.detach().clone()
    st.joint_act = torch.zeros_like(st.joint_qd)
    st.body_f_ext = f
    out = df.sim.SemiImplicitIntegrator().forward(env.model, st, env.sim_dt, env.sim_substeps, env.MM_caching_frequency)
    assert "body_f_ext" not in out.__dict__
    gq_out = torch.ones_like(out.joint_q)
    (out.joint_q * gq_out).sum().backward()
    from diffrl_b200.dflex_api.sim import _engine_for
    eng = _engine_for(env.model)
    o = WrenchOracle(eng.desc)
    q0 = st.joint_q.cpu().numpy().reshape(2, -1)
    qd0 = st.joint_qd.cpu().numpy().reshape(2, -1)
    fn = f.detach().cpu().numpy()
    oq, _ = o.forward_ext(q0, qd0, np.zeros_like(qd0), None, fn, env.sim_substeps, env.MM_caching_frequency, env.sim_dt)
    assert W.rel_err(out.joint_q.detach().cpu().numpy(), oq) < 1e-5
    ex = o.exact_gradient_ext(q0[0], qd0[0], np.zeros_like(qd0[0]), None, fn[0], np.ones(q0.shape[1]), np.zeros(qd0.shape[1]),
                              env.sim_substeps, env.MM_caching_frequency, env.sim_dt)[4]
    assert W.rel_err(f.grad[0].cpu().numpy(), ex) < 4 * 1e-5, W.rel_err(f.grad[0].cpu().numpy(), ex)
    # the derived body_f_s dump includes the wrench
    _ = out.body_f_s


# ------------------------------------------------------------------ refusals
def test_bad_wrench_inputs_are_refused():
    import torch
    from diffrl_b200.engine import SimStepFunction
    model, meta, inp = W.golden_batch("AntEnv", N)
    eng = _engine(model, meta, "auto")
    L = eng.L
    args = (_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), None, meta["S"], meta["mm"], meta["dt"])
    for bad in (torch.zeros((N, L, 5), device="cuda:0"), torch.zeros((N, L + 1, 6), device="cuda:0"),
                torch.zeros((N, L, 6), dtype=torch.float64, device="cuda:0"), torch.zeros((N, L, 6))):
        with pytest.raises(ValueError):
            eng.forward(*args, f_ext=bad)
        with pytest.raises(ValueError):
            SimStepFunction.apply(eng, meta["S"], meta["mm"], meta["dt"], _t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), None, bad)
    eng.forward(*args, f_ext=torch.zeros((N * L, 6), device="cuda:0"))     # the flat layout is accepted


def test_graphed_rollout_refuses_a_wrench():
    import torch
    from diffrl_b200.envs.locomotion import AntEnv
    from diffrl_b200.rollout import GraphedRollout
    env = AntEnv(num_envs=8, no_grad=False, device="cuda:0")
    L = env.model.link_count // env.num_envs
    env.set_external_wrench(torch.zeros((8, L, 6), device="cuda:0"))
    with pytest.raises(RuntimeError, match="external wrench"):
        GraphedRollout(env, horizon=4)
    with pytest.raises(ValueError):
        env.set_external_wrench(torch.zeros((8, L, 5), device="cuda:0"))


def test_articulation_whose_wrench_kernels_do_not_fit_is_refused():
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    from test_gpu_random_articulations import _chain
    # the longest chain whose plain kernels fit (test_gpu_random_articulations: 100 links fit, 104 do not)
    L = 104
    while True:
        desc, _ = articulation_from_model(_chain(L), 1)
        try:
            eng = ArticulationEngine(desc, 4, "cuda:0")
            break
        except _capi.DfxError:
            L -= 1
    f = torch.zeros((4, L, 6), device="cuda:0")
    q = torch.zeros((4, eng.Q), device="cuda:0")
    q[:, 6] = 1.0
    with pytest.raises(_capi.DfxError, match="with the external wrench and its cotangent staged"):
        eng.forward(q, torch.zeros((4, eng.D), device="cuda:0"), torch.zeros((4, eng.D), device="cuda:0"), None, 2, 2, 1 / 480,
                    f_ext=f)
    print("chain of %d links: plain kernels fit, wrench kernels refused" % L)
