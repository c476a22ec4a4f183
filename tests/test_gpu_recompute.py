"""Recompute adjoint (include/dfx.h dfx_*_backward_recompute, diffrl_b200.set_adjoint_mode("recompute")): no tape is kept, each
env-step's forward is re-run into a one-env-step workspace inside its adjoint launch.  The forward is deterministic, so the
recomputed tape IS the stored tape, and the adjoint is deterministic too (fixed-point cotangent scatter for the muscle model,
one owner per body for the contact cotangents of the others), so the gradients are those of the stored-tape path: every
comparison here is bitwise (torch.equal), on the same saved forward state and the same actions."""
import contextlib
import ctypes

import numpy as np
import pytest

from emu_util import EmuSim, load_golden

pytestmark = pytest.mark.gpu

ARTICULATIONS = ["AntEnv", "HumanoidEnv", "SNUHumanoidEnv", "CartPoleSwingUpEnv", "HopperEnv", "CheetahEnv"]
ENVS = ARTICULATIONS
MM = {"AntEnv": 16, "HumanoidEnv": 48, "SNUHumanoidEnv": 8, "CartPoleSwingUpEnv": 4, "HopperEnv": 16, "CheetahEnv": 16}
LANE_GROUP = 41          # dfx_set_flags: default 9 + bit 5 (keep the articulation on the lane-group kernels)


@contextlib.contextmanager
def pack_settings(flags=9, tile_envs=0, bf16=False):
    """Settings read when a pack is created, restored afterwards."""
    from diffrl_b200 import _capi
    lib = _capi.lib()
    lib.dfx_set_flags(flags)
    lib.dfx_set_tile_envs(tile_envs)
    lib.dfx_set_tape_dtype(1 if bf16 else 0)
    try:
        yield lib
    finally:
        lib.dfx_set_flags(9)
        lib.dfx_set_tile_envs(0)
        lib.dfx_set_tape_dtype(0)


@contextlib.contextmanager
def adjoint_mode(mode):
    import diffrl_b200
    diffrl_b200.set_adjoint_mode(mode)
    try:
        yield
    finally:
        diffrl_b200.set_adjoint_mode("tape")


def _inputs(name, N, seed=0):
    """(emu, q, qd, act, musc or None, substeps, mm_freq, dt): N environments drawn from the golden states, perturbed."""
    import torch
    d, model = load_golden(name)
    n0 = int(d["meta/num_envs"])
    emu = EmuSim(model, n0)
    Q, D, M = emu.desc.Q, emu.desc.D, emu.desc.M
    rng = np.random.default_rng(seed)
    p = "case%d/" % (int(d["meta/num_cases"]) - 1)
    pick = rng.integers(0, n0, N)
    t = lambda a: torch.tensor(np.ascontiguousarray(a, np.float32).ravel(), device="cuda:0")
    q0 = d[p + "q0"].reshape(n0, Q)[pick]
    qd0 = d[p + "qd0"].reshape(n0, D)[pick] * rng.uniform(0.8, 1.2, (N, 1))
    act = d[p + "act"].reshape(n0, D)[pick] * rng.uniform(0.5, 1.5, (N, D))
    musc = np.clip(d[p + "musc"].reshape(n0, M)[pick] * rng.uniform(0.5, 1.5, (N, M)), 0.0, 1.0) if M else None
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    return emu, t(q0), t(qd0), t(act), None if musc is None else t(musc), S, mm, dt


def _configs(name):
    """(flags, tile width, bf16 tape) of every kernel this articulation can run on: each tile width that exists, fp32 and bf16
    tape, and the lane-group kernels (fp32 only: they ignore the tape dtype)."""
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    emu = _inputs(name, 1)[0]
    out = [(LANE_GROUP, 0, False)]
    for E in (32, 16, 8):
        with pack_settings(tile_envs=E):
            if int(_capi.lib().dfx_pack_query(ArticulationEngine(emu.desc, 1, "cuda:0").pack, 9)) == E:
                out += [(9, E, False), (9, E, True)]
    return out


@pytest.mark.parametrize("name", ARTICULATIONS)
def test_recomputed_tape_equals_stored_tape(name):
    """Every kernel family, tile width and tape dtype: the rows and H^-1 blocks the recompute leaves in the workspace, and its end
    state, equal the stored tape and the forward's outputs bitwise; so do the cotangents of the two adjoints."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    N = 33
    emu, q, qd, act, musc, S, mm, dt = _inputs(name, N, seed=1)
    gq_out = torch.linspace(-1.0, 1.0, q.numel(), device="cuda:0")
    gqd_out = torch.linspace(1.0, -1.0, qd.numel(), device="cuda:0")
    for flags, E, bf16 in _configs(name):
        with pack_settings(flags, E, bf16) as lib:
            eng = ArticulationEngine(emu.desc, N, "cuda:0")
            assert int(lib.dfx_pack_query(eng.pack, 9)) == E and int(lib.dfx_pack_query(eng.pack, 10)) == int(bf16 and E > 0)
            q1, qd1, tape, _ = eng.forward(q, qd, act, musc, S, mm, dt)
            g_tape = eng.backward(act, musc, tape, gq_out, gqd_out, S, mm, dt)
            ws = eng.recompute_workspace(S, mm)
            assert ws.numel() == tape.numel() + N * (eng.Q + eng.D)
            ws.fill_(float("nan"))                   # nothing of the workspace's previous contents may survive
            g_rec = eng.backward_recompute(q, qd, act, musc, gq_out, gqd_out, S, mm, dt, workspace=ws)
            cfg = (name, flags, E, bf16)
            assert torch.equal(eng.tape_rows(ws, S), eng.tape_rows(tape, S)), cfg
            assert torch.equal(eng.tape_hinv(ws, S, mm), eng.tape_hinv(tape, S, mm)), cfg
            q_end, qd_end = eng.workspace_end_state(ws, S, mm)
            assert torch.equal(q_end, q1) and torch.equal(qd_end, qd1), cfg
            for a, b in zip(g_rec, g_tape):
                assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), cfg


@pytest.mark.parametrize("N", [1, 7, 33])
@pytest.mark.parametrize("cfg", [(16, 16), (1, 1), (5, 16), (16, 3)])
def test_step_gradients_equal_for_substep_patterns(N, cfg):
    """dfx_step_backward_recompute == dfx_step_backward, bitwise, on the batch sizes and (substeps, mm_freq) patterns of
    test_gpu_edges.py, on the tile kernels and on the lane-group kernels."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    S, mm = cfg
    emu, q, qd, act, _, _, _, dt = _inputs("AntEnv", N, seed=N)
    dt = dt * S / 16.0
    for flags in (9, LANE_GROUP):
        with pack_settings(flags):
            eng = ArticulationEngine(emu.desc, N, "cuda:0")
            _, _, tape, _ = eng.forward(q, qd, act, None, S, mm, dt)
            gq_out, gqd_out = torch.ones_like(q), torch.ones_like(qd)
            g_tape = eng.backward(act, None, tape, gq_out, gqd_out, S, mm, dt)
            g_rec = eng.backward_recompute(q, qd, act, None, gq_out, gqd_out, S, mm, dt)
            for a, b in zip(g_rec[:3], g_tape[:3]):
                assert torch.equal(a, b), (N, cfg, flags)


def test_null_cotangents_and_null_outputs():
    """NULL cotangents mean zero and NULL outputs skip the write, as in the stored-tape adjoint."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    emu, q, qd, act, _, S, mm, dt = _inputs("CheetahEnv", 5)
    eng = ArticulationEngine(emu.desc, 5, "cuda:0")
    _, _, tape, _ = eng.forward(q, qd, act, None, S, mm, dt)
    for gq_out, gqd_out in ((torch.ones_like(q), None), (None, torch.ones_like(qd)), (None, None)):
        for need in ((True, True, True, False), (False, False, True, False), (True, False, False, False)):
            g_tape = eng.backward(act, None, tape, gq_out, gqd_out, S, mm, dt, need=need)
            g_rec = eng.backward_recompute(q, qd, act, None, gq_out, gqd_out, S, mm, dt, need=need)
            for a, b in zip(g_rec, g_tape):
                assert (a is None) == (b is None) and (a is None or torch.equal(a, b))


def _rollout(name, n, T, mode, seed=11, episode_length=3, single_launch=True, fused_map=True, poison=False):
    """T env.steps of a fresh env in the given adjoint mode: (loss, action gradients, launches in forward, launches in backward)."""
    import torch
    import diffrl_b200.envs as envs
    from diffrl_b200 import _capi
    with adjoint_mode(mode):
        torch.manual_seed(0)
        env = getattr(envs, name)(num_envs=n, device="cuda:0", no_grad=False, MM_caching_frequency=MM[name], episode_length=episode_length)
        env.single_launch_step = single_launch
        env.fused_action_map = fused_map
        env.clear_grad(); env.reset(); env.initialize_trajectory()
        if poison:                               # a NaN joint angle: the humanoids' gradient guard zeroes what flows from it
            with torch.no_grad():
                q = env.state.joint_q.clone()
                q.view(n, -1)[3, 9] = float("nan")
                env.state.joint_q = q
        g = torch.Generator(device="cuda:0").manual_seed(seed)
        acts = [((torch.rand((n, env.num_actions), generator=g, device="cuda:0") * 2 - 1) * 1.5).requires_grad_() for _ in range(T)]
        w = torch.linspace(0.5, 1.5, env.num_obs, device="cuda:0")
        l0 = _capi.lib().dfx_launch_count()
        loss = 0.0
        for a in acts:
            obs, rew, done, extras = env.step(a)
            loss = loss + rew.sum() + (obs * w).sum() * 1e-2 + (extras["obs_before_reset"] * w).sum() * 3e-3
        l1 = _capi.lib().dfx_launch_count()
    loss.backward()                              # (outside the context: the mode of the forward must stick)
    l2 = _capi.lib().dfx_launch_count()
    return loss.detach(), torch.stack([a.grad for a in acts]), l1 - l0, l2 - l1


@pytest.mark.parametrize("name", ENVS)
def test_env_rollouts_equal_in_both_modes(name):
    """env.step() rollouts of 7 steps with terminations inside the window: the single-launch step (dfx_env_step_backward_recompute)
    and the mapped step (dfx_step_backward_mapped_recompute) give the loss and action gradients of tape mode bitwise; the
    recompute mode's forward launches no more kernels."""
    import torch
    n, T = 40, 7
    for single in (True, False):
        ref = _rollout(name, n, T, "tape", single_launch=single)
        rec = _rollout(name, n, T, "recompute", single_launch=single)
        assert torch.equal(rec[0], ref[0]) and torch.equal(rec[1], ref[1]), (name, single)
        assert rec[2] == ref[2]


def test_drop_in_integrator_gradients_equal_in_both_modes():
    """The drop-in SemiImplicitIntegrator path (SimStepFunction, dfx_step_backward_recompute) on Ant and SNU (muscles)."""
    import torch
    for name in ("AntEnv", "SNUHumanoidEnv"):
        ref = _rollout(name, 24, 5, "tape", single_launch=False, fused_map=False)
        rec = _rollout(name, 24, 5, "recompute", single_launch=False, fused_map=False)
        assert torch.equal(rec[0], ref[0]) and torch.equal(rec[1], ref[1]), name


def test_nan_guard_in_recompute_mode():
    """A poisoned Humanoid environment: the single-launch step's gradient guard acts the same in both modes."""
    import torch
    ref = _rollout("HumanoidEnv", 8, 3, "tape", poison=True)
    rec = _rollout("HumanoidEnv", 8, 3, "recompute", poison=True)
    assert torch.equal(rec[1], ref[1])
    keep = torch.arange(8, device="cuda:0") != 3
    assert torch.isfinite(rec[1][:, keep]).all()


def test_graphed_rollout_equals_in_both_modes():
    import torch
    import diffrl_b200.envs as envs
    from diffrl_b200.rollout import GraphedRollout
    n, T = 48, 6
    acts = torch.rand((T, n, 8), generator=torch.Generator().manual_seed(2)) * 2 - 1
    res = []
    for mode in ("tape", "recompute"):
        with adjoint_mode(mode):
            env = envs.AntEnv(num_envs=n, device="cuda:0", no_grad=False, MM_caching_frequency=16, episode_length=4)
            env.clear_grad(); env.reset(); env.initialize_trajectory()
            roll = GraphedRollout(env, T)
            out = []
            for _ in range(2):                   # two chained windows
                loss, grad = roll(acts)
                out.append((loss.clone(), grad.clone()))
            res.append(out)
    for (l1, g1), (l2, g2) in zip(*res):
        assert torch.equal(l1, l2) and torch.equal(g1, g2)


def test_launch_counts():
    """One launch per env-step adjoint on the tile kernels (forward and adjoint in the same CTA); two (the forward, then the
    stored-tape adjoint) on the lane-group kernels."""
    from diffrl_b200.engine import ArticulationEngine
    emu, q, qd, act, _, S, mm, dt = _inputs("AntEnv", 40)
    for flags, launches in ((9, 1), (LANE_GROUP, 2)):
        with pack_settings(flags) as lib:
            eng = ArticulationEngine(emu.desc, 40, "cuda:0")
            l0 = lib.dfx_launch_count()
            eng.backward_recompute(q, qd, act, None, q, qd, S, mm, dt)
            assert lib.dfx_launch_count() - l0 == launches, flags
    for name in ENVS:                            # env.step: one adjoint launch per step, as in tape mode
        ref, rec = _rollout(name, 16, 2, "tape"), _rollout(name, 16, 2, "recompute")
        assert rec[3] == ref[3] == 2, name


def _peak_rollout(n, T, mode):
    """Ant n x T, loss = sum of rewards: (peak bytes allocated above the start, action gradients, tape bytes of one env-step)."""
    import torch
    import diffrl_b200.envs as envs
    with adjoint_mode(mode):
        env = envs.AntEnv(num_envs=n, device="cuda:0", no_grad=False, MM_caching_frequency=16)
        env.clear_grad(); env.reset(); env.initialize_trajectory()
        g = torch.Generator(device="cuda:0").manual_seed(7)
        acts = (torch.rand((T, n, 8), generator=g, device="cuda:0") * 2 - 1).requires_grad_()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        loss = 0.0
        for t in range(T):
            obs, rew, done, _ = env.step(acts[t])
            loss = loss + rew.sum()
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    eng = env.model._engine
    return peak, acts.grad.detach().clone(), 4 * eng.tape_floats(16, 16), eng


def test_recompute_memory_stays_bounded():
    """Ant 4096 x 64: recompute mode peaks below one workspace plus an allowance per env-step for what the graph keeps (the
    step's input and output states, the actions, their clipped copies and gradients: 4 x N x (Q + D + A) floats), under a fifth
    of tape mode, with bitwise equal gradients.  Then 4096 x 1000 -- about 112 GB of tape, more than the device holds -- runs
    in recompute mode within the same bound."""
    import torch
    n, T = 4096, 64
    peak_tape, g_tape, tape_step, _ = _peak_rollout(n, T, "tape")
    peak_rec, g_rec, _, eng = _peak_rollout(n, T, "recompute")
    ws = 4 * int(eng.lib.dfx_recompute_workspace_floats(eng.pack, n, 16, 16))
    allowance = 4 * 4 * n * (eng.Q + eng.D + 8)
    print("Ant 4096 x 64: peak tape %.2f GB, recompute %.3f GB (workspace %.0f MB, allowance %.2f MB / env-step)"
          % (peak_tape / 1e9, peak_rec / 1e9, ws / 1e6, allowance / 1e6))
    assert peak_tape >= T * tape_step
    assert peak_rec <= ws + T * allowance
    assert peak_rec * 5 < peak_tape
    assert torch.equal(g_rec, g_tape)
    del g_tape, g_rec
    T = 1000
    assert T * tape_step > torch.cuda.get_device_properties(0).total_memory
    peak, g, _, _ = _peak_rollout(n, T, "recompute")
    print("Ant 4096 x 1000 recompute: peak %.2f GB" % (peak / 1e9))
    assert peak <= ws + T * allowance
    assert torch.isfinite(g).all()


def test_argument_validation():
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.env_ops import DfxEnvTransitionAdj, _bind
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import DfxActionMap
    emu, q, qd, act, _, S, mm, dt = _inputs("AntEnv", 4)
    eng = ArticulationEngine(emu.desc, 4, "cuda:0")
    lib = _capi.lib()
    _bind(lib)
    z, p = ctypes.c_void_p(0), ctypes.c_void_p(q.data_ptr())
    ws = eng.recompute_workspace(S, mm)
    w = ctypes.c_void_p(ws.data_ptr())
    strength = torch.ones(8, device="cuda:0")
    m = DfxActionMap(8, 6, 0, 1.0, 0.0, 1.0, strength.data_ptr())
    # a transition the entry accepts (only the pointers below are missing)
    tr = DfxEnvTransitionAdj(kind=1)
    tr.walker.num_q, tr.walker.num_qd, tr.walker.num_act, tr.walker.num_obs = eng.Q, eng.D, 8, 37
    for f in ("q_sim", "qd_sim", "used", "reset", "gq_sim", "gqd_sim", "g_used"):
        setattr(tr, f, q.data_ptr())
    bad = 1                                      # cudaErrorInvalidValue
    for qq, qqd, ww in ((z, p, w), (p, z, w), (p, p, z)):
        assert lib.dfx_step_backward_recompute(eng.pack, 4, S, mm, dt, qq, qqd, p, z, ww, z, z, z, z, z, z, z) == bad
        assert lib.dfx_step_backward_mapped_recompute(eng.pack, 4, S, mm, dt, qq, qqd, ctypes.byref(m), p, z, ww, z, z, z, z, z, z, z) == bad
        assert lib.dfx_env_step_backward_recompute(eng.pack, 4, S, mm, dt, qq, qqd, ctypes.byref(m), p, z, ww, ctypes.byref(tr), z, z, z, z) == bad
    assert lib.dfx_recompute_workspace_floats(eng.pack, 0, S, mm) == -1
    with pytest.raises(ValueError):
        import diffrl_b200
        diffrl_b200.set_adjoint_mode("checkpoint")
