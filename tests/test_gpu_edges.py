"""Edge cases of the C ABI on the GPU: batch sizes around the CTA tile, single substep, mass-matrix
period longer than the step, a model without contacts, argument validation, NULL gradient outputs."""
import ctypes

import numpy as np
import pytest

from emu_util import EmuSim, load_golden
from tolerances import GRAD_RTOL, fwd_rtol

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.abs(a - b).max() / (np.abs(b).max() + 1e-30)


def _case(name, N, seed=0):
    d, model = load_golden(name)
    n0 = int(d["meta/num_envs"])
    emu = EmuSim(model, n0)
    Q, D = emu.desc.Q, emu.desc.D
    rng = np.random.default_rng(seed)
    p = "case%d/" % (int(d["meta/num_cases"]) - 1)
    pick = rng.integers(0, n0, N)
    q0 = d[p + "q0"].reshape(n0, Q)[pick].copy()
    qd0 = d[p + "qd0"].reshape(n0, D)[pick] * rng.uniform(0.8, 1.2, (N, 1)).astype(np.float32)
    act = d[p + "act"].reshape(n0, D)[pick] * rng.uniform(0.5, 1.5, (N, D)).astype(np.float32)
    emu.N = N
    return d, emu, q0.astype(np.float32), qd0.astype(np.float32), act.astype(np.float32)


@pytest.mark.parametrize("N", [1, 7, 8, 9, 33])
@pytest.mark.parametrize("cfg", [(16, 16), (1, 1), (5, 16), (16, 3)])
def test_batch_sizes_and_substep_patterns(N, cfg):
    import torch
    from diffrl_b200.engine import ArticulationEngine
    S, mm = cfg
    d, emu, q0, qd0, act = _case("AntEnv", N, seed=N)
    dt = float(d["meta/dt"]) * S / 16.0
    eq, eqd, etape, _ = emu.forward(q0.ravel(), qd0.ravel(), act.ravel(), None, S, mm, dt)
    gqo, gqdo = np.ones_like(q0).ravel(), np.ones_like(qd0).ravel()
    egq, egqd, egact, _ = emu.backward(act.ravel(), None, etape, gqo, gqdo, S, mm, dt)
    eng = ArticulationEngine(emu.desc, N, "cuda:0")
    t = lambda a: torch.tensor(a.ravel(), device="cuda:0")
    q, qd, tape, _ = eng.forward(t(q0), t(qd0), t(act), None, S, mm, dt)
    assert tape.numel() == eng.tape_floats(S, mm) >= etape.size      # (tile kernels pad the tape to whole 32-env tiles)
    gq, gqd, gact, _ = eng.backward(t(act), None, tape, t(gqo), t(gqdo), S, mm, dt)
    assert rel(q.cpu().numpy(), eq) < fwd_rtol("AntEnv") and rel(qd.cpu().numpy(), eqd) < fwd_rtol("AntEnv")
    assert rel(gq.cpu().numpy(), egq) < 4 * GRAD_RTOL and rel(gact.cpu().numpy(), egact) < 4 * GRAD_RTOL


def test_null_gradient_outputs_and_cotangents():
    """NULL output pointers skip the write (reference: empty adjoint tensor => skip, adjoint.h:336-346);
    NULL cotangents mean zero."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    d, emu, q0, qd0, act = _case("CheetahEnv", 5)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    eng = ArticulationEngine(emu.desc, 5, "cuda:0")
    t = lambda a: torch.tensor(a.ravel(), device="cuda:0")
    q, qd, tape, _ = eng.forward(t(q0), t(qd0), t(act), None, S, mm, dt)
    full = eng.backward(t(act), None, tape, torch.ones_like(q), None, S, mm, dt)
    only_act = eng.backward(t(act), None, tape, torch.ones_like(q), torch.zeros_like(qd), S, mm, dt, need=(False, False, True, False))
    assert only_act[0] is None and only_act[1] is None
    assert torch.allclose(full[2], only_act[2], rtol=1e-5, atol=1e-6 * float(full[2].abs().max()))


def test_argument_validation_returns_cuda_error_codes():
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    d, emu, q0, qd0, act = _case("AntEnv", 4)
    eng = ArticulationEngine(emu.desc, 4, "cuda:0")
    lib = _capi.lib()
    z = ctypes.c_void_p(0)
    q = torch.tensor(q0.ravel(), device="cuda:0")
    p = ctypes.c_void_p(q.data_ptr())
    assert lib.dfx_step_forward(eng.pack, 4, 16, 16, 1.0 / 60, z, p, p, z, p, p, z, None, z) == 1      # cudaErrorInvalidValue
    assert lib.dfx_step_forward(eng.pack, 0, 16, 16, 1.0 / 60, p, p, p, z, p, p, z, None, z) == 1
    assert lib.dfx_step_backward(eng.pack, 4, 16, 16, 1.0 / 60, p, z, z, z, z, z, z, z, z, z) == 1      # no tape
    assert lib.dfx_set_group_size(5) != 0 and lib.dfx_set_group_size(0) == 0


def test_pack_rejects_malformed_models():
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    d, emu, *_ = _case("AntEnv", 2)
    bad = emu.desc
    bad.arrays["joint_parent"] = bad.arrays["joint_parent"].copy()
    bad.arrays["joint_parent"][1] = 5          # parent after child
    with pytest.raises(_capi.DfxError):
        ArticulationEngine(bad, 2, "cuda:0")


def test_cartpole_has_no_contacts_and_fixed_root():
    import torch
    from diffrl_b200.engine import ArticulationEngine
    d, emu, q0, qd0, act = _case("CartPoleSwingUpEnv", 6)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    eq, eqd, etape, _ = emu.forward(q0.ravel(), qd0.ravel(), act.ravel(), None, S, mm, dt)
    eng = ArticulationEngine(emu.desc, 6, "cuda:0")
    assert eng.C == 0
    t = lambda a: torch.tensor(a.ravel(), device="cuda:0")
    q, qd, _, _ = eng.forward(t(q0), t(qd0), t(act), None, S, mm, dt, want_tape=False)
    assert rel(q.cpu().numpy(), eq) < 1e-5 and rel(qd.cpu().numpy(), eqd) < 1e-5


def _snu_case(N, seed=3):
    import torch
    d, model = load_golden("SNUHumanoidEnv")
    n0 = int(d["meta/num_envs"])
    emu = EmuSim(model, n0)
    Q, D, M = emu.desc.Q, emu.desc.D, emu.desc.M
    rng = np.random.default_rng(seed)
    p = "case%d/" % (int(d["meta/num_cases"]) - 1)
    pick = rng.integers(0, n0, N)
    t = lambda a: torch.tensor(np.ascontiguousarray(a, np.float32).ravel(), device="cuda:0")
    q0, qd0 = d[p + "q0"].reshape(n0, Q)[pick], d[p + "qd0"].reshape(n0, D)[pick]
    act = d[p + "act"].reshape(n0, D)[pick]
    musc = np.clip(d[p + "musc"].reshape(n0, M)[pick] * rng.uniform(0.5, 1.5, (N, M)), 0.0, 1.0)
    return d, emu, t(q0), t(qd0), t(act), t(musc)


def test_muscle_model_scatter_is_bit_reproducible():
    """152 muscles and 88 contact points scatter wrenches / cotangents into 11 bodies through the fixed-point
    accumulators (dfx_phases.h): integer sums do not depend on the order of the atomics, so forward AND
    backward results are bit-identical from run to run (and agree across group widths)."""
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    N = 64
    d, emu, q0, qd0, act, musc = _snu_case(N)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    eng = ArticulationEngine(emu.desc, N, "cuda:0")
    gq, gqd = torch.ones_like(q0), torch.ones_like(qd0)
    outs = []
    try:
        for grp in (32, 32, 16, 32):
            _capi.lib().dfx_set_group_size(grp)
            q, qd, tape, _ = eng.forward(q0, qd0, act, musc, S, mm, dt)
            g = eng.backward(act, musc, tape, gq, gqd, S, mm, dt)
            outs.append([x.clone() for x in (q, qd, tape) + tuple(g)])
    finally:
        _capi.lib().dfx_set_group_size(0)
    for other in (outs[1], outs[3]):
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)
    for a, b in zip(outs[0][:2] + outs[0][3:], outs[2][:2] + outs[2][3:]):   # 16 lanes: same sums, other lane mapping
        assert rel(b.cpu().numpy(), a.cpu().numpy()) < 5e-5
    assert all(torch.isfinite(x).all() for x in outs[0])


def test_non_finite_contribution_poisons_the_sum():
    """A NaN activation cannot be represented in the fixed-point accumulators: it must surface as NaN in the
    state of THAT environment (poison bit), never be dropped, and must not leak into its CTA neighbours."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    N = 8
    d, emu, q0, qd0, act, musc = _snu_case(N)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    eng = ArticulationEngine(emu.desc, N, "cuda:0")
    ref_q, ref_qd, _, _ = eng.forward(q0, qd0, act, musc, S, mm, dt, want_tape=False)
    bad = musc.clone().view(N, -1)
    bad[3, 17] = float("nan")
    q, qd, _, _ = eng.forward(q0, qd0, act, bad.reshape(-1), S, mm, dt, want_tape=False)
    qd, ref_qd = qd.view(N, -1), ref_qd.view(N, -1)
    assert torch.isnan(qd[3]).any()
    keep = [i for i in range(N) if i != 3]
    assert torch.equal(qd[keep], ref_qd[keep])
    huge = musc.clone().view(N, -1)
    huge[5, :] = 1.0e30                      # beyond the accumulator range: loud, not wrapped around
    q, qd, _, _ = eng.forward(q0, qd0, act, huge.reshape(-1), S, mm, dt, want_tape=False)
    assert not torch.isfinite(qd.view(N, -1)[5]).all()
    assert torch.equal(qd.view(N, -1)[[0, 1, 2, 4, 6, 7]], ref_qd[[0, 1, 2, 4, 6, 7]])


def test_launch_plan_keeps_a_full_wave_of_ant_resident():
    """4096 Ant environments fit one wave of CTAs on the device's SMs (132 on an H100 SXM; forward and adjoint): DESIGN.md
    section 4."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    d, emu, *_ = _case("AntEnv", 1)
    eng = ArticulationEngine(emu.desc, 1, "cuda:0")
    for bwd in (0, 1):
        out = (ctypes.c_int * 6)()
        assert eng.lib.dfx_launch_plan(eng.pack, bwd, out) == 0
        lanes, envs_per_cta, ctas_per_sm, smem, stride, pack = list(out)
        assert (lanes, envs_per_cta) == (32, 32)          # tile kernel: one CTA = 32 environments, lane = environment
        assert envs_per_cta * ctas_per_sm * sms >= 4096
        assert smem == pack + envs_per_cta * stride * 4 and (smem + 1024) * ctas_per_sm <= 227 * 1024


@pytest.mark.parametrize("name", ["AntEnv", "HopperEnv", "CheetahEnv", "CartPoleSwingUpEnv"])
def test_tile_and_lane_group_kernels_agree(name):
    """The small articulations run on the 32-environment tile kernels (dfx_tile.cu) by default; flag bit 5 keeps them
    on the lane-group kernels (dfx_kernels.cu).  Same phase code, different mapping: results agree to rounding of
    the contact / gather order, the tape has the same size up to tile padding, and N need not be a multiple of 32."""
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    N = 75
    d, emu, q0, qd0, act = _case(name, N, seed=5)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    t = lambda a: torch.tensor(a.ravel(), device="cuda:0")
    gq_out = torch.linspace(-1.0, 1.0, q0.size, device="cuda:0")
    gqd_out = torch.linspace(1.0, -1.0, qd0.size, device="cuda:0")
    res = []
    lib = _capi.lib()
    try:
        for flags in (9, 41):
            lib.dfx_set_flags(flags)
            eng = ArticulationEngine(emu.desc, N, "cuda:0")
            assert int(lib.dfx_pack_query(eng.pack, 9)) == (32 if flags == 9 else 0)
            q, qd, tape, _ = eng.forward(t(q0), t(qd0), t(act), None, S, mm, dt)
            g = eng.backward(t(act), None, tape, gq_out, gqd_out, S, mm, dt)
            res.append([q, qd, eng.tape_rows(tape, S)] + [x for x in g if x is not None])
    finally:
        lib.dfx_set_flags(9)
    for a, b in zip(*res):
        assert rel(a.cpu().numpy(), b.cpu().numpy()) < 2e-5


def test_ant_65536_envs_equal_their_64_env_pattern():
    """BASELINE.json configs[4] size on ONE device (2048 tiles, 1.7 GB of tape per env-step): 65 536 environments that
    repeat a 64-environment pattern give, environment by environment, the results of the 64-environment batch
    (64-bit tape offsets, tile padding, grid far beyond one wave)."""
    import torch
    from diffrl_b200.engine import ArticulationEngine
    d, emu, q0, qd0, act = _case("AntEnv", 64, seed=9)
    S, mm, dt = int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])
    t = lambda a: torch.tensor(np.ascontiguousarray(a).ravel(), device="cuda:0")
    small = ArticulationEngine(emu.desc, 64, "cuda:0")
    gq_s, gqd_s = torch.linspace(-1.0, 1.0, q0.size, device="cuda:0"), torch.linspace(1.0, -1.0, qd0.size, device="cuda:0")
    q, qd, tape, _ = small.forward(t(q0), t(qd0), t(act), None, S, mm, dt)
    g_small = small.backward(t(act), None, tape, gq_s, gqd_s, S, mm, dt)
    N, rep = 65536, 65536 // 64
    big = ArticulationEngine(emu.desc, N, "cuda:0")
    tile = lambda a: t(np.tile(a, (rep, 1)))
    Q, D = emu.desc.Q, emu.desc.D
    Q_, QD_, TP, _ = big.forward(tile(q0), tile(qd0), tile(act), None, S, mm, dt)
    assert TP.numel() == big.tape_floats(S, mm) and TP.numel() * 4 > 1.5e9
    assert torch.equal(Q_.view(rep, 64 * Q), q.view(1, -1).expand(rep, -1))
    assert torch.equal(QD_.view(rep, 64 * D), qd.view(1, -1).expand(rep, -1))
    G = big.backward(tile(act), None, TP, gq_s.view(64, Q).repeat(rep, 1).reshape(-1), gqd_s.view(64, D).repeat(rep, 1).reshape(-1), S, mm, dt)
    for a, b, w in zip(G[:3], g_small[:3], (Q, D, D)):
        ref = b.view(1, 64 * w).expand(rep, -1)
        assert (a.view(rep, 64 * w) - ref).abs().max() <= 2e-5 * ref.abs().max()


@pytest.mark.parametrize("name,width", [("HumanoidEnv", 8), ("SNUHumanoidEnv", 16)])
def test_launch_plan_keeps_sixteen_humanoids_per_sm(name, width):
    """The large articulations run on the compact scratch layouts (csrc/dfx_pack.h: mass-matrix temporaries overlaid on
    the per-substep temporaries, H^-1 read from the tape by the adjoint) so that 16 environments stay resident per SM,
    forward and adjoint: the Humanoid as two 8-environment CTAs that hide each other's barrier waits, the SNU model as
    one 16-environment CTA of 16 warps (its 152 muscles fill the item slots, DESIGN.md section 3)."""
    from diffrl_b200.engine import ArticulationEngine
    d, model = load_golden(name)
    eng = ArticulationEngine.from_model(model, "cuda:0", int(d["meta/num_envs"]))
    assert int(eng.lib.dfx_pack_query(eng.pack, 9)) == width
    for bwd in (0, 1):
        out = (ctypes.c_int * 6)()
        assert eng.lib.dfx_launch_plan(eng.pack, bwd, out) == 0
        lanes, envs_per_cta, ctas_per_sm, smem, stride, pack = list(out)
        assert envs_per_cta == width and envs_per_cta * ctas_per_sm >= 16, list(out)
        assert smem == pack + envs_per_cta * stride * 4 and (smem + 1024) * (16 // width) <= 227 * 1024
