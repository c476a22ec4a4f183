"""The CUDA step and its adjoint on random articulations (tests/random_articulation.py) against the fp64 oracle, on every kernel
family that exists for each model: N = 75 environments (a partial last tile), the patterns of RandomModel.patterns().

* forward: per environment and element against the f64 oracle (parity_util.check_forward_against's conditioning rule);
* adjoint: per environment and gradient block against the exact complex-step gradient (exact_util.check_against_exact),
  bound EXACT_GRAD_FACTOR x the host emulation's measured error (tolerances.RANDOM_GRAD_MEASURED), never below
  EXACT_GRAD_FLOOR; only environments on a switching surface may be excluded;
* size twins run on the tile kernel and the lane-group specialisation of the articulation they copy (and, with flag bit 4,
  on the run-time-generic lane-group instantiation); their recompute adjoint equals tape mode bit for bit; their bf16-tape
  adjoint meets the same rule against the host emulation of the same bf16 rounding;
* a random tree built through the public dflex API (ModelBuilder, SemiImplicitIntegrator under autograd) against the oracle
  built from the same finalized Model.

Prints, per model and family, the kernel that ran, the worst ratio of error to bound and the exclusions."""
import ctypes

import numpy as np
import pytest

import exact_util as X
import random_articulation as R
from emu_util import build_emu, load_golden
from test_random_articulations_emu import MODELS, batch, check_forward, model
from emu_util import EmuSim
from tolerances import (BF16_TAPE_ACTION_GRAD_RTOL, BF16_TAPE_STATE_GRAD_RTOL, BF16_TAPE_STATE_GRAD_RTOL_DEFAULT,
                        EXACT_GRAD_FACTOR, EXACT_GRAD_FLOOR, random_grad_tol)

pytestmark = pytest.mark.gpu

N = 75
VARIANTS = ["auto", "tile8", "tile16", "tile32", "group8", "group16", "group32", "group8g", "group16g", "group32g"]
SPECIAL_GROUP = {"AntEnv": 16, "CartPoleSwingUpEnv": 16, "HopperEnv": 16, "CheetahEnv": 16, "HumanoidEnv": 32,
                 "SNUHumanoidEnv": 32}     # dfx_kernels.cu launch(): the lane-group width of each DFX_SPECIAL instantiation


def _select(variant):
    """test_gpu_golden._select, plus 'groupNg': lane groups of N forced onto the generic <0,0,0,0,0> instantiation (flag 4)"""
    from test_gpu_golden import _select as select
    from diffrl_b200 import _capi
    select(variant.rstrip("g"))
    if variant.endswith("g"):
        _capi.lib().dfx_set_flags(9 | 32 | 4)


def _t(a):
    import torch
    return None if a is None else torch.tensor(np.ascontiguousarray(a).ravel(), device="cuda:0")


def _kernel(eng, lib, rm, variant):
    tile = int(lib.dfx_pack_query(eng.pack, 9))
    if tile:
        return "tile%d" % tile
    plan = (ctypes.c_int * 6)()
    lib.dfx_launch_plan(eng.pack, 0, plan)
    special = rm.twin_of is not None and not variant.endswith("g") and SPECIAL_GROUP[rm.twin_of] == plan[0]
    # (inferred from the sizes, the flags and the group width, as launch() in dfx_kernels.cu dispatches: not queried)
    return "group%d %s" % (plan[0], "specialised (by dispatch rule)" if special else "generic")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", MODELS)
def test_cuda_step_matches_oracle_on_random_articulation(name, variant):
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    rm = model(name)
    if variant.endswith("g") and rm.twin_of is None:
        pytest.skip("a generic model runs on the generic instantiation in every group variant")
    o = R.oracle(rm)
    desc, inp, idx = batch(rm)
    lib = _capi.lib()
    _select(variant)
    try:
        eng = ArticulationEngine(desc, N, "cuda:0")
        tile = int(lib.dfx_pack_query(eng.pack, 9))
        if variant.startswith("tile") and tile != int(variant[4:]):
            pytest.skip("no %s-environment tile kernel for %s" % (variant[4:], name))
        if variant != "auto":
            assert (tile == 0) == variant.startswith("group")
        if rm.twin_of is None:
            assert tile == 0, (name, "a generic model must not select a tile kernel", tile)
        else:
            # the twin runs on the kernel of the articulation it copies
            _, gm = load_golden(rm.twin_of)
            ref = ArticulationEngine.from_model(gm, "cuda:0", int(load_golden(rm.twin_of)[0]["meta/num_envs"]))
            assert int(lib.dfx_pack_query(ref.pack, 9)) == tile, (name, variant)
            if variant == "auto":
                assert tile != 0, (name, "the twin must run on its model's tile kernel")
        kernel = _kernel(eng, lib, rm, variant)
        ratio, excluded_all = 0.0, []
        for S, mm in rm.patterns():
            dt = rm.pattern_dt(S)
            what = "%s %s (%d, %d)" % (name, variant, S, mm)
            q, qd, tape, _ = eng.forward(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), S, mm, dt)
            check_forward(what, rm.name, o, inp, q.cpu().numpy().reshape(N, -1), qd.cpu().numpy().reshape(N, -1), S, mm, dt)
            g = eng.backward(_t(inp["act"]), _t(inp["musc"]), tape, _t(inp["gq_out"]), _t(inp["gqd_out"]), S, mm, dt)
            got = [x.cpu().numpy().reshape(N, -1)[idx] for x in g if x is not None]
            ex = R.exact_gradients(rm, inp, idx, S, mm, dt)
            tol = random_grad_tol(rm.name, S)
            worst, excluded = X.check_against_exact(what, o, inp, idx, got, ex, tol, S, mm, dt,
                                                    max_excluded=max(2, len(idx) // 20))
            ratio = max(ratio, max(v / tol[b] for b, v in worst.items()))
            excluded_all += [(S, mm, e) for e in excluded]
            if rm.twin_of is not None:
                # recompute mode (the fused recompute launch's bulk copies follow the row layout): the same bound
                gr = eng.backward_recompute(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), _t(inp["gq_out"]),
                                            _t(inp["gqd_out"]), S, mm, dt)
                for a, b in zip(g, gr):
                    assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), (what, "recompute differs from tape mode")
        print("%s %s: kernel %s, worst error / bound %.2f, %d exclusion(s) %s" % (name, variant, kernel, ratio, len(excluded_all),
                                                                                  excluded_all))
    finally:
        _select("auto")


@pytest.mark.parametrize("twin_of", R.TWINS)
def test_bf16_tape_on_twins(twin_of):
    """bf16 tape (tile kernels only): the forward is bit-identical to the fp32-tape run, and each gradient's error against the
    exact gradient (relative to its largest component over the sampled environments) is at most EXACT_GRAD_FACTOR times the
    error of the host emulation of the same bf16 rounding (EmuSim.tape_bf16) -- the rule the fp32 adjoint is held to.
    Printed beside it: the BF16_TAPE_* tolerances, measured on the DiffRL models' own states, do not bound every twin's
    batch -- the emulation itself moves the Hopper twin's state gradients by 4.8e-2 through the bf16 tape."""
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    rm = R.twin(twin_of)
    desc, inp, idx = batch(rm)
    lib = _capi.lib()
    S, mm = rm.S, rm.mm
    dt = rm.pattern_dt(S)
    eng32 = ArticulationEngine(desc, N, "cuda:0")
    lib.dfx_set_tape_dtype(1)
    try:
        eng = ArticulationEngine(desc, N, "cuda:0")
    finally:
        lib.dfx_set_tape_dtype(0)
    assert eng.tape_bf16 and int(lib.dfx_pack_query(eng.pack, 9)) == int(lib.dfx_pack_query(eng32.pack, 9)) != 0
    q32, qd32, _, _ = eng32.forward(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), S, mm, dt)
    q, qd, tape, _ = eng.forward(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), S, mm, dt)
    assert torch.equal(q, q32) and torch.equal(qd, qd32)
    g = [x.cpu().numpy().reshape(N, -1)[idx] for x in eng.backward(_t(inp["act"]), _t(inp["musc"]), tape, _t(inp["gq_out"]),
                                                                   _t(inp["gqd_out"]), S, mm, dt) if x is not None]
    emu = EmuSim(rm.model, 1, es=8, path_passes=True)
    emu.N = N
    emu.tape_bf16 = True
    _, _, etape, _ = emu.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt)
    ge = [x.reshape(N, -1)[idx] for x in emu.backward(inp["act"], inp["musc"], etape, inp["gq_out"], inp["gqd_out"], S, mm, dt)
          if x is not None]
    ex = R.exact_gradients(rm, inp, idx, S, mm, dt)
    rel = lambda a, b: float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())
    err, emu_err = [rel(a, x) for a, x in zip(g, ex)], [rel(a, x) for a, x in zip(ge, ex)]
    within = (max(err[:2]) <= BF16_TAPE_STATE_GRAD_RTOL.get(twin_of, BF16_TAPE_STATE_GRAD_RTOL_DEFAULT)
              and err[2] <= BF16_TAPE_ACTION_GRAD_RTOL)
    print("%s bf16 tape against the exact gradient: kernel %s, emulation %s; within BF16_TAPE_*: %s" % (
        rm.name, ["%.1e" % e for e in err], ["%.1e" % e for e in emu_err], within))
    for k, (e, m) in enumerate(zip(err, emu_err)):
        assert e <= max(EXACT_GRAD_FLOOR, EXACT_GRAD_FACTOR * m), (rm.name, k, e, m)


@pytest.mark.parametrize("variant", ["auto", "tile8", "tile16", "tile32"])
@pytest.mark.parametrize("twin_of", R.TWINS)
def test_recomputed_tape_equals_stored_tape_on_twins(twin_of, variant):
    """The fused recompute tile kernel re-runs the forward inside the adjoint launch: on the twins -- frames that are not
    axis-aligned -- its rows, H^-1 blocks, end state and cotangents equal tape mode's bit for bit.  (The joint-local transforms
    are formed with explicitly rounded products, dfx_math.h xf_mul_rn: left to the compiler's FMA contraction they differed
    between the two kernels in the last bits from the second substep on.)"""
    import torch
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    rm = R.twin(twin_of)
    desc, inp, _ = batch(rm)
    lib = _capi.lib()
    _select(variant)
    try:
        eng = ArticulationEngine(desc, N, "cuda:0")
        tile = int(lib.dfx_pack_query(eng.pack, 9))
        if variant != "auto" and tile != int(variant[4:]):
            pytest.skip("no %s-environment tile kernel for %s" % (variant[4:], twin_of))
        for S, mm in rm.patterns():
            dt = rm.pattern_dt(S)
            q, qd, tape, _ = eng.forward(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), S, mm, dt)
            g = eng.backward(_t(inp["act"]), _t(inp["musc"]), tape, _t(inp["gq_out"]), _t(inp["gqd_out"]), S, mm, dt)
            ws = eng.recompute_workspace(S, mm)
            ws.fill_(float("nan"))
            gr = eng.backward_recompute(_t(inp["q0"]), _t(inp["qd0"]), _t(inp["act"]), _t(inp["musc"]), _t(inp["gq_out"]),
                                        _t(inp["gqd_out"]), S, mm, dt, workspace=ws)
            cfg = (rm.name, variant, tile, S, mm)
            assert torch.equal(eng.tape_rows(ws, S), eng.tape_rows(tape, S)), cfg
            assert torch.equal(eng.tape_hinv(ws, S, mm), eng.tape_hinv(tape, S, mm)), cfg
            q_end, qd_end = eng.workspace_end_state(ws, S, mm)
            assert torch.equal(q_end, q) and torch.equal(qd_end, qd), cfg
            for a, b in zip(g, gr):
                assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), cfg
    finally:
        _select("auto")


# ------------------------------------------------------------------ an articulation whose scratch cannot fit shared memory
def _chain(L):
    rng = np.random.default_rng(5)
    return R._build(rng, [R.FREE] + [R.REVOLUTE] * (L - 1), list(range(-1, L - 1)), [L - 1] * 4)


def _scratch_floats(L):
    """max(forward, backward) floats of per-environment scratch of the chain of L links, from the host emulation's pack"""
    from diffrl_b200.modelpack import articulation_from_model
    lib = build_emu()
    desc, _ = articulation_from_model(_chain(L), 1)
    st = desc.as_struct()
    err = ctypes.create_string_buffer(256)
    pack = lib.emu_pack_create(ctypes.byref(st), err, 256)
    assert pack, err.value
    try:
        return max(lib.emu_pack_query(pack, 5), lib.emu_pack_query(pack, 6))   # DFX_QUERY_{FWD,BWD}_SCRATCH_FLOATS
    finally:
        lib.emu_pack_destroy(pack)


def test_engine_refuses_articulation_whose_scratch_exceeds_shared_memory():
    """A chain whose scratch alone exceeds 227 KB (sized on the host emulation's pack) raises a DfxError that names the cause
    when the engine is built, instead of a launch failing with cudaErrorInvalidConfiguration.  Walking down 4 links at a time
    (the pack, which grows with L^2, shares the budget): the first chain that fits steps normally, and the one 4 links longer,
    just over the limit, is refused."""
    from diffrl_b200 import _capi
    from diffrl_b200.engine import ArticulationEngine
    from diffrl_b200.modelpack import articulation_from_model
    L = 64
    while _scratch_floats(L) * 4 + 1024 <= 227 * 1024:
        L += 1
    def build(L):
        desc, _ = articulation_from_model(_chain(L), 1)
        try:
            return ArticulationEngine(desc, 4, "cuda:0"), None
        except _capi.DfxError as e:
            return None, str(e)

    eng, msg = build(L)
    assert eng is None, ("a chain whose scratch alone exceeds 227 KB must be refused", L)
    while eng is None:
        assert "too large for the step kernels: the" in msg and "227 KB of one CTA" in msg, msg
        refused, L = L, L - 4
        eng, msg = build(L)
    assert build(refused)[0] is None and eng is not None, (refused, L)
    rm = R.RandomModel("chain", _chain(L), 2, 2, None, [])
    print("chain of %d links refused, %d links fit" % (refused, L))
    rng = np.random.default_rng(0)
    q = np.stack([R.random_state(rm, rng, 0.5)[0] for _ in range(4)])
    qd = np.zeros((4, eng.D), np.float32)
    act = np.zeros((4, eng.D), np.float32)
    qo, qdo, tape, _ = eng.forward(_t(q), _t(qd), _t(act), None, 2, 2, 2 * R.DT_SUB)
    gq_out, gqd_out = np.ones((4, eng.Q), np.float32), np.ones((4, eng.D), np.float32)
    g = eng.backward(_t(act), None, tape, _t(gq_out), _t(gqd_out), 2, 2, 2 * R.DT_SUB)
    o = R.oracle(rm)
    oq, _ = o.forward(q, qd, act, None, 2, 2, 2 * R.DT_SUB, "f64")
    assert np.abs(qo.cpu().numpy() - oq).max() <= 1e-4 * np.abs(oq).max()
    # the adjoint of environment 0 per block against the exact gradient, within EXACT_GRAD_FACTOR x the host emulation's
    # error on the same input, the larger of its builds without and with FMA contraction (the rule of the other models)
    ex = [x[None] for x in o.exact_gradient(q[0], qd[0], act[0], None, gq_out[0], gqd_out[0], 2, 2, 2 * R.DT_SUB) if x is not None]
    emu_err = {}
    for extra in ((), ("-ffp-contract=fast", "-mfma")):
        emu = EmuSim(rm.model, 1, extra=extra)
        _, _, etape, _ = emu.forward(q[0], qd[0], act[0], None, 2, 2, 2 * R.DT_SUB)
        ge = [x[None] for x in emu.backward(act[0], None, etape, gq_out[0], gqd_out[0], 2, 2, 2 * R.DT_SUB) if x is not None]
        for b, e in X.block_errors(o.desc, ge, ex).items():
            emu_err[b] = max(emu_err.get(b, 0.0), float(e[0]))
    err = X.block_errors(o.desc, [x.cpu().numpy().reshape(4, -1)[:1] for x in g if x is not None], ex)
    for b in err:
        assert err[b][0] <= max(EXACT_GRAD_FLOOR, EXACT_GRAD_FACTOR * emu_err[b]), (b, err[b][0], emu_err[b])


# ------------------------------------------------------------------ one random tree through the public dflex API
def test_model_builder_random_tree_through_public_api():
    """A random tree built with dflex.sim.ModelBuilder (random_articulation.builder_model), stepped with
    SemiImplicitIntegrator.forward under autograd: q', qd' against the f64 oracle built from the same finalized Model
    (parity_util's rule), and the gradient of a scalar loss per block against the exact gradient, within EXACT_GRAD_FACTOR x
    the host emulation's error on the same input (never below EXACT_GRAD_FLOOR)."""
    import torch
    import dflex as df
    S, mm, dt = 16, 4, 1.0 / 60.0
    model, (q, qd, act) = R.builder_model("cuda:0")
    o = R.Oracle.from_model(model, 1)
    desc = o.desc
    rng = np.random.default_rng(1)
    wq, wqd = rng.standard_normal(desc.Q).astype(np.float32), rng.standard_normal(desc.D).astype(np.float32)
    state = model.state()
    state.joint_q = torch.tensor(q, device="cuda:0", requires_grad=True)
    state.joint_qd = torch.tensor(qd, device="cuda:0", requires_grad=True)
    state.joint_act = torch.tensor(act, device="cuda:0", requires_grad=True)
    out = df.sim.SemiImplicitIntegrator().forward(model, state, dt, S, mm)
    loss = (out.joint_q * torch.tensor(wq, device="cuda:0")).sum() + (out.joint_qd * torch.tensor(wqd, device="cuda:0")).sum()
    loss.backward()
    inp = dict(q0=q[None], qd0=qd[None], act=act[None], musc=None)
    check_forward("ModelBuilder tree", "builder", o, inp, out.joint_q.detach().cpu().numpy()[None],
                  out.joint_qd.detach().cpu().numpy()[None], S, mm, dt)
    got = [x.grad.cpu().numpy()[None] for x in (state.joint_q, state.joint_qd, state.joint_act)]
    ex = [x[None] for x in o.exact_gradient(q, qd, act, None, wq, wqd, S, mm, dt) if x is not None]
    emu = EmuSim(model, 1)
    _, _, tape, _ = emu.forward(q, qd, act, None, S, mm, dt)
    ge = [x[None] for x in emu.backward(act, None, tape, wq, wqd, S, mm, dt) if x is not None]
    emu_err = X.block_errors(desc, ge, ex)
    tol = {b: max(EXACT_GRAD_FLOOR, EXACT_GRAD_FACTOR * float(e[0])) for b, e in emu_err.items()}
    inp.update(gq_out=wq[None], gqd_out=wqd[None])
    worst, _ = X.check_against_exact("ModelBuilder tree", o, inp, np.array([0]), got, ex, tol, S, mm, dt, max_excluded=0)
    print("ModelBuilder tree: L=%d D=%d C=%d, worst error / bound %.2f" % (desc.L, desc.D, desc.C, max(worst[b] / tol[b] for b in tol)))
