"""The step and its adjoint on random articulations (tests/random_articulation.py), in the host emulation of every kernel
formulation, against the fp64 oracle -- per environment, per element (forward) and per gradient block (adjoint, against
the exact complex-step gradient).  The six DiffRL articulations are the only trees the golden tests step; these models
exercise the tree data of dfx_pack_build.h (parents in non-depth-first order, chains, subtree and path lists, contacts
grouped by body, muscle groups) on other shapes: size twins of the six, and generic models with every joint type, fixed /
planar / free roots, a forest, L up to 40 and D > 32.

The formulations (tests/emu_util.py build flags):
  group    es = 1: the lane-group kernels' level-by-level tree recursions;
  tile32   es = 32, path passes: the 32-environment tile kernels' strided scratch and path / subtree passes;
  tile8m1  es = 8, path passes, layout mode 1 (compact scratch);
  tile8m3  es = 8, path passes, layout mode 3 (compact scratch, global H^-1);
  fused    es = 8, path passes, layout mode 3, -DDFX_EMU_FUSED_PHASES=1 (the merged phases of the tile kernels);
  fma      es = 1 with FMA contraction, as nvcc compiles the kernels (the other builds keep -ffp-contract=off).  Some
           environments' errors are several times larger with contraction than without (the Hopper twin's (1, 1) action
           gradients among them), and the kernels contract.

The worst error per block over the formulations is what tolerances.RANDOM_GRAD_MEASURED records; the GPU test
(tests/test_gpu_random_articulations.py) holds the kernels to EXACT_GRAD_FACTOR times it."""
import ctypes

import numpy as np
import pytest

from emu_util import EmuSim, build_emu
import exact_util as X
from parity_util import check_forward_against
import random_articulation as R
from tolerances import RANDOM_GRAD_MEASURED, RANDOM_SAMPLE, fwd_rtol, random_grad_tol

N = 75
FORMULATIONS = {
    "group": dict(),
    "tile32": dict(es=32, path_passes=True),
    "tile8m1": dict(es=8, path_passes=True, layout_mode=1),
    "tile8m3": dict(es=8, path_passes=True, layout_mode=3),
    "fused": dict(es=8, path_passes=True, layout_mode=3, extra=("-DDFX_EMU_FUSED_PHASES=1",)),
    "fma": dict(extra=("-ffp-contract=fast", "-mfma")),
}
MODELS = ["twin_" + n for n in R.TWINS] + ["gen_" + k for k in R.GENERIC]


def model(name):
    return R.twin(name[len("twin_"):]) if name.startswith("twin_") else R.generic(name[len("gen_"):])


def batch(rm):
    return R.make_batch(rm, N, RANDOM_SAMPLE.get(rm.name, N), seed=1)


def oracle_forward_one(o, inp, S, mm, dt):
    """forward_one of parity_util.check_forward_against: the f64 oracle from a (perturbed) state of environment i"""
    def f(i, qi, qdi):
        m = None if inp["musc"] is None else inp["musc"][i:i + 1]
        return o.forward(qi[None], qdi[None], inp["act"][i:i + 1], m, S, mm, dt, "f64")
    return f


def check_forward(what, name, o, inp, q, qd, S, mm, dt):
    """per environment and element against the f64 oracle, with parity_util's conditioning rule"""
    desc = o.desc
    oq, oqd = o.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt, "f64")
    return check_forward_against(oracle_forward_one(o, inp, S, mm, dt), q, qd, oq, oqd, inp["q0"], inp["qd0"], desc.Q, desc.D,
                                 fwd_rtol(name), what)


@pytest.mark.parametrize("name", MODELS)
def test_random_batch_visits_every_branch(name):
    rm = model(name)
    o = R.oracle(rm)
    desc, inp, idx = batch(rm)
    sub = {k: (None if v is None else v[idx]) for k, v in inp.items()}
    for S, mm in rm.patterns():
        cov = X.branch_coverage(o, sub, S, mm, rm.pattern_dt(S))
        missing = [b for b in X.branches_of_model(desc) if cov[b] == 0]
        assert not missing, (name, (S, mm), cov)


@pytest.mark.parametrize("name", MODELS)
def test_emulated_step_matches_oracle_on_random_articulation(name):
    rm = model(name)
    o = R.oracle(rm)
    desc, inp, idx = batch(rm)
    worst = {}
    for form, flags in FORMULATIONS.items():
        emu = EmuSim(rm.model, 1, **flags)
        emu.N = N
        for S, mm in rm.patterns():
            dt = rm.pattern_dt(S)
            what = "%s %s (%d, %d)" % (name, form, S, mm)
            q, qd, tape, _ = emu.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt)
            check_forward(what, rm.name, o, inp, q, qd, S, mm, dt)
            g = emu.backward(inp["act"], inp["musc"], tape, inp["gq_out"], inp["gqd_out"], S, mm, dt)
            got = [x.reshape(N, -1)[idx] for x in g if x is not None]
            ex = R.exact_gradients(rm, inp, idx, S, mm, dt)
            w, _ = X.check_against_exact(what, o, inp, idx, got, ex, random_grad_tol(rm.name, S), S, mm, dt,
                                         max_excluded=max(2, len(idx) // 20))
            for b, v in w.items():
                key = (b, "1x1" if S == 1 else "multi")
                worst[key] = max(worst.get(key, 0.0), v)
    print(name, "worst over formulations and patterns:", {"%s/%s" % k: "%.1e" % v for k, v in sorted(worst.items())})
    for (b, kind), v in worst.items():
        assert v <= RANDOM_GRAD_MEASURED[rm.name][b][0 if kind == "multi" else 1], (name, b, kind, v)


# ------------------------------------------------------------------ dfx_pack_create's refusals (the same build_pack)
def _create(model_dict):
    from diffrl_b200.modelpack import articulation_from_model
    lib = build_emu()
    desc, _ = articulation_from_model(model_dict, 1)
    err = ctypes.create_string_buffer(256)
    st = desc.as_struct()
    pack = lib.emu_pack_create(ctypes.byref(st), err, 256)
    if pack:
        lib.emu_pack_destroy(pack)
    return pack, err.value.decode()


def _edited(**fields):
    m = dict(R.generic("mixed").model)
    for k, v in fields.items():
        m[k] = v
    return m


def test_pack_create_accepts_the_random_models():
    for rm in R.all_models():
        pack, msg = _create(rm.model)
        assert pack, (rm.name, msg)


def test_pack_create_rejects_child_before_parent():
    m = R.generic("mixed").model
    parent = m["joint_parent"].copy()
    k = int(np.nonzero(parent > 0)[0][0])
    parent[k] = k + 1                                    # a child listed before its parent
    pack, msg = _create(_edited(joint_parent=parent))
    assert not pack and msg == "link %d: parent %d must precede it" % (k, k + 1), msg


def test_pack_create_rejects_unknown_joint_type():
    m = R.generic("mixed").model
    t = m["joint_type"].copy()
    k = int(np.nonzero(t == R.REVOLUTE)[0][0])
    t[k] = 7
    pack, msg = _create(_edited(joint_type=t))
    assert not pack and msg == "link %d: unknown joint type 7" % k, msg


def test_pack_create_rejects_contact_on_out_of_range_body():
    m = R.generic("mixed").model
    for bad in (len(m["joint_type"]), -1):
        body = m["contact_body0"].copy()
        body[3] = bad
        pack, msg = _create(_edited(contact_body0=body))
        assert not pack and msg == "contact_body0 out of range (expected env-local link index)", (bad, msg)
