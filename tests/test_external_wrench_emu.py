"""External link wrenches (include/dfx.h DfxExternalWrench) in the host emulation of every kernel formulation, against the fp64
oracle (tests/wrench_oracle/wrench_oracle.c: oracle/dflex_oracle.c with the wrench applied).

  * the oracle's complex-step wrench gradient equals fp64 central differences of its own forward;
  * the six emulated formulations (as tests/test_random_articulations_emu.py: lane group, tile32, tile8 layouts 1 and 3, fused
    phases, FMA contraction) agree with the oracle on random wrenches, per block -- q', qd' and gq, gqd, gact, g_f_ext -- within
    wrench_util.wrench_tol (4x the measured emulation error, never below 1e-6);
  * a zero wrench steps bit for bit as the step without one (state, tape and cotangents)."""
import numpy as np
import pytest

import wrench_util as W
from wrench_util import WrenchEmuSim, WrenchOracle, wrench_tol

FORMULATIONS = {
    "group": dict(),
    "tile32": dict(es=32, path_passes=True),
    "tile8m1": dict(es=8, path_passes=True, layout_mode=1),
    "tile8m3": dict(es=8, path_passes=True, layout_mode=3),
    "fused": dict(es=8, path_passes=True, layout_mode=3, extra=("-DDFX_EMU_FUSED_PHASES=1",)),
    "fma": dict(extra=("-ffp-contract=fast", "-mfma")),
}


def _emu(model, meta, flags):
    emu = WrenchEmuSim(model, meta["num_envs"], **flags)
    emu.N = W.N
    return emu


def test_oracle_wrench_gradient_matches_central_differences():
    model, meta, inp = W.golden_batch("AntEnv")
    o = WrenchOracle.from_model(model, meta["num_envs"])
    f = W.random_wrench(model, meta["num_envs"], W.N, 7).astype(np.float64)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    e = 0
    g = o.exact_gradient_ext(inp["q0"][e], inp["qd0"][e], inp["act"][e], None, f[e], inp["gq_out"][e], inp["gqd_out"][e], S, mm, dt)[4]

    def loss(fe):
        q, qd = o.forward_ext(inp["q0"][e:e + 1], inp["qd0"][e:e + 1], inp["act"][e:e + 1], None, fe[None], S, mm, dt)
        return float(np.dot(q.ravel(), inp["gq_out"][e].astype(np.float64)) + np.dot(qd.ravel(), inp["gqd_out"][e].astype(np.float64)))
    fd = np.zeros_like(g)
    for idx in np.ndindex(*g.shape):
        h = 1e-6 * (1.0 + abs(f[e][idx]))
        fp, fm = f[e].copy(), f[e].copy()
        fp[idx] += h
        fm[idx] -= h
        fd[idx] = (loss(fp) - loss(fm)) / (2 * h)
    assert np.abs(fd).max() > 0
    assert W.rel_err(g, fd) < 1e-6, W.rel_err(g, fd)


@pytest.mark.parametrize("name", W.ENVS)
def test_emulated_wrench_matches_oracle(name):
    model, meta, inp = W.golden_batch(name)
    o = WrenchOracle.from_model(model, meta["num_envs"])
    f = W.random_wrench(model, meta["num_envs"], W.N, 7)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    for form, flags in FORMULATIONS.items():
        emu = _emu(model, meta, flags)
        q, qd, tape, _ = emu.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt, f_ext=f)
        g = emu.backward(inp["act"], inp["musc"], tape, inp["gq_out"], inp["gqd_out"], S, mm, dt, f_ext=f)
        err = W.oracle_errors(o, inp, f.astype(np.float64), q, qd, (g[0], g[1], g[2], g[4]), meta)
        for block, v in err.items():
            assert v <= wrench_tol(name, block), (name, form, block, v, wrench_tol(name, block))


@pytest.mark.parametrize("name", W.ENVS)
def test_zero_wrench_is_the_plain_step_bit_for_bit(name):
    model, meta, inp = W.golden_batch(name)
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    zero = np.zeros_like(W.random_wrench(model, meta["num_envs"], W.N, 7))
    for form, flags in FORMULATIONS.items():
        emu = _emu(model, meta, flags)
        a = emu.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt)
        b = emu.forward(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt, f_ext=zero)
        for x, y in zip(a[:3], b[:3]):
            assert np.array_equal(x, y), (name, form)
        ga = emu.backward(inp["act"], inp["musc"], a[2], inp["gq_out"], inp["gqd_out"], S, mm, dt)
        gb = emu.backward(inp["act"], inp["musc"], b[2], inp["gq_out"], inp["gqd_out"], S, mm, dt, f_ext=zero)
        for x, y in zip(ga, gb[:4]):
            assert (x is None and y is None) or np.array_equal(x, y), (name, form)
