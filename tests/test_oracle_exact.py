"""The exact gradient reference (complex-step build of the C oracle, liboracle_c64.so) and the step adjoint's math against it,
on the CPU:
* the real part of the complex forward is the fp64 forward;
* the complex-step gradient is the derivative of the fp64 forward: it equals fp64 central differences wherever those are
  trustworthy;
* the reference's own stored fp32 gradients lie within the per-block floor recorded in tests/tolerances.py;
* the host emulation of this project's adjoint (the same dfx_phases.h / dfx_step.h the kernels compile) holds every
  environment and every gradient block to the bound the GPU kernels are held to (tests/test_gpu_exact_adjoint.py), on the
  golden states + noise and on explicit pushes into every branch of the contact and limit model, for every H-refresh
  pattern of exact_util.patterns."""
import numpy as np
import pytest

from conftest import ENVS
from emu_util import EmuSim, load_golden
import exact_util as X
from tolerances import EXACT_GRAD_MEASURED, EXACT_SAMPLE, exact_grad_tol


def _golden_inputs(name, k):
    d, _ = load_golden(name)
    n0 = int(d["meta/num_envs"])
    o = X._oracle(name)
    Q, D, M = o.desc.Q, o.desc.D, o.desc.M
    p = "case%d/" % k
    return dict(q0=d[p + "q0"].reshape(n0, Q), qd0=d[p + "qd0"].reshape(n0, D), act=d[p + "act"].reshape(n0, D),
                musc=d[p + "musc"].reshape(n0, M) if M else None, gq_out=d[p + "gq_out"].reshape(n0, Q),
                gqd_out=d[p + "gqd_out"].reshape(n0, D))


def _batch(name):
    return X.make_batch(name, 75, EXACT_SAMPLE[name], seed=1)


@pytest.mark.parametrize("name", ENVS)
def test_complex_forward_real_part_equals_f64(name):
    o = X._oracle(name)
    _, inp, idx = _batch(name)
    for S, mm in X.patterns(name)[:2]:
        dt = X.pattern_dt(name, S)
        m = None if inp["musc"] is None else inp["musc"][idx]
        a = o.forward(inp["q0"][idx], inp["qd0"][idx], inp["act"][idx], m, S, mm, dt, precision="f64")
        c = o.forward(inp["q0"][idx], inp["qd0"][idx], inp["act"][idx], m, S, mm, dt, precision="c64")
        for x, y in zip(a, c):
            assert np.abs(x - y).max() <= 1e-13 * np.abs(x).max(), (name, S, mm)


def _fd_trustworthy(o, q, qd, act, musc, S, mm, dt, eps):
    """the f64 branch signature is the same at every +-h of the central differences (h = eps (1 + |x|), the step of
    oracle_fd_gradient), for the state inputs q and qd"""
    h0, _ = o.branches(q[None], qd[None], act[None], None if musc is None else musc[None], S, mm, dt, "f64")
    rows_q, rows_qd = [], []
    for vec, width in ((0, q.size), (1, qd.size)):
        for i in range(width):
            for s in (1.0, -1.0):
                pq, pqd = q.astype(np.float64), qd.astype(np.float64)
                x = pq if vec == 0 else pqd
                x[i] += s * eps * (1.0 + abs(x[i]))
                rows_q.append(pq); rows_qd.append(pqd)
    n = len(rows_q)
    hp, _ = o.branches(np.array(rows_q), np.array(rows_qd), np.repeat(act[None], n, 0),
                       None if musc is None else np.repeat(musc[None], n, 0), S, mm, dt, "f64")
    return bool((hp == h0[0]).all())


@pytest.mark.parametrize("name", ENVS)
def test_exact_gradient_matches_fp64_finite_differences(name):
    """On every environment where central differences are trustworthy (no branch switch within +-h, and FD at eps and
    eps/4 agree to 1e-7), the complex-step gradient equals them to 1e-6 of its largest component.  At most 3 of the 10-12
    environments may be untrustworthy (SNU's golden case 0 starts at reset, with contact points exactly on the ground)."""
    o = X._oracle(name)
    S, mm, dt = X.config(name)
    _, inp, idx = _batch(name)
    envs = [("golden case %d" % k, _golden_inputs(name, k), e) for k in range(int(load_golden(name)[0]["meta/num_cases"])) for e in range(2)]
    envs += [("batch", inp, int(i)) for i in idx[np.linspace(0, len(idx) - 1, 6).round().astype(np.int64)]]
    untrusted = []
    for what, g, e in envs:
        m = None if g["musc"] is None else g["musc"][e]
        args = (g["q0"][e], g["qd0"][e], g["act"][e], m, g["gq_out"][e], g["gqd_out"][e], S, mm, dt)
        ex = np.concatenate([x for x in o.exact_gradient(*args) if x is not None])
        fd = np.concatenate([x for x in o.fd_gradient(*args, eps=1e-6) if x is not None])
        fd4 = np.concatenate([x for x in o.fd_gradient(*args, eps=0.25e-6) if x is not None])
        if np.abs(fd - fd4).max() > 1e-7 * np.abs(fd).max() or not _fd_trustworthy(o, g["q0"][e], g["qd0"][e], g["act"][e], m, S, mm, dt, 1e-6):
            untrusted.append((what, e))
            continue
        err = np.abs(ex - fd).max() / np.abs(ex).max()
        assert err <= 1e-6, (name, what, e, err)
    assert len(untrusted) <= 3, (name, untrusted)


@pytest.mark.parametrize("name", ENVS)
def test_reference_fp32_gradients_within_recorded_floor(name):
    """The reference's own fp32 gradients (tests/golden) against the exact gradient, per block: the 'ref' column of
    tolerances.EXACT_GRAD_MEASURED, which is what it measures."""
    o = X._oracle(name)
    d, _ = load_golden(name)
    S, mm, dt = X.config(name)
    worst = {}
    for k in range(int(d["meta/num_cases"])):
        g = _golden_inputs(name, k)
        p = "case%d/" % k
        n0 = g["q0"].shape[0]
        ex = X.exact_gradients(name, g, np.arange(n0), S, mm, dt)
        got = [d[p + "grad_q"].reshape(n0, -1), d[p + "grad_qd"].reshape(n0, -1), d[p + "grad_act"].reshape(n0, -1)]
        if g["musc"] is not None:
            got.append(d[p + "grad_musc"].reshape(n0, -1))
        for b, e in X.block_errors(o.desc, got, ex).items():
            worst[b] = max(worst.get(b, 0.0), float(e.max()))
    print(name, "reference fp32 vs exact, per block:", {b: "%.1e" % v for b, v in worst.items()})
    for b, v in worst.items():
        assert v <= EXACT_GRAD_MEASURED[name][b][0], (name, b, v)


@pytest.mark.parametrize("name", ENVS)
def test_regime_batch_visits_every_branch(name):
    """The batch of the exact-gradient tests enters every branch of the contact and limit model the articulation has, on
    every H-refresh pattern (the golden states alone never push Ant past an upper limit, nor Hopper past a lower one or into
    its Coulomb cap)."""
    o = X._oracle(name)
    desc, inp, idx = _batch(name)
    sub = {k: (None if v is None else v[idx]) for k, v in inp.items()}
    for S, mm in X.patterns(name):
        cov = X.branch_coverage(o, sub, S, mm, X.pattern_dt(name, S))
        missing = [b for b in X.branches_of_model(desc) if cov[b] == 0]
        assert not missing, (name, (S, mm), cov)
    if name != "CartPoleSwingUpEnv":
        assert X.branches_of_model(desc) == ["penetrate", "vn_neg", "cap_viscous", "cap_coulomb", "lower", "upper"]


def emulation_gradients(name, inp, idx, S, mm, dt):
    d, model = load_golden(name)
    emu = EmuSim(model, int(d["meta/num_envs"]))
    emu.N = len(idx)
    sel = lambda k: None if inp[k] is None else np.ascontiguousarray(inp[k][idx]).ravel()
    _, _, tape, _ = emu.forward(sel("q0"), sel("qd0"), sel("act"), sel("musc"), S, mm, dt)
    g = emu.backward(sel("act"), sel("musc"), tape, sel("gq_out"), sel("gqd_out"), S, mm, dt)
    return [x.reshape(len(idx), -1) for x in g if x is not None]


@pytest.mark.parametrize("name", ENVS)
def test_emulated_adjoint_matches_exact_gradient(name):
    """Every environment, every block, every H-refresh pattern: the host emulation of dfx_phases.h's adjoint within the bound
    of tolerances.exact_grad_tol, as the CUDA kernels are.  An independent check of the adjoint's math without a GPU."""
    o = X._oracle(name)
    desc, inp, idx = _batch(name)
    for S, mm in X.patterns(name):
        dt = X.pattern_dt(name, S)
        ex = X.exact_gradients(name, inp, idx, S, mm, dt)
        got = emulation_gradients(name, inp, idx, S, mm, dt)
        worst, _ = X.check_against_exact("%s (%d, %d) emulation" % (name, S, mm), o, inp, idx, got, ex, exact_grad_tol(name, S),
                                         S, mm, dt, max_excluded=max(2, len(idx) // 20))
        print(name, (S, mm), {b: "%.1e" % v for b, v in worst.items()})
