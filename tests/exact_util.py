"""Exact (complex-step) gradients of the C oracle and the per-environment, per-block comparison against them, shared by
tests/test_oracle_exact.py (host emulation and the reference's stored gradients, CPU) and tests/test_gpu_exact_adjoint.py
(the CUDA adjoint kernels).

The oracle's complex-step build (oracle/dflex_oracle.c, liboracle_c64.so) differentiates its fp64 forward pass exactly,
branch by branch.  That is the quantity the fp32 reverse-mode adjoints of the reference and of this project both
approximate, so every environment and every block of its gradient can be held to a tolerance -- not a median."""
import os
import sys
from concurrent.futures import ProcessPoolExecutor
import multiprocessing

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE, os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from emu_util import load_golden  # noqa: E402
from oracle import BRANCHES, Oracle  # noqa: E402

ULP = 1.2e-7          # one fp32 ulp, relative


def config(name):
    d, _ = load_golden(name)
    return int(d["meta/substeps"]), int(d["meta/mass_matrix_freq"]), float(d["meta/dt"])


def patterns(name):
    """(substeps, mass-matrix period) patterns of the H-refresh schedule: the env's default, one substep, a refresh every
    substep, every third substep with a short last segment, one refresh longer than the step, and (7, 3)."""
    S, mm, _ = config(name)
    S3 = S if S % 3 else S - 1
    out = [(S, mm), (1, 1), (S, 1), (S3, 3), (S, S + 5), (7, 3)]
    return list(dict.fromkeys(out))


def pattern_dt(name, S):
    """dt of a pattern with S substeps: the substep dt stays the env's own."""
    S0, _, dt = config(name)
    return dt * S / S0


# ------------------------------------------------------------------ gradient blocks
def blocks(desc):
    """[(block name, gradient index (0 gq, 1 gqd, 2 gact, 3 gmusc), slice)].  Each block is normalised by its own largest
    |exact| component, so an error in a small block cannot hide under a large one."""
    free = int(desc.arrays["joint_type"][0]) == 4
    Q, D, M = desc.Q, desc.D, desc.M
    if free:
        out = [("gq_root_pos", 0, slice(0, 3)), ("gq_root_quat", 0, slice(3, 7)), ("gq_joints", 0, slice(7, Q)),
               ("gqd_root_ang", 1, slice(0, 3)), ("gqd_root_lin", 1, slice(3, 6)), ("gqd_joints", 1, slice(6, D)),
               ("gact_joints", 2, slice(6, D))]
    else:
        out = [("gq_joints", 0, slice(0, Q)), ("gqd_joints", 1, slice(0, D)), ("gact_joints", 2, slice(0, D))]
    if M:
        out.append(("gmusc", 3, slice(0, M)))
    return out


def block_errors(desc, got, exact):
    """got, exact: lists [gq, gqd, gact(, gmusc)] of [n, w] arrays -> {block: [n] max |got - exact| / max |exact| over the
    block} (blocks whose exact gradient is zero in an environment get max |got| / 1)."""
    out = {}
    for bname, gi, sl in blocks(desc):
        g = np.asarray(got[gi], np.float64)[:, sl]
        x = np.asarray(exact[gi], np.float64)[:, sl]
        scale = np.abs(x).max(axis=1)
        out[bname] = np.abs(g - x).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


# ------------------------------------------------------------------ inputs
def _limited_joints(desc):
    """coordinate / dof indices of the 1-dof joints that carry a finite limit"""
    a = desc.arrays
    L = desc.L
    q0, d0 = int(a["joint_q_start"][0]), int(a["joint_qd_start"][0])
    out = []
    for i in range(L):
        if int(a["joint_type"][i]) not in (0, 1):
            continue
        cs, ds = int(a["joint_q_start"][i]) - q0, int(a["joint_qd_start"][i]) - d0
        lo, hi = float(a["joint_limit_lower"][cs]), float(a["joint_limit_upper"][cs])
        if float(a["joint_limit_ke"][i]) > 0 and abs(lo) < 100 and abs(hi) < 100:
            out.append((cs, ds, lo, hi))
    return out


def _quat_rotate(q, v):
    u, w = np.asarray(q[:3], np.float64), float(q[3])
    v = np.asarray(v, np.float64)
    return v * (2 * w * w - 1) + np.cross(u, v) * w * 2 + u * np.dot(u, v) * 2


def _root_axes(desc):
    """(height coordinate, its sign, its dof, lateral dof) of the root: the free joint's y / x components, or the planar
    root's prismatic joints along world y and x.  None for a fixed root."""
    a = desc.arrays
    t0 = int(a["joint_type"][0])
    if t0 == 4:
        return 1, 1.0, 4, 3
    if t0 != 0:
        return None
    world = []
    X_pj, axis = np.ravel(a["joint_X_pj"]), np.ravel(a["joint_axis"])
    for i in range(desc.L):
        if int(a["joint_type"][i]) != 0:
            break
        v, j = axis[i * 3: i * 3 + 3], i          # the axis through the parent frames (prismatic joints do not rotate)
        while j >= 0:
            v = _quat_rotate(X_pj[j * 7 + 3: j * 7 + 7], v)
            j = int(a["joint_parent"][j])
        world.append(v)
    up = int(np.argmax([abs(w[1]) for w in world]))
    lat = int(np.argmax([abs(w[0]) if k != up else -1 for k, w in enumerate(world)]))
    return up, float(np.sign(world[up][1])), up, lat


def regime_rows(desc, q, qd, act, musc, act_range, musc_range):
    """Explicit pushes of one base state into the branches of the contact and limit model: every limited joint a few mrad
    beyond its lower / upper limit with velocity into and out of the limit (and alternating lower / upper), the root
    lowered into the ground with lateral (and downward) velocity, the root lifted clear, actions at +-1.5x their range."""
    rows = []

    def row(dq=None, dqd=None, a=None, m=None):
        rq, rqd = q.copy(), qd.copy()
        ra, rm = act.copy(), None if musc is None else musc.copy()
        if dq: dq(rq)
        if dqd: dqd(rqd)
        if a is not None: ra = a
        if m is not None: rm = m
        rows.append((rq, rqd, ra, rm))

    lim = _limited_joints(desc)
    if lim:
        for side in ("lower", "upper", "alternate"):
            for into in (True, False):
                def set_q(rq, side=side):
                    for k, (cs, _, lo, hi) in enumerate(lim):
                        low = side == "lower" or (side == "alternate" and k % 2 == 0)
                        rq[cs] = lo - 3e-3 * (1 + k % 3) if low else hi + 3e-3 * (1 + k % 3)

                def set_qd(rqd, side=side, into=into):
                    for k, (_, ds, _, _) in enumerate(lim):
                        low = side == "lower" or (side == "alternate" and k % 2 == 0)
                        rqd[ds] = (-0.5 if low else 0.5) * (1.0 if into else -1.0)
                row(set_q, set_qd)
    ax = _root_axes(desc)
    if ax is not None and desc.C > 0:
        hq, sgn, hd, ld = ax
        for depth, vdown in ((0.03, 0.0), (0.06, -0.5)):
            def lower(rq, depth=depth):
                rq[hq] -= sgn * depth

            def slide(rqd, vdown=vdown):
                rqd[ld] = 2.5
                rqd[hd] = sgn * vdown
            row(lower, slide)

        def lift(rq):
            rq[hq] += sgn * 1.0
        row(lift)
    for s in (1.0, -1.0):
        row(a=(1.5 * s * act_range).astype(act.dtype),
            m=None if musc is None else (1.5 * musc_range if s > 0 else 0.0 * musc_range).astype(musc.dtype))
    return rows


def make_batch(name, n_total, n_exact, seed=0):
    """n_total environments: the regime rows and golden states + noise at n_exact spread positions (first and last tile
    and between: these are the environments with exact gradients), other golden + noise states elsewhere.
    Returns (desc, inputs dict of [n_total, w] float32 arrays + gq_out / gqd_out, sample indices)."""
    d, model = load_golden(name)
    n0 = int(d["meta/num_envs"])
    o = Oracle.from_model(model, n0)
    desc = o.desc
    Q, D, M = desc.Q, desc.D, desc.M
    rng = np.random.default_rng(seed)
    cases = [k for k in range(int(d["meta/num_cases"]))]
    allq = np.concatenate([d["case%d/q0" % k].reshape(n0, Q) for k in cases])
    allqd = np.concatenate([d["case%d/qd0" % k].reshape(n0, D) for k in cases])
    alla = np.concatenate([d["case%d/act" % k].reshape(n0, D) for k in cases])
    allm = np.concatenate([d["case%d/musc" % k].reshape(n0, M) for k in cases]) if M else None
    act_range = np.abs(alla).max(axis=0).astype(np.float32)
    musc_range = np.abs(allm).max(axis=0).astype(np.float32) if M else None

    def noisy(n):
        pick = rng.integers(0, allq.shape[0], n)
        q = (allq[pick] + 2e-3 * rng.standard_normal((n, Q))).astype(np.float32)
        qd = (allqd[pick] + 2e-2 * rng.standard_normal((n, D))).astype(np.float32)
        a = (alla[pick] * rng.uniform(0.5, 1.5, (n, D))).astype(np.float32)
        m = (allm[pick] * rng.uniform(0.5, 1.5, (n, M))).astype(np.float32) if M else None
        return q, qd, a, m

    q, qd, a, m = noisy(n_total)
    sample = np.unique(np.linspace(0, n_total - 1, n_exact).round().astype(np.int64))
    base = noisy(1)
    regime = regime_rows(desc, base[0][0], base[1][0], base[2][0], None if M == 0 else base[3][0], act_range, musc_range)
    assert len(regime) <= len(sample), (name, len(regime), len(sample))
    # regime rows at every k-th sampled position, so they land in the first tile, the last tile and between
    slots = sample[np.linspace(0, len(sample) - 1, len(regime)).round().astype(np.int64)] if regime else []
    for i, (rq, rqd, ra, rm) in zip(slots, regime):
        q[i], qd[i], a[i] = rq, rqd, ra
        if M:
            m[i] = rm
    inp = dict(q0=q, qd0=qd, act=a, musc=m,
               gq_out=rng.standard_normal((n_total, Q)).astype(np.float32),
               gqd_out=rng.standard_normal((n_total, D)).astype(np.float32))
    return desc, inp, sample


# ------------------------------------------------------------------ exact gradients (a process pool: one job per environment)
_oracles = {}


def _oracle(name):
    if name not in _oracles:
        d, model = load_golden(name)
        _oracles[name] = Oracle.from_model(model, int(d["meta/num_envs"]))
    return _oracles[name]


def _exact_job(job):
    name, S, mm, dt, q, qd, a, m, gq, gqd = job
    return _oracle(name).exact_gradient(q, qd, a, m, gq, gqd, S, mm, dt)


_cache = {}


def exact_gradients(name, inp, idx, S, mm, dt):
    """[gq, gqd, gact(, gmusc)] as [len(idx), w] fp64 arrays: the exact gradients of environments idx (computed once per
    set of inputs and pattern; the fp64 oracle reads the fp32 inputs exactly)."""
    key = (name, S, mm, dt, tuple(int(i) for i in idx)) + tuple(inp[k][idx].tobytes() for k in ("q0", "qd0", "act", "gq_out", "gqd_out"))
    if key in _cache:
        return _cache[key]
    m = inp["musc"]
    jobs = [(name, S, mm, dt, inp["q0"][i], inp["qd0"][i], inp["act"][i], None if m is None else m[i], inp["gq_out"][i],
             inp["gqd_out"][i]) for i in idx]
    workers = max(1, min(16, len(os.sched_getaffinity(0)), len(jobs)))
    if workers == 1:
        res = [_exact_job(j) for j in jobs]
    else:
        with ProcessPoolExecutor(workers, mp_context=multiprocessing.get_context("spawn")) as pool:
            res = list(pool.map(_exact_job, jobs, chunksize=max(1, len(jobs) // (4 * workers))))
    out = [np.stack([r[k] for r in res]) for k in range(4 if res[0][3] is not None else 3)]
    _cache[key] = out
    return out


# ------------------------------------------------------------------ switching surfaces
def _probes(q_row, qd_row):
    yield q_row * (1.0 + ULP), qd_row * (1.0 - ULP)
    yield q_row * (1.0 - ULP), qd_row * (1.0 + ULP)


def on_switching_surface(o, inp, i, S, mm, dt):
    """True when environment i's branch sequence is not determined at fp32 resolution: the f32 and f64 builds of the oracle
    take different branches, or the f64 build's branch signature changes under a +-1-ulp perturbation of the state.
    There fp32 and fp64 may legitimately differentiate different branches."""
    m = inp["musc"]
    mi = None if m is None else m[i:i + 1]
    a = inp["act"][i:i + 1]
    h64, _ = o.branches(inp["q0"][i:i + 1], inp["qd0"][i:i + 1], a, mi, S, mm, dt, "f64")
    h32, _ = o.branches(inp["q0"][i:i + 1], inp["qd0"][i:i + 1], a, mi, S, mm, dt, "f32")
    if h32[0] != h64[0]:
        return True
    for pq, pqd in _probes(inp["q0"][i].astype(np.float64), inp["qd0"][i].astype(np.float64)):
        hp, _ = o.branches(pq[None], pqd[None], a, mi, S, mm, dt, "f64")
        if hp[0] != h64[0]:
            return True
    return False


def check_against_exact(what, o, inp, idx, got, exact, tol, S, mm, dt, max_excluded):
    """got / exact: [gq, gqd, gact(, gmusc)] rows of environments idx.  Every environment must hold every block within
    tol[block]; one that does not may only sit on a switching surface (on_switching_surface), at most max_excluded of them.
    Returns ({block: worst error over the checked environments}, excluded environments)."""
    err = block_errors(o.desc, got, exact)
    bad = sorted({int(k) for b, e in err.items() for k in np.nonzero(e > tol[b])[0]})
    excluded, failures = [], []
    for k in bad:
        if on_switching_surface(o, inp, int(idx[k]), S, mm, dt):
            excluded.append(int(idx[k]))
        else:
            failures.append("env %d: " % idx[k] + ", ".join("%s %.2e > %.2e" % (b, err[b][k], tol[b]) for b in err if err[b][k] > tol[b]))
    keep = np.setdiff1d(np.arange(len(idx)), [k for k in bad if int(idx[k]) in excluded])
    worst = {b: float(e[keep].max()) if len(keep) else 0.0 for b, e in err.items()}
    if excluded:
        print("%s: %d environment(s) on a switching surface excluded: %s" % (what, len(excluded), excluded))
    assert not failures, (what, failures)
    assert len(excluded) <= max_excluded, (what, "too many environments on switching surfaces", excluded)
    return worst, excluded


def branch_coverage(o, inp, S, mm, dt):
    """counts of every branch (BRANCHES order) summed over the batch, in the f64 oracle"""
    _, c = o.branches(inp["q0"], inp["qd0"], inp["act"], inp["musc"], S, mm, dt, "f64")
    return dict(zip(BRANCHES, c.sum(axis=0).tolist()))


def branches_of_model(desc):
    """the branches the model has at all: the contact branches with a ground and contacts, lower / upper with a limited joint"""
    out = []
    if desc.ground and desc.C > 0:
        out += ["penetrate", "vn_neg", "cap_viscous", "cap_coulomb"]
    if _limited_joints(desc):
        out += ["lower", "upper"]
    return out
