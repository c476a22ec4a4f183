"""Test infrastructure of the link state (include/dfx.h dfx_link_state_forward / _backward; tests/test_link_state_emu.py on the host
emulation, tests/test_gpu_link_state.py on the kernels):
  * LinkEmuSim: the host emulation with the link-state entries (tests/host_emu/dfx_emu_link.cpp, a library of its own);
  * LinkOracle: the fp64 / complex-step link state of the C oracle, and the tethered rollout built on it
    (tests/link_oracle/link_oracle.c: the unchanged wrench oracle plus the link state);
  * batches of the six DiffRL articulations and of the random articulations (every joint type, exact_util.regime_rows, non-unit
    quaternions), cotangents, and the per-environment, per-block error measures."""
import ctypes
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE, os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from emu_util import EmuSim, fptr, load_golden  # noqa: E402
import exact_util as X  # noqa: E402
from oracle import Oracle  # noqa: E402
import random_articulation as R  # noqa: E402
from diffrl_b200.modelpack import DfxDerived, DfxModelDesc, articulation_from_model  # noqa: E402

_F = ctypes.POINTER(ctypes.c_float)
_D = ctypes.POINTER(ctypes.c_double)
EMU_LINK_SRC = os.path.join(HERE, "host_emu", "dfx_emu_link.cpp")
ORACLE_LINK_SRC = os.path.join(HERE, "link_oracle", "link_oracle.c")

DIFFRL = ["CartPoleSwingUpEnv", "AntEnv", "HopperEnv", "CheetahEnv", "HumanoidEnv", "SNUHumanoidEnv"]
RANDOM = ["twin_" + n for n in R.TWINS] + ["gen_" + k for k in R.GENERIC]
MODELS = DIFFRL + RANDOM
N = 75

# the emulated formulations of the kernels (as tests/test_random_articulations_emu.py)
FORMULATIONS = {
    "group": dict(),
    "tile32": dict(es=32, path_passes=True),
    "tile8m1": dict(es=8, path_passes=True, layout_mode=1),
    "tile8m3": dict(es=8, path_passes=True, layout_mode=3),
    "fused": dict(es=8, path_passes=True, layout_mode=3, extra=("-DDFX_EMU_FUSED_PHASES=1",)),
    "fma": dict(extra=("-ffp-contract=fast", "-mfma")),
}


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def _headers():
    csrc = os.path.join(ROOT, "diffrl_b200", "csrc")
    return [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")] + [os.path.join(ROOT, "include", "dfx.h")]


# ------------------------------------------------------------------ host emulation with the link-state entries
def build_emu_link(es=1, path_passes=False, layout_mode=0, extra=()):
    """tests/host_emu/dfx_emu_link.cpp with the build flags of emu_util.build_emu (same arguments)"""
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra))
    lib_path = os.path.join(HERE, "host_emu", "libdfx_emu_link_es%d%s%s%s.so" % (es, "_path" if path_passes else "",
                                                                                  "_lm%d" % layout_mode if layout_mode else "", tag))
    deps = [EMU_LINK_SRC, os.path.join(HERE, "host_emu", "dfx_emu.cpp")] + _headers()
    if _stale(lib_path, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17"] + ([] if any("contract" in x for x in extra) else ["-ffp-contract=off"])
                              + list(extra) + ["-DDFX_ES=%d" % es, "-DDFX_EMU_PATH_PASSES=%d" % int(path_passes)]
                              + (["-DDFX_EMU_LAYOUT_MODE=%d" % layout_mode] if layout_mode else [])
                              + ["-shared", "-fPIC", "-o", lib_path, EMU_LINK_SRC])
    lib = ctypes.CDLL(lib_path)
    lib.emu_pack_create.restype = ctypes.c_void_p
    lib.emu_pack_create.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_char_p, ctypes.c_int]
    lib.emu_pack_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_tape_floats.restype = ctypes.c_longlong
    lib.emu_tape_floats.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    I, Dbl = ctypes.c_int, ctypes.c_double
    lib.emu_step_forward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, _F, _F, _F, _F, _F, _F, _F, ctypes.POINTER(DfxDerived)]
    lib.emu_step_backward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, _F, _F, _F, _F, _F, _F, _F, _F, _F]
    lib.emu_link_state_forward.argtypes = [ctypes.c_void_p, I, _F, _F, _F, _F, _F]
    lib.emu_link_state_backward.argtypes = [ctypes.c_void_p, I, _F, _F, _F, _F, _F, _F, _F]
    return lib


class LinkEmuSim(EmuSim):
    """EmuSim on the library with the link-state entries."""

    def __init__(self, model, num_envs, es=1, path_passes=False, layout_mode=0, extra=()):
        self.lib = build_emu_link(es, path_passes, layout_mode, extra)
        self.desc, self.N = articulation_from_model(model, num_envs)
        err = ctypes.create_string_buffer(256)
        st = self.desc.as_struct()
        self.pack = self.lib.emu_pack_create(ctypes.byref(st), err, 256)
        if not self.pack:
            raise RuntimeError(err.value.decode())

    def link_state(self, q, qd):
        """(X_sc [N, L, 7], X_sm [N, L, 7], v_s [N, L, 6]) fp32"""
        N, L = self.N, self.desc.L
        q, qd = np.ascontiguousarray(q, np.float32), np.ascontiguousarray(qd, np.float32)
        out = (np.empty((N, L, 7), np.float32), np.empty((N, L, 7), np.float32), np.empty((N, L, 6), np.float32))
        self.lib.emu_link_state_forward(self.pack, N, fptr(q), fptr(qd), *(fptr(o) for o in out))
        return out

    def link_state_backward(self, q, qd, g_X_sc, g_X_sm, g_v_s):
        """(gq [N, Q], gqd [N, D]); a None cotangent is zero"""
        N, d = self.N, self.desc
        f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        gq, gqd = np.empty((N, d.Q), np.float32), np.empty((N, d.D), np.float32)
        self.lib.emu_link_state_backward(self.pack, N, fptr(f(q)), fptr(f(qd)), fptr(f(g_X_sc)), fptr(f(g_X_sm)), fptr(f(g_v_s)),
                                         fptr(gq), fptr(gqd))
        return gq, gqd


# ------------------------------------------------------------------ the oracle's link state
_oracle_libs = {}


def _oracle_link_lib(precision):
    """tests/link_oracle/link_oracle.c built as oracle/Makefile builds the oracle: f64 (REAL = double) or c64 (complex step)"""
    if precision not in _oracle_libs:
        path = os.path.join(HERE, "link_oracle", "liblink_oracle_%s.so" % precision)
        deps = [ORACLE_LINK_SRC, os.path.join(HERE, "wrench_oracle", "wrench_oracle.c"), os.path.join(ROOT, "oracle", "dflex_oracle.c"),
                os.path.join(ROOT, "include", "dfx.h")]
        if _stale(path, deps):
            real = ["-DREAL=double"] if precision == "f64" else ["-fcx-limited-range", "-DORACLE_COMPLEX", "-DREAL=double _Complex"]
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall",
                                   "-Wno-unused-function"] + real + ["-o", path, ORACLE_LINK_SRC, "-lm"])
        lib = ctypes.CDLL(path)
        S, I, Dbl = ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_double
        lib.oracle_link_state.argtypes = [S, I] + [_D] * 5
        lib.oracle_tether_rollout.argtypes = [S, I, I, I, Dbl, Dbl] + [_D] * 6
        if precision == "c64":
            lib.oracle_link_state_gradient.argtypes = [S, Dbl] + [_D] * 7
            lib.oracle_tether_rollout_gradient.argtypes = [S, I, I, I, Dbl, Dbl, Dbl] + [_D] * 11
        assert lib.oracle_real_bytes() == {"f64": 8, "c64": 16}[precision]
        _oracle_libs[precision] = lib
    return _oracle_libs[precision]


def _p(a):
    return None if a is None else a.ctypes.data_as(_D)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, np.float64).ravel()


class LinkOracle(Oracle):
    """Oracle plus the link state (fp64), its exact gradient and the tethered rollout (complex step, one environment)."""

    def link_state(self, q, qd):
        """(X_sc [n, L, 7], X_sm [n, L, 7], v_s [n, L, 6]) fp64"""
        d = self.desc
        q, qd = _f64(q), _f64(qd)
        n = q.size // d.Q
        out = (np.empty((n, d.L, 7)), np.empty((n, d.L, 7)), np.empty((n, d.L, 6)))
        _oracle_link_lib("f64").oracle_link_state(ctypes.byref(self.struct), n, _p(q), _p(qd), *(_p(o) for o in out))
        return out

    def link_state_gradient(self, q, qd, g_X_sc, g_X_sm, g_v_s, h=1e-30):
        """(gq [Q], gqd [D]) of sum(g . (X_sc, X_sm, v_s)) for ONE environment, exact (complex step); None cotangents are zero"""
        d = self.desc
        gq, gqd = np.zeros(d.Q), np.zeros(d.D)
        _oracle_link_lib("c64").oracle_link_state_gradient(ctypes.byref(self.struct), float(h), _p(_f64(q)), _p(_f64(qd)), _p(_f64(g_X_sc)),
                                                           _p(_f64(g_X_sm)), _p(_f64(g_v_s)), _p(gq), _p(gqd))
        return gq, gqd

    def tether_rollout(self, q, qd, act, musc, target, k, substeps, mm_freq, dt):
        """ONE environment, act [T, D]: the link state (X_sc [L, 7], X_sm [L, 7], v_s [L, 6]) at the end of T env-steps, each under
        the tether wrench (0, k (target - X_sm.p)) of the state it starts from"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        out = np.empty(d.L * 20)
        _oracle_link_lib("f64").oracle_tether_rollout(ctypes.byref(self.struct), act.shape[0], substeps, mm_freq, float(dt), float(k), _p(_f64(q)),
                                                      _p(_f64(qd)), _p(_f64(act)), _p(_f64(musc)), _p(_f64(target)), _p(out))
        L = d.L
        return out[:L * 7].reshape(L, 7), out[L * 7:L * 14].reshape(L, 7), out[L * 14:].reshape(L, 6)

    def tether_rollout_gradient(self, q, qd, act, musc, target, k, g_X_sc, g_X_sm, g_v_s, substeps, mm_freq, dt, h=1e-30):
        """(gq [Q], gqd [D], gact [T, D]) of sum(g . final link state) of tether_rollout, exact (complex step)"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        gq, gqd, gact = np.zeros(d.Q), np.zeros(d.D), np.zeros(act.size)
        _oracle_link_lib("c64").oracle_tether_rollout_gradient(
            ctypes.byref(self.struct), act.shape[0], substeps, mm_freq, float(dt), float(k), float(h), _p(_f64(q)), _p(_f64(qd)),
            _p(_f64(act)), _p(_f64(musc)), _p(_f64(target)), _p(_f64(g_X_sc)), _p(_f64(g_X_sm)), _p(_f64(g_v_s)), _p(gq), _p(gqd), _p(gact))
        return gq, gqd, gact.reshape(act.shape)


# ------------------------------------------------------------------ models and batches
def model_of(name):
    """(model dict, num_envs it holds) of a DiffRL golden model or a random articulation"""
    if name in DIFFRL:
        d, model = load_golden(name)
        return model, int(d["meta/num_envs"])
    rm = R.twin(name[len("twin_"):]) if name.startswith("twin_") else R.generic(name[len("gen_"):])
    return rm.model, 1


def oracle_of(name):
    model, ne = model_of(name)
    desc, _ = articulation_from_model(model, ne)
    return LinkOracle(desc)


def _quat_slices(desc):
    """coordinate slices of the quaternions of the ball and free joints"""
    a = desc.arrays
    q0 = int(a["joint_q_start"][0])
    out = []
    for i in range(desc.L):
        t, c = int(a["joint_type"][i]), int(a["joint_q_start"][i]) - q0
        if t == R.BALL:
            out.append(slice(c, c + 4))
        elif t == R.FREE:
            out.append(slice(c + 3, c + 7))
    return out


def batch(name, n=N, seed=3):
    """(desc, q [n, Q], qd [n, D], cotangents (g_X_sc, g_X_sm, g_v_s) [n, L, 7/7/6]) fp32: the step batches of the model
    (exact_util.make_batch / random_articulation.make_batch: golden or random states, every regime row), every quaternion of
    every third environment scaled off the unit sphere (|q| in [0.8, 1.25]), standard-normal cotangents"""
    if name in DIFFRL:
        desc, inp, _ = X.make_batch(name, n, n, seed=seed)
    else:
        rm = R.twin(name[len("twin_"):]) if name.startswith("twin_") else R.generic(name[len("gen_"):])
        desc, inp, _ = R.make_batch(rm, n, n, seed=seed)
    rng = np.random.default_rng([seed, 11])
    q, qd = inp["q0"].copy(), inp["qd0"].copy()
    for e in range(0, n, 3):
        for sl in _quat_slices(desc):
            q[e, sl] *= np.float32(rng.uniform(0.8, 1.25))
    L = desc.L
    g = (rng.standard_normal((n, L, 7)).astype(np.float32), rng.standard_normal((n, L, 7)).astype(np.float32),
         rng.standard_normal((n, L, 6)).astype(np.float32))
    return desc, q, qd, g


# ------------------------------------------------------------------ error measures
FWD_BLOCKS = (("X_sc_p", 0, slice(0, 3)), ("X_sc_q", 0, slice(3, 7)), ("X_sm_p", 1, slice(0, 3)), ("X_sm_q", 1, slice(3, 7)),
              ("v_w", 2, slice(0, 3)), ("v_o", 2, slice(3, 6)))


def forward_errors(got, ref):
    """{block: [n]}: per environment, the largest |got - ref| of the block's elements over the block's largest |ref| (positions,
    quaternions, angular and linear velocities of all links)"""
    out = {}
    for bname, k, sl in FWD_BLOCKS:
        g = np.asarray(got[k], np.float64)[:, :, sl].reshape(len(got[k]), -1)
        r = np.asarray(ref[k], np.float64)[:, :, sl].reshape(len(ref[k]), -1)
        scale = np.abs(r).max(axis=1)
        out[bname] = np.abs(g - r).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


def grad_blocks(desc):
    """the gq / gqd blocks of exact_util.blocks (root position / quaternion / joints, root angular / linear / joints)"""
    return [(b, gi, sl) for b, gi, sl in X.blocks(desc) if gi in (0, 1)]


def grad_errors(desc, gq, gqd, exact_gq, exact_gqd):
    """{block: [n]} per environment, as exact_util.block_errors"""
    got, ex = [gq, gqd], [exact_gq, exact_gqd]
    out = {}
    for bname, gi, sl in grad_blocks(desc):
        g = np.asarray(got[gi], np.float64)[:, sl]
        x = np.asarray(ex[gi], np.float64)[:, sl]
        if g.shape[1] == 0:
            continue
        scale = np.abs(x).max(axis=1)
        out[bname] = np.abs(g - x).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


_exact_cache = {}


def exact_link_gradients(name, o, q, qd, g):
    """(gq [n, Q], gqd [n, D]) exact, per environment (cached per model and inputs)"""
    key = (name, q.tobytes(), qd.tobytes()) + tuple(x.tobytes() for x in g)
    if key not in _exact_cache:
        res = [o.link_state_gradient(q[e], qd[e], g[0][e], g[1][e], g[2][e]) for e in range(q.shape[0])]
        _exact_cache[key] = (np.stack([r[0] for r in res]), np.stack([r[1] for r in res]))
    return _exact_cache[key]


def reference(name, o, q, qd):
    """the fp64 link state of the batch (cached)"""
    key = ("fwd", name, q.tobytes(), qd.tobytes())
    if key not in _exact_cache:
        _exact_cache[key] = o.link_state(q, qd)
    return _exact_cache[key]


# ------------------------------------------------------------------ the tethered rollout
TETHER_T = 4            # env-steps
TETHER_K = 20.0         # N/m
TETHER_OFFSET = (0.1, 0.05, -0.1)    # target = the start's centre of mass + this (m, world axes)


def tether_target(X_sm):
    """[n, L, 3] fp32: every link's centre of mass at the start, shifted by TETHER_OFFSET"""
    return (np.asarray(X_sm)[:, :, :3] + np.asarray(TETHER_OFFSET)).astype(np.float32)


def tether_wrench(X_sm, target):
    """[n, L, 6] fp32: (0, k (target - X_sm.p)) per link"""
    f = np.zeros(X_sm.shape[:2] + (6,), np.float32)
    f[:, :, 3:] = np.float32(TETHER_K) * (target - X_sm[:, :, :3])
    return f


def tether_case(name, n, seed=5):
    """(model, num_envs, meta, q0 [n, Q], qd0 [n, D], acts [T, n, D]) of golden case 0: the first n environments (tiled), actions
    of the golden case scaled by random factors per env-step"""
    import wrench_util as W
    model, meta, inp = W.golden_batch(name, n)
    rng = np.random.default_rng(seed)
    acts = np.stack([(inp["act"] * rng.uniform(0.5, 1.5, inp["act"].shape)).astype(np.float32) for _ in range(TETHER_T)])
    return model, meta, inp["q0"], inp["qd0"], acts


def emu_tether_rollout(link_emu, step_emu, q, qd, acts, target, g, S, mm, dt):
    """the tethered rollout and its adjoint in the host emulation, chained by hand: returns (final link state, gq, gqd, gact [T, n, D])"""
    saved = []
    for t in range(acts.shape[0]):
        X_sm = link_emu.link_state(q, qd)[1]
        f = tether_wrench(X_sm, target)
        q2, qd2, tape, _ = step_emu.forward(q, qd, acts[t], None, S, mm, dt, f_ext=f)
        saved.append((q, qd, f, tape))
        q, qd = q2, qd2
    out = link_emu.link_state(q, qd)
    gq, gqd = link_emu.link_state_backward(q, qd, *g)
    gact = np.zeros_like(acts)
    for t in reversed(range(acts.shape[0])):
        qt, qdt, f, tape = saved[t]
        gq_in, gqd_in, ga, _, gf = step_emu.backward(acts[t], None, tape, gq, gqd, S, mm, dt, f_ext=f)
        gact[t] = ga.reshape(acts[t].shape)
        g_X_sm = np.zeros(f.shape[:2] + (7,), np.float32)
        g_X_sm[:, :, :3] = -np.float32(TETHER_K) * gf[:, :, 3:]
        lq, lqd = link_emu.link_state_backward(qt, qdt, None, g_X_sm, None)
        gq, gqd = gq_in.reshape(lq.shape) + lq, gqd_in.reshape(lqd.shape) + lqd
    return out, gq, gqd, gact


def rel_err(got, ref):
    """max |got - ref| / max |ref|"""
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def tether_errors(o, q0, qd0, acts, target, g, gq, gqd, gact, S, mm, dt, envs):
    """{gq, gqd, gact: worst over environments `envs` of rel_err against the oracle's exact gradient}"""
    err = dict(gq=0.0, gqd=0.0, gact=0.0)
    for e in envs:
        ex = o.tether_rollout_gradient(q0[e], qd0[e], acts[:, e], None, target[e], TETHER_K, g[0][e], g[1][e], g[2][e], S, mm, dt)
        for k, got, x in zip(("gq", "gqd", "gact"), (gq[e], gqd[e], gact[:, e]), ex):
            err[k] = max(err[k], rel_err(got, x))
    return err
