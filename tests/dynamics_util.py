"""Test infrastructure of the dynamics state (include/dfx.h dfx_dynamics_state_forward / _backward; tests/test_dynamics_state_emu.py on
the host emulation, tests/test_gpu_dynamics_state.py on the kernels):
  * DynamicsEmuSim: the host emulation with the dynamics-state entries and the external-wrench step entries
    (tests/host_emu/dfx_emu_dynamics.cpp, a library of its own);
  * DynamicsOracle: the fp64 / complex-step dynamics state of the C oracle, and a rollout of env-steps ending in it
    (tests/dynamics_oracle/dynamics_oracle.c: the unchanged wrench oracle plus the dynamics state);
  * batches (link_util.batch's states with random actuation, muscle activations, wrenches and NON-symmetric g_H) and the
    per-environment, per-block error measures."""
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

import link_util as LU  # noqa: E402
import wrench_util as W  # noqa: E402
from emu_util import fptr  # noqa: E402
from wrench_util import WrenchEmuSim, build_emu_ext  # noqa: E402
from oracle import Oracle  # noqa: E402
from diffrl_b200.modelpack import DfxModelDesc, articulation_from_model  # noqa: E402

_F = ctypes.POINTER(ctypes.c_float)
_D = ctypes.POINTER(ctypes.c_double)
EMU_DYN_SRC = os.path.join(HERE, "host_emu", "dfx_emu_dynamics.cpp")
ORACLE_DYN_SRC = os.path.join(HERE, "dynamics_oracle", "dynamics_oracle.c")

DIFFRL, RANDOM, MODELS, FORMULATIONS = LU.DIFFRL, LU.RANDOM, LU.MODELS, LU.FORMULATIONS
N = 75
model_of = LU.model_of
rel_err = LU.rel_err
FIELDS = ("joint_qdd", "joint_tau", "H")


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


# ------------------------------------------------------------------ host emulation with the dynamics-state entries
def build_emu_dynamics(es=1, path_passes=False, layout_mode=0, extra=()):
    """tests/host_emu/dfx_emu_dynamics.cpp with the build flags of emu_util.build_emu (same arguments)"""
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra))
    lib_path = os.path.join(HERE, "host_emu", "libdfx_emu_dynamics_es%d%s%s%s.so" % (es, "_path" if path_passes else "",
                                                                                      "_lm%d" % layout_mode if layout_mode else "", tag))
    deps = [EMU_DYN_SRC, os.path.join(HERE, "host_emu", "dfx_emu_ext.cpp"), os.path.join(HERE, "host_emu", "dfx_emu.cpp")] + LU._headers()
    if _stale(lib_path, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17"] + ([] if any("contract" in x for x in extra) else ["-ffp-contract=off"])
                              + list(extra) + ["-DDFX_ES=%d" % es, "-DDFX_EMU_PATH_PASSES=%d" % int(path_passes)]
                              + (["-DDFX_EMU_LAYOUT_MODE=%d" % layout_mode] if layout_mode else [])
                              + ["-shared", "-fPIC", "-o", lib_path, EMU_DYN_SRC])
    lib = ctypes.CDLL(lib_path)
    ref = build_emu_ext(es, path_passes, layout_mode, extra)
    for name in ("emu_pack_create", "emu_pack_destroy", "emu_tape_floats", "emu_step_forward", "emu_step_backward",
                 "emu_step_forward_ext", "emu_step_backward_ext"):
        f, r = getattr(lib, name), getattr(ref, name)
        f.argtypes = r.argtypes
        f.restype = r.restype
    I = ctypes.c_int
    lib.emu_pack_set_gravity.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_float, I]
    lib.emu_dynamics_state_forward.argtypes = [ctypes.c_void_p, I] + [_F] * 8
    lib.emu_dynamics_state_backward.argtypes = [ctypes.c_void_p, I] + [_F] * 13
    return lib


def _c32(a):
    return None if a is None else np.ascontiguousarray(a, np.float32)


class DynamicsEmuSim(WrenchEmuSim):
    """WrenchEmuSim on the library with the dynamics-state entries."""

    def __init__(self, model, num_envs, es=1, path_passes=False, layout_mode=0, extra=()):
        self.lib = build_emu_dynamics(es, path_passes, layout_mode, extra)
        self.desc, self.N = articulation_from_model(model, num_envs)
        err = ctypes.create_string_buffer(256)
        st = self.desc.as_struct()
        self.pack = self.lib.emu_pack_create(ctypes.byref(st), err, 256)
        if not self.pack:
            raise RuntimeError(err.value.decode())

    def set_ground(self, on):
        g = self.desc.gravity
        self.lib.emu_pack_set_gravity(self.pack, float(g[0]), float(g[1]), float(g[2]), int(bool(on)))

    def dynamics_state(self, q, qd, act, musc, f_ext):
        """(joint_qdd [N, D], joint_tau [N, D], H [N, D, D]) fp32"""
        N, D = self.N, self.desc.D
        out = (np.empty((N, D), np.float32), np.empty((N, D), np.float32), np.empty((N, D, D), np.float32))
        self.lib.emu_dynamics_state_forward(self.pack, N, *(fptr(_c32(x)) for x in (q, qd, act, musc, f_ext)), *(fptr(o) for o in out))
        return out

    def dynamics_state_backward(self, q, qd, act, musc, f_ext, g_qdd, g_tau, g_H):
        """(gq [N, Q], gqd [N, D], gact [N, D], gmusc [N, M] or None, g_f_ext [N, L, 6] or None); a None cotangent is zero"""
        N, d = self.N, self.desc
        gq, gqd, gact = np.empty((N, d.Q), np.float32), np.empty((N, d.D), np.float32), np.empty((N, d.D), np.float32)
        gmusc = np.empty((N, d.M), np.float32) if d.M else None
        gf = np.empty((N, d.L, 6), np.float32) if f_ext is not None else None
        self.lib.emu_dynamics_state_backward(self.pack, N, *(fptr(_c32(x)) for x in (q, qd, act, musc, f_ext, g_qdd, g_tau, g_H)),
                                             fptr(gq), fptr(gqd), fptr(gact), fptr(gmusc), fptr(gf))
        return gq, gqd, gact, gmusc, gf


# ------------------------------------------------------------------ the oracle's dynamics state
_oracle_libs = {}


def _oracle_dyn_lib(precision):
    """tests/dynamics_oracle/dynamics_oracle.c built as oracle/Makefile builds the oracle: f64 or c64 (complex step)"""
    if precision not in _oracle_libs:
        path = os.path.join(HERE, "dynamics_oracle", "libdynamics_oracle_%s.so" % precision)
        deps = [ORACLE_DYN_SRC, os.path.join(HERE, "wrench_oracle", "wrench_oracle.c"), os.path.join(ROOT, "oracle", "dflex_oracle.c"),
                os.path.join(ROOT, "include", "dfx.h")]
        if _stale(path, deps):
            real = ["-DREAL=double"] if precision == "f64" else ["-fcx-limited-range", "-DORACLE_COMPLEX", "-DREAL=double _Complex"]
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall",
                                   "-Wno-unused-function"] + real + ["-o", path, ORACLE_DYN_SRC, "-lm"])
        lib = ctypes.CDLL(path)
        S, I, Dbl = ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_double
        lib.oracle_dynamics_state.argtypes = [S, I] + [_D] * 8
        lib.oracle_dynamics_rollout.argtypes = [S, I, I, I, Dbl] + [_D] * 5
        if precision == "c64":
            lib.oracle_dynamics_state_gradient.argtypes = [S, Dbl] + [_D] * 13
            lib.oracle_dynamics_rollout_gradient.argtypes = [S, I, I, I, Dbl, Dbl] + [_D] * 8
        assert lib.oracle_real_bytes() == {"f64": 8, "c64": 16}[precision]
        _oracle_libs[precision] = lib
    return _oracle_libs[precision]


def _p(a):
    return None if a is None else a.ctypes.data_as(_D)


def _f64(a):
    return np.ascontiguousarray(a, np.float64).ravel()


class DynamicsOracle(Oracle):
    """Oracle plus the dynamics state (fp64), its exact gradient and the rollout ending in it (complex step, one environment)."""

    def set_ground(self, on):
        self.struct.ground = int(bool(on))

    def _zeros(self, n, musc, f_ext):
        d = self.desc
        musc = np.zeros(max(1, n * d.M)) if musc is None else _f64(musc)
        f_ext = np.zeros(n * d.L * 6) if f_ext is None else _f64(f_ext)
        return musc, f_ext

    def dynamics_state(self, q, qd, act, musc=None, f_ext=None):
        """(joint_qdd [n, D], joint_tau [n, D], H [n, D, D]) fp64"""
        d = self.desc
        q, qd, act = _f64(q), _f64(qd), _f64(act)
        n = q.size // d.Q
        musc, f_ext = self._zeros(n, musc, f_ext)
        out = (np.empty((n, d.D)), np.empty((n, d.D)), np.empty((n, d.D, d.D)))
        _oracle_dyn_lib("f64").oracle_dynamics_state(ctypes.byref(self.struct), n, _p(q), _p(qd), _p(act), _p(musc), _p(f_ext),
                                                     *(_p(o) for o in out))
        return out

    def dynamics_state_gradient(self, q, qd, act, musc, f_ext, g_qdd, g_tau, g_H, h=1e-30):
        """(gq [Q], gqd [D], gact [D], gmusc [M] or None, g_f_ext [L, 6]) of sum(g . outputs), ONE environment, exact"""
        d = self.desc
        musc, f_ext = self._zeros(1, musc, f_ext)
        gq, gqd, gact, gf = np.zeros(d.Q), np.zeros(d.D), np.zeros(d.D), np.zeros(d.L * 6)
        gm = np.zeros(d.M) if d.M else None
        g = [None if x is None else _f64(x) for x in (g_qdd, g_tau, g_H)]
        _oracle_dyn_lib("c64").oracle_dynamics_state_gradient(ctypes.byref(self.struct), float(h), _p(_f64(q)), _p(_f64(qd)),
                                                              _p(_f64(act)), _p(musc), _p(f_ext), *(_p(x) for x in g), _p(gq), _p(gqd),
                                                              _p(gact), _p(gm), _p(gf))
        return gq, gqd, gact, gm, gf.reshape(d.L, 6)

    def rollout(self, q, qd, act, substeps, mm_freq, dt):
        """ONE environment without muscles, act [T+1, D]: T env-steps, then (qdd, tau, H, q_T, qd_T) of the end state under act[T]"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        T = act.shape[0] - 1
        out = np.empty(2 * d.D + d.D * d.D + d.Q + d.D)
        _oracle_dyn_lib("f64").oracle_dynamics_rollout(ctypes.byref(self.struct), T, substeps, mm_freq, float(dt), _p(_f64(q)),
                                                       _p(_f64(qd)), _p(_f64(act)), _p(np.zeros(1)), _p(out))
        return split_rollout(d, out)

    def rollout_gradient(self, q, qd, act, g, substeps, mm_freq, dt, h=1e-30):
        """(gq [Q], gqd [D], gact [T+1, D]) of sum(g . rollout output) (g as split_rollout returns it), exact"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        T = act.shape[0] - 1
        gq, gqd, gact = np.zeros(d.Q), np.zeros(d.D), np.zeros(act.size)
        gflat = np.concatenate([np.ravel(x) for x in g]).astype(np.float64)
        _oracle_dyn_lib("c64").oracle_dynamics_rollout_gradient(ctypes.byref(self.struct), T, substeps, mm_freq, float(dt), float(h),
                                                                _p(_f64(q)), _p(_f64(qd)), _p(_f64(act)), _p(np.zeros(1)), _p(gflat),
                                                                _p(gq), _p(gqd), _p(gact))
        return gq, gqd, gact.reshape(act.shape)


def split_rollout(d, out):
    D, Q = d.D, d.Q
    k = 2 * D + D * D
    return out[:D], out[D:2 * D], out[2 * D:k].reshape(D, D), out[k:k + Q], out[k + Q:k + Q + D]


def oracle_of(name, ground=None):
    model, ne = model_of(name)
    desc, _ = articulation_from_model(model, ne, ground=ground)
    return DynamicsOracle(desc)


# ------------------------------------------------------------------ batches
def batch(name, n=N, seed=3, wrench=True):
    """(desc, inputs dict(q, qd, act, musc, f_ext), cotangents (g_qdd, g_tau, g_H)) fp32: link_util.batch's states (golden or
    random states with every regime row, quaternions off the unit sphere), actuation of the size of the golden actions
    (standard normal x 0.5 x the drive's scale), muscle activations in [0, 1], wrench_util.random_wrench (None without),
    standard-normal cotangents with g_H NOT symmetric"""
    desc, q, qd, _ = LU.batch(name, n, seed)
    model, ne = model_of(name)
    rng = np.random.default_rng([seed, 17])
    D, M, L = desc.D, desc.M, desc.L
    act = (rng.standard_normal((n, D)) * 0.5).astype(np.float32)
    musc = rng.uniform(0.0, 1.0, (n, M)).astype(np.float32) if M else None
    f_ext = W.random_wrench(model, ne, n, seed) if wrench else None
    g = (rng.standard_normal((n, D)).astype(np.float32), rng.standard_normal((n, D)).astype(np.float32),
         rng.standard_normal((n, D, D)).astype(np.float32))
    return desc, dict(q=q, qd=qd, act=act, musc=musc, f_ext=f_ext), g


# ------------------------------------------------------------------ error measures
def forward_errors(got, ref):
    """{field: [n]}: per environment, max |got - ref| over the field's max |ref|"""
    out = {}
    for name, g, r in zip(FIELDS, got, ref):
        g, r = np.asarray(g, np.float64).reshape(len(r), -1), np.asarray(r, np.float64).reshape(len(r), -1)
        scale = np.abs(r).max(axis=1)
        out[name] = np.abs(g - r).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


GRAD_NAMES = ("gq", "gqd", "gact", "gmusc", "g_f_ext")


def grad_errors(got, exact):
    """{gradient: [n]}: per environment, max |got - exact| over max |exact| of the environment's whole gradient (every input):
    a block a million times smaller than the rest is within the rounding of the sums that form the large ones"""
    n = len(exact[0])
    env_max = np.zeros(n)
    for x in exact:
        if x is not None:
            env_max = np.maximum(env_max, np.abs(np.asarray(x, np.float64).reshape(n, -1)).max(axis=1, initial=0.0))
    out = {}
    for name, g, x in zip(GRAD_NAMES, got, exact):
        if g is None or x is None:
            continue
        g, x = np.asarray(g, np.float64).reshape(n, -1), np.asarray(x, np.float64).reshape(n, -1)
        out[name] = np.abs(g - x).max(axis=1, initial=0.0) / np.where(env_max > 0, env_max, 1.0)
    return out


_cache = {}


def exact_gradients(name, o, inp, g, envs):
    """[gq, gqd, gact, gmusc, g_f_ext] exact for environments `envs`, stacked (cached per model, ground and inputs)"""
    key = (name, o.struct.ground, tuple(envs)) + tuple(None if x is None else x.tobytes() for x in (*inp.values(), *g))
    if key not in _cache:
        rows = []
        for e in envs:
            pick = lambda x: None if x is None else x[e]
            rows.append(o.dynamics_state_gradient(inp["q"][e], inp["qd"][e], inp["act"][e], pick(inp["musc"]), pick(inp["f_ext"]),
                                                  g[0][e], g[1][e], g[2][e]))
        _cache[key] = [None if rows[0][k] is None else np.stack([r[k] for r in rows]) for k in range(5)]
        if inp["f_ext"] is None:
            _cache[key][4] = None
    return _cache[key]


def reference(name, o, inp):
    key = ("fwd", name, o.struct.ground) + tuple(None if x is None else x.tobytes() for x in inp.values())
    if key not in _cache:
        _cache[key] = o.dynamics_state(inp["q"], inp["qd"], inp["act"], inp["musc"], inp["f_ext"])
    return _cache[key]


def finite_rows(*arrays):
    """[n] bool: environments whose arrays are all finite"""
    ok = None
    for a in arrays:
        if a is None:
            continue
        a = np.asarray(a).reshape(len(a), -1)
        f = np.isfinite(a).all(axis=1)
        ok = f if ok is None else ok & f
    return ok


# ------------------------------------------------------------------ the convention check
def convention_error(qd, qdd, qd_out, dt_sub):
    """[n]: |qd_out - (qd + dt qdd)| per environment over the fp32 rounding of that update, 2^-23 (|qd| + |dt qdd|) + 1 ulp"""
    qd, qdd, qd_out = (np.asarray(x, np.float64) for x in (qd, qdd, qd_out))
    upd = qd + np.float64(np.float32(dt_sub)) * qdd
    scale = 2.0 ** -23 * (np.abs(qd) + np.abs(np.float64(np.float32(dt_sub)) * qdd)) + np.finfo(np.float32).tiny
    return (np.abs(qd_out - upd) / scale).max(axis=1)
