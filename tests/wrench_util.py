"""Test infrastructure of the external wrench (include/dfx.h DfxExternalWrench; tests/test_external_wrench_emu.py on the host
emulation, tests/test_gpu_external_wrench.py on the kernels):
  * WrenchEmuSim: the host emulation with the _ex entries (tests/host_emu/dfx_emu_ext.cpp, a library of its own);
  * WrenchOracle: the fp64 / complex-step oracle with the wrench applied (tests/wrench_oracle/wrench_oracle.c, the unchanged
    oracle/dflex_oracle.c plus the wrench);
  * golden states of the six DiffRL articulations with a seeded random wrench per environment and link, per-block errors
    against the oracle, and their bounds (WRENCH_MEASURED, wrench_tol)."""
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
from oracle import Oracle  # noqa: E402
from diffrl_b200.modelpack import DfxDerived, DfxModelDesc  # noqa: E402

_F = ctypes.POINTER(ctypes.c_float)
_D = ctypes.POINTER(ctypes.c_double)
EMU_EXT_SRC = os.path.join(HERE, "host_emu", "dfx_emu_ext.cpp")
ORACLE_EXT_SRC = os.path.join(HERE, "wrench_oracle", "wrench_oracle.c")


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def _headers():
    csrc = os.path.join(ROOT, "diffrl_b200", "csrc")
    return [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".h")] + [os.path.join(ROOT, "include", "dfx.h")]


# ------------------------------------------------------------------ host emulation with the _ex entries
def build_emu_ext(es=1, path_passes=False, layout_mode=0, extra=()):
    """tests/host_emu/dfx_emu_ext.cpp with the build flags of emu_util.build_emu (same arguments)"""
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra))
    lib_path = os.path.join(HERE, "host_emu", "libdfx_emu_ext_es%d%s%s%s.so" % (es, "_path" if path_passes else "",
                                                                                 "_lm%d" % layout_mode if layout_mode else "", tag))
    deps = [EMU_EXT_SRC, os.path.join(HERE, "host_emu", "dfx_emu.cpp")] + _headers()
    if _stale(lib_path, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17"] + ([] if any("contract" in x for x in extra) else ["-ffp-contract=off"])
                              + list(extra) + ["-DDFX_ES=%d" % es, "-DDFX_EMU_PATH_PASSES=%d" % int(path_passes)]
                              + (["-DDFX_EMU_LAYOUT_MODE=%d" % layout_mode] if layout_mode else [])
                              + ["-shared", "-fPIC", "-o", lib_path, EMU_EXT_SRC])
    lib = ctypes.CDLL(lib_path)
    lib.emu_pack_create.restype = ctypes.c_void_p
    lib.emu_pack_create.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_char_p, ctypes.c_int]
    lib.emu_pack_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_tape_floats.restype = ctypes.c_longlong
    lib.emu_tape_floats.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    I, Dbl = ctypes.c_int, ctypes.c_double
    lib.emu_step_forward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, _F, _F, _F, _F, _F, _F, _F, ctypes.POINTER(DfxDerived)]
    lib.emu_step_backward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, _F, _F, _F, _F, _F, _F, _F, _F, _F]
    lib.emu_step_forward_ext.argtypes = lib.emu_step_forward.argtypes + [_F]
    lib.emu_step_backward_ext.argtypes = lib.emu_step_backward.argtypes + [_F, _F]
    return lib


class WrenchEmuSim(EmuSim):
    """EmuSim on the library with the _ex entries: forward / backward take f_ext [N, L, 6] (None: the entries without one)."""

    def __init__(self, model, num_envs, es=1, path_passes=False, layout_mode=0, extra=()):
        from diffrl_b200.modelpack import articulation_from_model
        self.lib = build_emu_ext(es, path_passes, layout_mode, extra)
        self.desc, self.N = articulation_from_model(model, num_envs)
        err = ctypes.create_string_buffer(256)
        st = self.desc.as_struct()
        self.pack = self.lib.emu_pack_create(ctypes.byref(st), err, 256)
        if not self.pack:
            raise RuntimeError(err.value.decode())

    def forward(self, q, qd, act, musc, substeps, mm_freq, dt, f_ext=None):
        """(q_out, qd_out, tape, {}) with a tape always"""
        if f_ext is None:
            return EmuSim.forward(self, q, qd, act, musc, substeps, mm_freq, dt)
        self.lib.emu_set_tape_bf16(int(self.tape_bf16))
        q, qd, act = (np.ascontiguousarray(x, np.float32) for x in (q, qd, act))
        musc = None if musc is None else np.ascontiguousarray(musc, np.float32)
        f_ext = np.ascontiguousarray(f_ext, np.float32)
        q_out, qd_out = np.empty_like(q), np.empty_like(qd)
        tp = np.zeros(self.lib.emu_tape_floats(self.pack, self.N, substeps, mm_freq), np.float32)
        self.lib.emu_step_forward_ext(self.pack, self.N, substeps, mm_freq, float(dt), fptr(q), fptr(qd), fptr(act), fptr(musc),
                                      fptr(q_out), fptr(qd_out), fptr(tp), None, fptr(f_ext))
        return q_out, qd_out, tp, {}

    def backward(self, act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt, f_ext=None):
        """(gq, gqd, gact, gmusc) and, with f_ext, g_f_ext [N, L, 6]"""
        if f_ext is None:
            return EmuSim.backward(self, act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt)
        N, d = self.N, self.desc
        act = np.ascontiguousarray(act, np.float32)
        musc = None if musc is None else np.ascontiguousarray(musc, np.float32)
        gq_out, gqd_out = np.ascontiguousarray(gq_out, np.float32), np.ascontiguousarray(gqd_out, np.float32)
        f_ext = np.ascontiguousarray(f_ext, np.float32)
        gq, gqd, gact = np.zeros(N * d.Q, np.float32), np.zeros(N * d.D, np.float32), np.zeros(N * d.D, np.float32)
        gmusc = np.zeros(N * d.M, np.float32) if d.M else None
        g_f_ext = np.zeros((N, d.L, 6), np.float32)
        self.lib.emu_step_backward_ext(self.pack, N, substeps, mm_freq, float(dt), fptr(act), fptr(musc), fptr(tape), fptr(gq_out),
                                       fptr(gqd_out), fptr(gq), fptr(gqd), fptr(gact), fptr(gmusc), fptr(f_ext), fptr(g_f_ext))
        return gq, gqd, gact, gmusc, g_f_ext


# ------------------------------------------------------------------ the oracle with the wrench
_oracle_libs = {}


def _oracle_ext_lib(precision):
    """tests/wrench_oracle/wrench_oracle.c built as oracle/Makefile builds the oracle: f64 (REAL = double) or c64 (complex step)"""
    if precision not in _oracle_libs:
        path = os.path.join(HERE, "wrench_oracle", "libwrench_oracle_%s.so" % precision)
        deps = [ORACLE_EXT_SRC, os.path.join(ROOT, "oracle", "dflex_oracle.c"), os.path.join(ROOT, "include", "dfx.h")]
        if _stale(path, deps):
            real = ["-DREAL=double"] if precision == "f64" else ["-fcx-limited-range", "-DORACLE_COMPLEX", "-DREAL=double _Complex"]
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall",
                                   "-Wno-unused-function"] + real + ["-o", path, ORACLE_EXT_SRC, "-lm"])
        lib = ctypes.CDLL(path)
        S, I, Dbl = ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_double
        lib.oracle_step_forward_ext.argtypes = [S, I, I, I, Dbl] + [_D] * 7
        if precision == "c64":
            lib.oracle_exact_gradient_ext.argtypes = [S, I, I, Dbl, Dbl] + [_D] * 12
        assert lib.oracle_real_bytes() == {"f64": 8, "c64": 16}[precision]
        _oracle_libs[precision] = lib
    return _oracle_libs[precision]


def _p(a):
    return None if a is None else a.ctypes.data_as(_D)


class WrenchOracle(Oracle):
    """Oracle plus forward_ext (fp64) and exact_gradient_ext (complex step, one environment) with a wrench [.., L, 6]."""

    def forward_ext(self, q, qd, act, musc, f_ext, substeps, mm_freq, dt):
        d = self.desc
        f = lambda a: np.ascontiguousarray(a, np.float64).ravel()
        q, qd, act, f_ext = f(q), f(qd), f(act), f(f_ext)
        n = q.size // d.Q
        musc = np.zeros(max(1, n * d.M)) if musc is None else f(musc)
        q_out, qd_out = np.empty_like(q), np.empty_like(qd)
        _oracle_ext_lib("f64").oracle_step_forward_ext(ctypes.byref(self.struct), n, substeps, mm_freq, float(dt), _p(q), _p(qd), _p(act),
                                                       _p(musc), _p(f_ext), _p(q_out), _p(qd_out))
        return q_out, qd_out

    def exact_gradient_ext(self, q, qd, act, musc, f_ext, gq_out, gqd_out, substeps, mm_freq, dt, h=1e-30):
        """gq, gqd, gact, gmusc (None without muscles), g_f_ext [L, 6] of sum(gq_out*q' + gqd_out*qd') for ONE environment"""
        d = self.desc
        f = lambda a: np.ascontiguousarray(a, np.float64).ravel()
        q, qd, act, f_ext, gq_out, gqd_out = f(q), f(qd), f(act), f(f_ext), f(gq_out), f(gqd_out)
        musc = np.zeros(max(1, d.M)) if musc is None else f(musc)
        gq, gqd, gact, gf = np.zeros(d.Q), np.zeros(d.D), np.zeros(d.D), np.zeros(d.L * 6)
        gm = np.zeros(d.M) if d.M else None
        _oracle_ext_lib("c64").oracle_exact_gradient_ext(ctypes.byref(self.struct), substeps, mm_freq, float(dt), float(h), _p(q), _p(qd),
                                                         _p(act), _p(musc), _p(f_ext), _p(gq_out), _p(gqd_out), _p(gq), _p(gqd), _p(gact),
                                                         _p(gm), _p(gf))
        return gq, gqd, gact, gm, gf.reshape(d.L, 6)


# ------------------------------------------------------------------ bounds
# Worst relative error per block (max |err| / max |oracle| over the block) of the six emulated formulations of
# tests/test_external_wrench_emu.py against the fp64 oracle: q', qd' (forward, N = 8 environments of golden case 0 at the model's
# own (substeps, mm_freq)) and gq, gqd, gact, g_f_ext (adjoint, first 3 environments, against the complex-step gradient), with
# random_wrench(seed 7).  A bound is WRENCH_FACTOR times it, never below WRENCH_FLOOR (the rule of tolerances.EXACT_GRAD_*).
WRENCH_MEASURED = {
    "CartPoleSwingUpEnv": dict(q=6.7e-8, qd=1.9e-6, gq=2.1e-7, gqd=5.4e-8, gact=1.7e-6, gf=1.7e-6),
    "AntEnv": dict(q=2.4e-7, qd=1.6e-6, gq=1.7e-6, gqd=4.4e-7, gact=9.0e-7, gf=1.5e-6),
    "HopperEnv": dict(q=5.5e-7, qd=5.8e-7, gq=4.8e-7, gqd=4.1e-7, gact=9.3e-7, gf=1.1e-6),
    "CheetahEnv": dict(q=1.7e-7, qd=1.9e-7, gq=3.8e-7, gqd=5.1e-7, gact=2.8e-7, gf=2.9e-7),
    "HumanoidEnv": dict(q=3.4e-7, qd=1.1e-6, gq=2.2e-5, gqd=3.3e-6, gact=2.1e-6, gf=1.2e-6),
    "SNUHumanoidEnv": dict(q=2.9e-7, qd=7.7e-6, gq=9.0e-6, gqd=2.7e-6, gact=5.3e-7, gf=3.5e-6),
}
WRENCH_FACTOR = 4.0
WRENCH_FLOOR = 1e-6


def wrench_tol(env_name, block):
    return max(WRENCH_FACTOR * WRENCH_MEASURED[env_name][block], WRENCH_FLOOR)

ENVS = ["CartPoleSwingUpEnv", "AntEnv", "HopperEnv", "CheetahEnv", "HumanoidEnv", "SNUHumanoidEnv"]
N = 8          # environments per batch (the golden case's first N, tiled when it has fewer)
EXACT = 3      # environments per batch whose adjoint is checked against the complex-step gradient (one forward per input)


def link_masses(model):
    return np.asarray(model["body_I_m"], np.float64).reshape(-1, 6, 6)[:, 3, 3]


def random_wrench(model, num_envs, n, seed):
    """[n, L, 6] fp32: per link a torque of ~0.1 m g and a force of ~0.5 m g (N, N m; world axes), m the link's mass.
    num_envs: copies of the articulation in `model`."""
    rng = np.random.default_rng(seed)
    m = link_masses(model)
    L = m.size // num_envs
    mg = 9.81 * m[:L]
    w = np.empty((n, L, 6))
    w[:, :, :3] = 0.1 * mg[None, :, None] * rng.standard_normal((n, L, 3))
    w[:, :, 3:] = 0.5 * mg[None, :, None] * rng.standard_normal((n, L, 3))
    return w.astype(np.float32)


def golden_batch(name, n=N, case=0):
    """(model, meta, inputs) of golden case `case`, the first n environments (tiled when the case has fewer)"""
    d, model = load_golden(name)
    p = "case%d/" % case
    ne = int(d["meta/num_envs"])
    # (num_envs: the golden model holds that many copies of the articulation -- EmuSim / Oracle.from_model / the engine take it)
    meta = dict(S=int(d["meta/substeps"]), mm=int(d["meta/mass_matrix_freq"]), dt=float(d["meta/dt"]), num_envs=ne)
    Q, D, M = int(d["meta/joint_coord_count"]) // ne, int(d["meta/joint_dof_count"]) // ne, int(d["meta/muscle_count"]) // ne

    def rows(key, w):
        a = np.asarray(d[p + key], np.float32).reshape(ne, w)
        return np.ascontiguousarray(np.tile(a, ((n + ne - 1) // ne, 1))[:n])
    inp = dict(q0=rows("q0", Q), qd0=rows("qd0", D), act=rows("act", D), gq_out=rows("gq_out", Q), gqd_out=rows("gqd_out", D),
               musc=rows("musc", M) if M else None)
    return model, meta, inp


def rel_err(got, ref):
    """max |got - ref| / max |ref| over the block"""
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def oracle_errors(o, inp, f_ext, q, qd, grads, meta, envs=EXACT):
    """Per block: forward q', qd' against the f64 oracle (all environments); gq, gqd, gact, g_f_ext against the complex-step
    gradient (the first `envs` environments).  grads = (gq, gqd, gact, g_f_ext) as [n, ...] arrays."""
    S, mm, dt = meta["S"], meta["mm"], meta["dt"]
    oq, oqd = o.forward_ext(inp["q0"], inp["qd0"], inp["act"], inp["musc"], f_ext, S, mm, dt)
    err = dict(q=rel_err(q, oq), qd=rel_err(qd, oqd))
    n = inp["q0"].shape[0]
    gq, gqd, gact, gf = (np.asarray(g).reshape(n, -1) for g in grads)
    ex = {k: [] for k in ("gq", "gqd", "gact", "gf")}
    for e in range(envs):
        m = None if inp["musc"] is None else inp["musc"][e]
        r = o.exact_gradient_ext(inp["q0"][e], inp["qd0"][e], inp["act"][e], m, f_ext[e], inp["gq_out"][e], inp["gqd_out"][e], S, mm, dt)
        for k, v in zip(("gq", "gqd", "gact", "gf"), (r[0], r[1], r[2], r[4])):
            ex[k].append(np.ravel(v))
    for k, g in zip(("gq", "gqd", "gact", "gf"), (gq, gqd, gact, gf)):
        err[k] = rel_err(g[:envs], np.stack(ex[k]))
    return err
