"""Test infrastructure of the Jacobian state (include/dfx.h dfx_jacobian_state_forward / _backward; tests/test_jacobian_state_emu.py
on the host emulation, tests/test_gpu_jacobian_state.py on the kernels):
  * JacobianEmuSim: the host emulation with the Jacobian-state entries (tests/host_emu/dfx_emu_jacobian.cpp, a library of its own);
  * JacobianOracle: the fp64 / complex-step Jacobian state of the C oracle (tests/jacobian_oracle/jacobian_oracle.c: the unchanged
    link oracle plus the Jacobian state);
  * the batches of link_util (every joint type, the regime rows, non-unit quaternions) with Jacobian cotangents, the reference
    rule that assembles J from the joint_S_s dump, and the per-environment, per-block error measures."""
import ctypes
import os
import subprocess

import numpy as np

import link_util as U
from emu_util import fptr
from diffrl_b200.modelpack import DfxModelDesc

HERE = U.HERE
ROOT = U.ROOT
_D = U._D
EMU_JAC_SRC = os.path.join(HERE, "host_emu", "dfx_emu_jacobian.cpp")
ORACLE_JAC_SRC = os.path.join(HERE, "jacobian_oracle", "jacobian_oracle.c")
MODELS, DIFFRL, RANDOM, FORMULATIONS, N = U.MODELS, U.DIFFRL, U.RANDOM, U.FORMULATIONS, U.N


# ------------------------------------------------------------------ host emulation with the Jacobian-state entries
def build_emu_jacobian(es=1, path_passes=False, layout_mode=0, extra=()):
    """tests/host_emu/dfx_emu_jacobian.cpp with the build flags of emu_util.build_emu (same arguments)"""
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra))
    lib_path = os.path.join(HERE, "host_emu", "libdfx_emu_jacobian_es%d%s%s%s.so" % (es, "_path" if path_passes else "",
                                                                                      "_lm%d" % layout_mode if layout_mode else "", tag))
    deps = [EMU_JAC_SRC, U.EMU_LINK_SRC, os.path.join(HERE, "host_emu", "dfx_emu.cpp")] + U._headers()
    if U._stale(lib_path, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17"] + ([] if any("contract" in x for x in extra) else ["-ffp-contract=off"])
                              + list(extra) + ["-DDFX_ES=%d" % es, "-DDFX_EMU_PATH_PASSES=%d" % int(path_passes)]
                              + (["-DDFX_EMU_LAYOUT_MODE=%d" % layout_mode] if layout_mode else [])
                              + ["-shared", "-fPIC", "-o", lib_path, EMU_JAC_SRC])
    lib = ctypes.CDLL(lib_path)
    lib.emu_pack_create.restype = ctypes.c_void_p
    lib.emu_pack_create.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_char_p, ctypes.c_int]
    lib.emu_pack_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_tape_floats.restype = ctypes.c_longlong
    lib.emu_tape_floats.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    I, Dbl, F = ctypes.c_int, ctypes.c_double, U._F
    from diffrl_b200.modelpack import DfxDerived
    lib.emu_step_forward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, F, F, F, F, F, F, F, ctypes.POINTER(DfxDerived)]
    lib.emu_step_backward.argtypes = [ctypes.c_void_p, I, I, I, Dbl, F, F, F, F, F, F, F, F, F]
    lib.emu_link_state_forward.argtypes = [ctypes.c_void_p, I, F, F, F, F, F]
    lib.emu_link_state_backward.argtypes = [ctypes.c_void_p, I, F, F, F, F, F, F, F]
    lib.emu_jacobian_state_forward.argtypes = [ctypes.c_void_p, I, F, F, F, F]
    lib.emu_jacobian_state_backward.argtypes = [ctypes.c_void_p, I, F, F, F, F, F, F]
    return lib


class JacobianEmuSim(U.LinkEmuSim):
    """LinkEmuSim on the library with the Jacobian-state entries."""

    def __init__(self, model, num_envs, es=1, path_passes=False, layout_mode=0, extra=()):
        self.lib = build_emu_jacobian(es, path_passes, layout_mode, extra)
        self.desc, self.N = U.articulation_from_model(model, num_envs)
        err = ctypes.create_string_buffer(256)
        st = self.desc.as_struct()
        self.pack = self.lib.emu_pack_create(ctypes.byref(st), err, 256)
        if not self.pack:
            raise RuntimeError(err.value.decode())

    def jacobian_state(self, q, qd):
        """(J [N, L, 6, D], body_a_s [N, L, 6]) fp32"""
        N, d = self.N, self.desc
        q, qd = np.ascontiguousarray(q, np.float32), np.ascontiguousarray(qd, np.float32)
        J, a = np.empty((N, d.L, 6, d.D), np.float32), np.empty((N, d.L, 6), np.float32)
        self.lib.emu_jacobian_state_forward(self.pack, N, fptr(q), fptr(qd), fptr(J), fptr(a))
        return J, a

    def jacobian_state_backward(self, q, qd, g_J, g_a):
        """(gq [N, Q], gqd [N, D]); a None cotangent is zero"""
        N, d = self.N, self.desc
        f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        gq, gqd = np.empty((N, d.Q), np.float32), np.empty((N, d.D), np.float32)
        self.lib.emu_jacobian_state_backward(self.pack, N, fptr(f(q)), fptr(f(qd)), fptr(f(g_J)), fptr(f(g_a)), fptr(gq), fptr(gqd))
        return gq, gqd


# ------------------------------------------------------------------ the oracle's Jacobian state
_oracle_libs = {}


def _oracle_jac_lib(precision):
    """tests/jacobian_oracle/jacobian_oracle.c built as oracle/Makefile builds the oracle: f64 or c64 (complex step)"""
    if precision not in _oracle_libs:
        path = os.path.join(HERE, "jacobian_oracle", "libjacobian_oracle_%s.so" % precision)
        deps = [ORACLE_JAC_SRC, U.ORACLE_LINK_SRC, os.path.join(HERE, "wrench_oracle", "wrench_oracle.c"),
                os.path.join(ROOT, "oracle", "dflex_oracle.c"), os.path.join(ROOT, "include", "dfx.h")]
        if U._stale(path, deps):
            real = ["-DREAL=double"] if precision == "f64" else ["-fcx-limited-range", "-DORACLE_COMPLEX", "-DREAL=double _Complex"]
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall",
                                   "-Wno-unused-function"] + real + ["-o", path, ORACLE_JAC_SRC, "-lm"])
        lib = ctypes.CDLL(path)
        S, I, Dbl = ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_double
        lib.oracle_jacobian_state.argtypes = [S, I] + [_D] * 4
        lib.oracle_controlled_rollout.argtypes = [S, I, I, I, Dbl, Dbl] + [_D] * 7
        if precision == "c64":
            lib.oracle_jacobian_state_gradient.argtypes = [S, Dbl] + [_D] * 6
            lib.oracle_controlled_rollout_gradient.argtypes = [S, I, I, I, Dbl, Dbl, Dbl] + [_D] * 10
        assert lib.oracle_real_bytes() == {"f64": 8, "c64": 16}[precision]
        _oracle_libs[precision] = lib
    return _oracle_libs[precision]


class JacobianOracle(U.LinkOracle):
    """LinkOracle plus the Jacobian state (fp64) and its exact gradient (complex step, one environment)."""

    def jacobian_state(self, q, qd):
        """(J [n, L, 6, D], body_a_s [n, L, 6]) fp64"""
        d = self.desc
        q, qd = U._f64(q), U._f64(qd)
        n = q.size // d.Q
        J, a = np.empty((n, d.L, 6, d.D)), np.empty((n, d.L, 6))
        _oracle_jac_lib("f64").oracle_jacobian_state(ctypes.byref(self.struct), n, U._p(q), U._p(qd), U._p(J), U._p(a))
        return J, a

    def jacobian_state_gradient(self, q, qd, g_J, g_a, h=1e-30):
        """(gq [Q], gqd [D]) of sum(g_J . J + g_a . body_a_s) for ONE environment, exact (complex step); None cotangents are zero"""
        d = self.desc
        gq, gqd = np.zeros(d.Q), np.zeros(d.D)
        _oracle_jac_lib("c64").oracle_jacobian_state_gradient(ctypes.byref(self.struct), float(h), U._p(U._f64(q)), U._p(U._f64(qd)),
                                                              U._p(U._f64(g_J)), U._p(U._f64(g_a)), U._p(gq), U._p(gqd))
        return gq, gqd

    def controlled_rollout(self, q, qd, u, musc, W, kappa, substeps, mm_freq, dt):
        """ONE environment, u [T, D], W [L, 6]: the end state (q [Q], qd [D]) of T env-steps, each under the actuation
        u_t + J(q_t)^T (W + kappa body_a_s(q_t, qd_t))"""
        d = self.desc
        u = np.asarray(u, np.float64).reshape(-1, d.D)
        q_out, qd_out = np.empty(d.Q), np.empty(d.D)
        _oracle_jac_lib("f64").oracle_controlled_rollout(ctypes.byref(self.struct), u.shape[0], substeps, mm_freq, float(dt), float(kappa),
                                                         U._p(U._f64(q)), U._p(U._f64(qd)), U._p(U._f64(u)), U._p(U._f64(musc)),
                                                         U._p(U._f64(W)), U._p(q_out), U._p(qd_out))
        return q_out, qd_out

    def controlled_rollout_gradient(self, q, qd, u, musc, W, kappa, g_q, g_qd, substeps, mm_freq, dt, h=1e-30):
        """(gq [Q], gqd [D], gu [T, D]) of g_q . q_T + g_qd . qd_T of controlled_rollout, exact (complex step)"""
        d = self.desc
        u = np.asarray(u, np.float64).reshape(-1, d.D)
        gq, gqd, gu = np.zeros(d.Q), np.zeros(d.D), np.zeros(u.size)
        _oracle_jac_lib("c64").oracle_controlled_rollout_gradient(
            ctypes.byref(self.struct), u.shape[0], substeps, mm_freq, float(dt), float(kappa), float(h), U._p(U._f64(q)),
            U._p(U._f64(qd)), U._p(U._f64(u)), U._p(U._f64(musc)), U._p(U._f64(W)), U._p(U._f64(g_q)), U._p(U._f64(g_qd)),
            U._p(gq), U._p(gqd), U._p(gu))
        return gq, gqd, gu.reshape(u.shape)


def oracle_of(name):
    model, ne = U.model_of(name)
    desc, _ = U.articulation_from_model(model, ne)
    return JacobianOracle(desc)


def batch(name, n=N, seed=3):
    """(desc, q [n, Q], qd [n, D], (g_J [n, L, 6, D], g_a [n, L, 6])) fp32: link_util.batch's states (every regime row, non-unit
    quaternions), standard-normal cotangents"""
    desc, q, qd, _ = U.batch(name, n, seed)
    rng = np.random.default_rng([seed, 13])
    g = (rng.standard_normal((n, desc.L, 6, desc.D)).astype(np.float32), rng.standard_normal((n, desc.L, 6)).astype(np.float32))
    return desc, q, qd, g


# ------------------------------------------------------------------ the reference rule and the error measures
def ancestor_mask(desc):
    """[L, D] bool: dof d moves link i (it belongs to i or to an ancestor of i) -- the reference's spatial_jacobian walk"""
    a = desc.arrays
    parent = np.asarray(a["joint_parent"], int)
    qs = np.asarray(a["joint_qd_start"], int) - int(a["joint_qd_start"][0])
    L, D = desc.L, desc.D
    m = np.zeros((L, D), bool)
    for i in range(L):
        j = i
        while j != -1:
            m[i, qs[j]:qs[j + 1]] = True
            j = parent[j]
    return m


def assemble_J(desc, S):
    """J [n, L, 6, D] from joint_S_s [n, D, 6] by the spatial.h:691-738 rule (S columns where the dof moves the link, 0 elsewhere)"""
    S = np.asarray(S).reshape(-1, desc.D, 6)
    m = ancestor_mask(desc)
    return np.where(m[None, :, None, :], np.transpose(S, (0, 2, 1))[:, None, :, :], np.zeros((), S.dtype)).astype(S.dtype)


FWD_BLOCKS = (("J_w", 0, slice(0, 3)), ("J_v", 0, slice(3, 6)), ("a_w", 1, slice(0, 3)), ("a_v", 1, slice(3, 6)))


def forward_errors(got, ref):
    """{block: [n]}: per environment, the largest |got - ref| of the block (angular and linear rows of J over all links and dofs,
    angular and linear bias accelerations) over the largest |ref| of its field (J or body_a_s) -- a planar articulation's angular
    bias accelerations are exactly 0 in fp64, so a per-block scale would divide rounding noise by nothing"""
    out = {}
    for bname, k, sl in FWD_BLOCKS:
        n = len(got[k])
        g = np.asarray(got[k], np.float64)[:, :, sl].reshape(n, -1)
        r = np.asarray(ref[k], np.float64)[:, :, sl].reshape(n, -1)
        scale = np.abs(np.asarray(ref[k], np.float64).reshape(n, -1)).max(axis=1)
        out[bname] = np.abs(g - r).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


grad_errors = U.grad_errors
rel_err = U.rel_err
_exact_cache = {}


def exact_gradients(name, o, q, qd, g):
    """(gq [n, Q], gqd [n, D]) exact, per environment (cached per model and inputs)"""
    key = (name, q.tobytes(), qd.tobytes()) + tuple(x.tobytes() for x in g)
    if key not in _exact_cache:
        res = [o.jacobian_state_gradient(q[e], qd[e], g[0][e], g[1][e]) for e in range(q.shape[0])]
        _exact_cache[key] = (np.stack([r[0] for r in res]), np.stack([r[1] for r in res]))
    return _exact_cache[key]


def reference(name, o, q, qd):
    """the fp64 Jacobian state of the batch (cached)"""
    key = ("fwd", name, q.tobytes(), qd.tobytes())
    if key not in _exact_cache:
        _exact_cache[key] = o.jacobian_state(q, qd)
    return _exact_cache[key]


# ------------------------------------------------------------------ the controlled rollout
CONTROL_T = 4           # env-steps
CONTROL_KAPPA = 0.05    # feedback gain of the bias accelerations (kg m, so kappa * body_a_s is a wrench)


def control_case(name, n, seed=5):
    """(model, meta, q0 [n, Q], qd0 [n, D], u [T, n, D], W [L, 6]) of golden case 0: the first n environments (tiled), the golden
    case's actions scaled by random factors per env-step as u, and a fixed task-space wrench W (small forces and torques on every
    link)"""
    model, meta, q0, qd0, acts = U.tether_case(name, n, seed)
    desc, _ = U.articulation_from_model(model, meta["num_envs"])
    rng = np.random.default_rng([seed, 17])
    W = (0.2 * rng.standard_normal((desc.L, 6))).astype(np.float32)
    return model, meta, q0, qd0, acts, W


def control_act(J, a, u_t, W):
    """act [n, D] = u_t + J^T (W + CONTROL_KAPPA body_a_s), per environment"""
    return (u_t + np.einsum("nlrd,nlr->nd", J, W[None] + np.float32(CONTROL_KAPPA) * a)).astype(np.float32)


def emu_control_rollout(emu, q, qd, u, W, g_q, g_qd, S, mm, dt):
    """the controlled rollout and its adjoint in the host emulation (one JacobianEmuSim for the step and the Jacobian state), chained
    by hand: returns (q_T, qd_T, gq, gqd, gu [T, n, D]) of the loss g_q . q_T + g_qd . qd_T"""
    n, D = q.shape[0], emu.desc.D
    saved = []
    for t in range(u.shape[0]):
        J, a = emu.jacobian_state(q, qd)
        act = control_act(J, a, u[t], W)
        q2, qd2, tape, _ = emu.forward(q, qd, act, None, S, mm, dt)
        saved.append((q, qd, J, a, act, tape))
        q, qd = q2.reshape(q.shape), qd2.reshape(qd.shape)
    qT, qdT = q, qd
    gq, gqd = g_q.astype(np.float32), g_qd.astype(np.float32)
    gu = np.zeros_like(u)
    for t in reversed(range(u.shape[0])):
        qt, qdt, J, a, act, tape = saved[t]
        gq_in, gqd_in, gact, _ = emu.backward(act, None, tape, gq, gqd, S, mm, dt)
        gact = gact.reshape(n, D)
        gu[t] = gact
        g_J = np.einsum("nd,nlr->nlrd", gact, W[None] + np.float32(CONTROL_KAPPA) * a).astype(np.float32)
        g_a = (np.float32(CONTROL_KAPPA) * np.einsum("nlrd,nd->nlr", J, gact)).astype(np.float32)
        jq, jqd = emu.jacobian_state_backward(qt, qdt, g_J, g_a)
        gq, gqd = gq_in.reshape(jq.shape) + jq, gqd_in.reshape(jqd.shape) + jqd
    return qT, qdT, gq, gqd, gu


def control_errors(o, q0, qd0, u, W, g_q, g_qd, gq, gqd, gu, S, mm, dt, envs):
    """{gq, gqd, gu: worst over environments `envs` of rel_err against the oracle's exact gradient}"""
    err = dict(gq=0.0, gqd=0.0, gu=0.0)
    for e in envs:
        ex = o.controlled_rollout_gradient(q0[e], qd0[e], u[:, e], None, W, CONTROL_KAPPA, g_q[e], g_qd[e], S, mm, dt)
        for k, got, x in zip(("gq", "gqd", "gu"), (gq[e], gqd[e], gu[:, e]), ex):
            err[k] = max(err[k], U.rel_err(got, x))
    return err
