"""ctypes front-end of the C restatement (oracle/dflex_oracle.c).  TEST INFRASTRUCTURE ONLY."""
import ctypes
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
from diffrl_b200.modelpack import DfxModelDesc, articulation_from_model  # noqa: E402  (struct definition only)

_D = ctypes.POINTER(ctypes.c_double)
_libs = {}
# columns of Oracle.branches' counts (dflex_oracle.c BR_*): penetrating contact points, of those with vn < 0, friction capped
# by kf |vt| (viscous) / by mu |fn| (Coulomb), joint coordinate below its lower / above its upper limit; summed over substeps
BRANCHES = ("penetrate", "vn_neg", "cap_viscous", "cap_coulomb", "lower", "upper")


def _lib(precision):
    if precision not in _libs:
        path = os.path.join(_HERE, "liboracle_%s.so" % precision)
        src = os.path.join(_HERE, "dflex_oracle.c")
        if not os.path.exists(path) or os.path.getmtime(src) > os.path.getmtime(path):
            subprocess.check_call(["make", "-s", "-C", _HERE])
        lib = ctypes.CDLL(path)
        lib.oracle_step_forward.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                            _D, _D, _D, _D, _D, _D, _D]
        lib.oracle_fd_gradient.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                           _D, _D, _D, _D, _D, _D, _D, _D, _D, _D]
        lib.oracle_branch_signature.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                                _D, _D, _D, _D, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int64)]
        if precision == "c64":
            lib.oracle_exact_gradient.argtypes = lib.oracle_fd_gradient.argtypes
        assert lib.oracle_real_bytes() == {"f32": 4, "f64": 8, "c64": 16}[precision]
        _libs[precision] = lib
    return _libs[precision]


def _p(a):
    return None if a is None else a.ctypes.data_as(_D)


class Oracle:
    """CPU oracle for one articulation description (``ArticulationDesc`` from diffrl_b200.modelpack)."""

    def __init__(self, desc):
        self.desc = desc
        self.struct = desc.as_struct()

    @classmethod
    def from_model(cls, model, num_envs):
        desc, _ = articulation_from_model(model, num_envs)
        return cls(desc)

    def forward(self, q, qd, act, musc, substeps, mm_freq, dt, precision="f32", want_traj=False):
        d = self.desc
        q = np.ascontiguousarray(q, np.float64).ravel(); qd = np.ascontiguousarray(qd, np.float64).ravel()
        act = np.ascontiguousarray(act, np.float64).ravel()
        n = q.size // d.Q
        musc = np.zeros(max(1, n * d.M)) if musc is None else np.ascontiguousarray(musc, np.float64).ravel()
        q_out, qd_out = np.empty_like(q), np.empty_like(qd)
        traj = np.empty((n, substeps, d.Q + d.D)) if want_traj else None
        _lib(precision).oracle_step_forward(ctypes.byref(self.struct), n, substeps, mm_freq, float(dt), _p(q), _p(qd), _p(act),
                                            _p(musc), _p(q_out), _p(qd_out), _p(traj))
        return (q_out, qd_out, traj) if want_traj else (q_out, qd_out)

    def _inputs(self, q, qd, act, musc):
        d = self.desc
        f = lambda a: np.ascontiguousarray(a, np.float64).ravel()
        q, qd, act = f(q), f(qd), f(act)
        n = q.size // d.Q
        musc = np.zeros(max(1, n * d.M)) if musc is None or d.M == 0 else f(musc)
        return n, q, qd, act, musc

    def branches(self, q, qd, act, musc, substeps, mm_freq, dt, precision="f64"):
        """Per environment: (hash [n] uint64 of the sequence of contact / limit branch decisions over all substeps,
        counts [n, 6] int64 in the order of BRANCHES), in the f32 or the f64 build."""
        n, q, qd, act, musc = self._inputs(q, qd, act, musc)
        h, c = np.zeros(n, np.uint64), np.zeros((n, len(BRANCHES)), np.int64)
        _lib(precision).oracle_branch_signature(ctypes.byref(self.struct), n, substeps, mm_freq, float(dt), _p(q), _p(qd), _p(act), _p(musc),
                                                h.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), c.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)))
        return h, c

    def exact_gradient(self, q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt, h=1e-30):
        """Complex-step derivative of sum(gq_out*q' + gqd_out*qd') for ONE environment: exact to rounding (no cancellation,
        no step-size error) for the branches the fp64 forward takes.  Returns gq, gqd, gact, gmusc (None without muscles)."""
        d = self.desc
        f = lambda a: np.ascontiguousarray(a, np.float64).ravel()
        q, qd, act, gq_out, gqd_out = f(q), f(qd), f(act), f(gq_out), f(gqd_out)
        musc = np.zeros(max(1, d.M)) if musc is None else f(musc)
        gq, gqd, gact = np.zeros(d.Q), np.zeros(d.D), np.zeros(d.D)
        gm = np.zeros(d.M) if d.M else None
        _lib("c64").oracle_exact_gradient(ctypes.byref(self.struct), substeps, mm_freq, float(dt), float(h), _p(q), _p(qd), _p(act),
                                          _p(musc), _p(gq_out), _p(gqd_out), _p(gq), _p(gqd), _p(gact), _p(gm))
        return gq, gqd, gact, gm

    def fd_gradient(self, q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt, eps=1e-6):
        """Central differences in fp64 of sum(gq_out*q' + gqd_out*qd') for ONE environment."""
        d = self.desc
        f = lambda a: np.ascontiguousarray(a, np.float64).ravel()
        q, qd, act, gq_out, gqd_out = f(q), f(qd), f(act), f(gq_out), f(gqd_out)
        musc = np.zeros(max(1, d.M)) if musc is None else f(musc)
        gq, gqd, gact = np.zeros(d.Q), np.zeros(d.D), np.zeros(d.D)
        gm = np.zeros(d.M) if d.M else None
        _lib("f64").oracle_fd_gradient(ctypes.byref(self.struct), substeps, mm_freq, float(dt), float(eps), _p(q), _p(qd), _p(act),
                                       _p(musc), _p(gq_out), _p(gqd_out), _p(gq), _p(gqd), _p(gact), _p(gm))
        return gq, gqd, gact, gm
