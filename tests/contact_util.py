"""Test infrastructure of the contact state (include/dfx.h dfx_contact_state_forward / _backward; tests/test_contact_state_emu.py on
the host emulation, tests/test_gpu_contact_state.py on the kernels):
  * ContactEmuSim: the host emulation with the contact-state entries and the external-wrench step entries
    (tests/host_emu/dfx_emu_contact.cpp, a library of its own);
  * ContactOracle: the fp64 / complex-step contact state of the C oracle, and a rollout of env-steps ending in it
    (tests/contact_oracle/contact_oracle.c: the unchanged link oracle plus the contact state);
  * batches of the six DiffRL articulations and of the random articulations (link_util.batch: every joint type, the
    exact_util.regime_rows, quaternions off the unit sphere; plus resting contacts and height-only cotangents), and the
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
from emu_util import fptr  # noqa: E402
from wrench_util import WrenchEmuSim, build_emu_ext  # noqa: E402
from oracle import Oracle  # noqa: E402
from diffrl_b200.modelpack import DfxModelDesc, articulation_from_model  # noqa: E402

_F = ctypes.POINTER(ctypes.c_float)
_D = ctypes.POINTER(ctypes.c_double)
EMU_CONTACT_SRC = os.path.join(HERE, "host_emu", "dfx_emu_contact.cpp")
ORACLE_CONTACT_SRC = os.path.join(HERE, "contact_oracle", "contact_oracle.c")

DIFFRL, RANDOM, MODELS, N, FORMULATIONS = LU.DIFFRL, LU.RANDOM, LU.MODELS, LU.N, LU.FORMULATIONS
model_of = LU.model_of
rel_err = LU.rel_err


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


# ------------------------------------------------------------------ host emulation with the contact-state entries
def build_emu_contact(es=1, path_passes=False, layout_mode=0, extra=()):
    """tests/host_emu/dfx_emu_contact.cpp with the build flags of emu_util.build_emu (same arguments)"""
    tag = "".join(c if c.isalnum() else "_" for c in "".join(extra))
    lib_path = os.path.join(HERE, "host_emu", "libdfx_emu_contact_es%d%s%s%s.so" % (es, "_path" if path_passes else "",
                                                                                     "_lm%d" % layout_mode if layout_mode else "", tag))
    deps = [EMU_CONTACT_SRC, os.path.join(HERE, "host_emu", "dfx_emu_ext.cpp"), os.path.join(HERE, "host_emu", "dfx_emu.cpp")] + LU._headers()
    if _stale(lib_path, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17"] + ([] if any("contract" in x for x in extra) else ["-ffp-contract=off"])
                              + list(extra) + ["-DDFX_ES=%d" % es, "-DDFX_EMU_PATH_PASSES=%d" % int(path_passes)]
                              + (["-DDFX_EMU_LAYOUT_MODE=%d" % layout_mode] if layout_mode else [])
                              + ["-shared", "-fPIC", "-o", lib_path, EMU_CONTACT_SRC])
    # the step and _ext entries' argtypes as wrench_util sets them, on this library
    lib = ctypes.CDLL(lib_path)
    ref = build_emu_ext(es, path_passes, layout_mode, extra)
    for name in ("emu_pack_create", "emu_pack_destroy", "emu_tape_floats", "emu_step_forward", "emu_step_backward",
                 "emu_step_forward_ext", "emu_step_backward_ext"):
        f, r = getattr(lib, name), getattr(ref, name)
        f.argtypes = r.argtypes
        f.restype = r.restype
    I = ctypes.c_int
    lib.emu_pack_set_gravity.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_float, I]
    lib.emu_contact_state_forward.argtypes = [ctypes.c_void_p, I, _F, _F, _F, _F, _F]
    lib.emu_contact_state_backward.argtypes = [ctypes.c_void_p, I, _F, _F, _F, _F, _F, _F, _F]
    return lib


class ContactEmuSim(WrenchEmuSim):
    """WrenchEmuSim on the library with the contact-state entries."""

    def __init__(self, model, num_envs, es=1, path_passes=False, layout_mode=0, extra=()):
        self.lib = build_emu_contact(es, path_passes, layout_mode, extra)
        self.desc, self.N = articulation_from_model(model, num_envs)
        err = ctypes.create_string_buffer(256)
        st = self.desc.as_struct()
        self.pack = self.lib.emu_pack_create(ctypes.byref(st), err, 256)
        if not self.pack:
            raise RuntimeError(err.value.decode())

    def set_ground(self, on):
        """dfx_pack_set_gravity with the model's gravity and the ground on or off"""
        g = self.desc.gravity
        self.lib.emu_pack_set_gravity(self.pack, float(g[0]), float(g[1]), float(g[2]), int(bool(on)))

    def contact_state(self, q, qd):
        """(contact_f [N, C, 3], contact_height [N, C], body_f_contact [N, L, 6]) fp32"""
        N, d = self.N, self.desc
        q, qd = np.ascontiguousarray(q, np.float32), np.ascontiguousarray(qd, np.float32)
        out = (np.empty((N, d.C, 3), np.float32), np.empty((N, d.C), np.float32), np.empty((N, d.L, 6), np.float32))
        self.lib.emu_contact_state_forward(self.pack, N, fptr(q), fptr(qd), *(fptr(o) for o in out))
        return out

    def contact_state_backward(self, q, qd, g_f, g_h, g_body):
        """(gq [N, Q], gqd [N, D]); a None cotangent is zero"""
        N, d = self.N, self.desc
        f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
        gq, gqd = np.empty((N, d.Q), np.float32), np.empty((N, d.D), np.float32)
        self.lib.emu_contact_state_backward(self.pack, N, fptr(f(q)), fptr(f(qd)), fptr(f(g_f)), fptr(f(g_h)), fptr(f(g_body)),
                                            fptr(gq), fptr(gqd))
        return gq, gqd


# ------------------------------------------------------------------ the oracle's contact state
_oracle_libs = {}


def _oracle_contact_lib(precision):
    """tests/contact_oracle/contact_oracle.c built as oracle/Makefile builds the oracle: f64 (REAL = double) or c64 (complex step)"""
    if precision not in _oracle_libs:
        path = os.path.join(HERE, "contact_oracle", "libcontact_oracle_%s.so" % precision)
        deps = [ORACLE_CONTACT_SRC, LU.ORACLE_LINK_SRC, os.path.join(HERE, "wrench_oracle", "wrench_oracle.c"),
                os.path.join(ROOT, "oracle", "dflex_oracle.c"), os.path.join(ROOT, "include", "dfx.h")]
        if _stale(path, deps):
            real = ["-DREAL=double"] if precision == "f64" else ["-fcx-limited-range", "-DORACLE_COMPLEX", "-DREAL=double _Complex"]
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall",
                                   "-Wno-unused-function"] + real + ["-o", path, ORACLE_CONTACT_SRC, "-lm"])
        lib = ctypes.CDLL(path)
        S, I, Dbl = ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_double
        lib.oracle_contact_state.argtypes = [S, I] + [_D] * 5
        lib.oracle_contact_rollout.argtypes = [S, I, I, I, Dbl] + [_D] * 5
        if precision == "c64":
            lib.oracle_contact_state_gradient.argtypes = [S, Dbl] + [_D] * 7
            lib.oracle_contact_rollout_gradient.argtypes = [S, I, I, I, Dbl, Dbl] + [_D] * 10
        assert lib.oracle_real_bytes() == {"f64": 8, "c64": 16}[precision]
        _oracle_libs[precision] = lib
    return _oracle_libs[precision]


_p, _f64 = LU._p, LU._f64


class ContactOracle(Oracle):
    """Oracle plus the contact state (fp64), its exact gradient and the rollout ending in it (complex step, one environment)."""

    def set_ground(self, on):
        self.struct.ground = int(bool(on))

    def contact_state(self, q, qd):
        """(contact_f [n, C, 3], contact_height [n, C], body_f_contact [n, L, 6]) fp64"""
        d = self.desc
        q, qd = _f64(q), _f64(qd)
        n = q.size // d.Q
        out = (np.empty((n, d.C, 3)), np.empty((n, d.C)), np.empty((n, d.L, 6)))
        _oracle_contact_lib("f64").oracle_contact_state(ctypes.byref(self.struct), n, _p(q), _p(qd), *(_p(o) for o in out))
        return out

    def contact_state_gradient(self, q, qd, g_f, g_h, g_body, h=1e-30):
        """(gq [Q], gqd [D]) of sum(g . (contact_f, contact_height, body_f_contact)) for ONE environment, exact (complex step)"""
        d = self.desc
        gq, gqd = np.zeros(d.Q), np.zeros(d.D)
        _oracle_contact_lib("c64").oracle_contact_state_gradient(ctypes.byref(self.struct), float(h), _p(_f64(q)), _p(_f64(qd)),
                                                                 _p(_f64(g_f)), _p(_f64(g_h)), _p(_f64(g_body)), _p(gq), _p(gqd))
        return gq, gqd

    def rollout(self, q, qd, act, musc, substeps, mm_freq, dt):
        """ONE environment, act [T, D]: the contact state (f [C, 3], height [C], body [L, 6]) at the end of T env-steps"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        out = np.empty(d.C * 4 + d.L * 6)
        _oracle_contact_lib("f64").oracle_contact_rollout(ctypes.byref(self.struct), act.shape[0], substeps, mm_freq, float(dt),
                                                          _p(_f64(q)), _p(_f64(qd)), _p(_f64(act)), _p(_f64(musc)), _p(out))
        C = d.C
        return out[:C * 3].reshape(C, 3), out[C * 3:C * 4], out[C * 4:].reshape(d.L, 6)

    def rollout_gradient(self, q, qd, act, musc, g, substeps, mm_freq, dt, h=1e-30):
        """(gq [Q], gqd [D], gact [T, D]) of sum(g . final contact state) of rollout, exact (complex step)"""
        d = self.desc
        act = np.asarray(act, np.float64).reshape(-1, d.D)
        gq, gqd, gact = np.zeros(d.Q), np.zeros(d.D), np.zeros(act.size)
        _oracle_contact_lib("c64").oracle_contact_rollout_gradient(
            ctypes.byref(self.struct), act.shape[0], substeps, mm_freq, float(dt), float(h), _p(_f64(q)), _p(_f64(qd)),
            _p(_f64(act)), _p(_f64(musc)), _p(_f64(g[0])), _p(_f64(g[1])), _p(_f64(g[2])), _p(gq), _p(gqd), _p(gact))
        return gq, gqd, gact.reshape(act.shape)


def oracle_of(name, ground=None):
    model, ne = model_of(name)
    desc, _ = articulation_from_model(model, ne, ground=ground)
    return ContactOracle(desc)


# ------------------------------------------------------------------ models and batches
def contacts_sorted(desc):
    """whether the Model's contacts are already grouped by body in ascending order (the pack's order)"""
    b = np.asarray(desc.arrays["contact_body0"][:desc.C])
    return bool(np.all(b[1:] >= b[:-1]))


def batch(name, n=N, seed=3):
    """(desc, q [n, Q], qd [n, D], cotangents (g_f [n, C, 3], g_h [n, C], g_body [n, L, 6])) fp32: link_util.batch's states
    (the step batches with every regime row, every third environment's quaternions off the unit sphere), every fifth environment
    at rest (qd = 0: resting contacts, |v_t| = 0), standard-normal cotangents -- every fourth environment with height
    cotangents only"""
    desc, q, qd, _ = LU.batch(name, n, seed)
    qd = qd.copy()
    qd[4::5] = 0.0
    rng = np.random.default_rng([seed, 13])
    C, L = desc.C, desc.L
    g_f = rng.standard_normal((n, C, 3)).astype(np.float32)
    g_h = rng.standard_normal((n, C)).astype(np.float32)
    g_body = rng.standard_normal((n, L, 6)).astype(np.float32)
    g_f[2::4] = 0.0
    g_body[2::4] = 0.0
    return desc, q, qd, (g_f, g_h, g_body)


# ------------------------------------------------------------------ error measures
# Forces are ke (up to 4e4 N/m) times millimetre depths of metre-sized positions: a depth carries an absolute fp32 rounding of
# about |p| 2^-23, so a force one of ke |p| 2^-23.  Each environment's force and torque blocks are normalised by their largest
# |ref| but never by less than this floor, so a point at the edge of contact is not measured against a zero force.
def force_floor(desc, ref_h):
    """[n]: max ke of the model times max(1, max |height|) of the environment times 2^-23 (N)"""
    ke = float(np.max(desc.arrays["shape_materials"].reshape(-1, 4)[:, 0])) if desc.C else 0.0
    ps = np.maximum(1.0, np.abs(np.asarray(ref_h, np.float64)).max(axis=1)) if desc.C else np.ones(len(ref_h))
    return ke * ps * 2.0 ** -23


FWD_BLOCKS = (("f", 0, None), ("height", 1, None), ("body_tau", 2, slice(0, 3)), ("body_F", 2, slice(3, 6)))


def forward_errors(desc, got, ref):
    """{block: [n]}: per environment, the largest |got - ref| of the block over max(its largest |ref|, the force floor;
    heights: 1 m)"""
    n = len(ref[1])
    floor = force_floor(desc, ref[1])
    out = {}
    for bname, k, sl in FWD_BLOCKS:
        g, r = np.asarray(got[k], np.float64), np.asarray(ref[k], np.float64)
        if sl is not None:
            g, r = g[..., sl], r[..., sl]
        g, r = g.reshape(n, -1), r.reshape(n, -1)
        if r.shape[1] == 0:
            continue
        scale = np.abs(r).max(axis=1)
        scale = np.maximum(scale, 1.0 if bname == "height" else floor)
        out[bname] = np.abs(g - r).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


# A gradient block is normalised by its largest |exact| component, but never by less than GRAD_FLOOR_REL of the environment's largest
# gradient component: a block a million times smaller than the rest (the velocity gradient of a point held at its Coulomb cap) is
# within the rounding of the sums that form the large ones (2^-23 times ~100 terms).
GRAD_FLOOR_REL = 100 * 2.0 ** -23


def grad_errors(desc, gq, gqd, exact_gq, exact_gqd):
    """{block: [n]} per environment and gradient block (link_util.grad_blocks), with the floor GRAD_FLOOR_REL"""
    got, ex = [gq, gqd], [np.asarray(exact_gq, np.float64), np.asarray(exact_gqd, np.float64)]
    env_max = np.maximum(np.abs(ex[0]).max(axis=1, initial=0.0), np.abs(ex[1]).max(axis=1, initial=0.0))
    out = {}
    for bname, gi, sl in LU.grad_blocks(desc):
        g = np.asarray(got[gi], np.float64)[:, sl]
        x = ex[gi][:, sl]
        if g.shape[1] == 0:
            continue
        scale = np.maximum(np.abs(x).max(axis=1), GRAD_FLOOR_REL * env_max)
        out[bname] = np.abs(g - x).max(axis=1) / np.where(scale > 0, scale, 1.0)
    return out


_exact_cache = {}


def _key(*arrays):
    return tuple(None if a is None else a.tobytes() for a in arrays)


def exact_contact_gradients(name, o, q, qd, g):
    """(gq [n, Q], gqd [n, D]) exact, per environment (cached per model, ground and inputs)"""
    key = (name, o.struct.ground) + _key(q, qd, *g)
    if key not in _exact_cache:
        res = [o.contact_state_gradient(q[e], qd[e], g[0][e], g[1][e], g[2][e]) for e in range(q.shape[0])]
        _exact_cache[key] = (np.stack([r[0] for r in res]), np.stack([r[1] for r in res]))
    return _exact_cache[key]


def reference(name, o, q, qd):
    """the fp64 contact state of the batch (cached)"""
    key = ("fwd", name, o.struct.ground) + _key(q, qd)
    if key not in _exact_cache:
        _exact_cache[key] = o.contact_state(q, qd)
    return _exact_cache[key]


# ------------------------------------------------------------------ switching surfaces
def one_ulp_sensitive(o, q, qd, e, rel=1e-3):
    """whether environment e sits on a contact switching surface: its fp64 contact state moves by more than `rel` of its scale
    when (q, qd) move by one fp32 ulp (each component up, then down)"""
    q1, qd1 = q[e:e + 1].astype(np.float32), qd[e:e + 1].astype(np.float32)
    base = o.contact_state(q1, qd1)
    scale = max(float(np.abs(base[0]).max(initial=0.0)), float(np.abs(base[2]).max(initial=0.0)), 1e-3)
    for d in (np.inf, -np.inf):
        moved = o.contact_state(np.nextafter(q1, np.float32(d)), np.nextafter(qd1, np.float32(d)))
        if max(float(np.abs(a - b).max(initial=0.0)) for a, b in zip(moved, base)) > rel * scale:
            return True
    return False


# ------------------------------------------------------------------ the convention check
def convention_errors(qd_on, qd_ext, qd_off):
    """[n] from the qd' of three one-substep env-steps of the same states -- ground on; ground off under f_ext = body_f_contact;
    ground off -- per environment, max |qd_ext - qd_on| over max |qd_on - qd_off| (the contact's own effect on the env-step).
    Environments without a penetrating point, or whose env-step is not finite on one of the three paths, are 0."""
    qd_on, qd_ext, qd_off = (np.asarray(x, np.float64).reshape(len(qd_on), -1) for x in (qd_on, qd_ext, qd_off))
    effect = np.abs(qd_on - qd_off).max(axis=1)
    ok = (effect > 0) & np.isfinite(qd_on).all(axis=1) & np.isfinite(qd_ext).all(axis=1) & np.isfinite(qd_off).all(axis=1)
    return np.where(ok, np.abs(qd_ext - qd_on).max(axis=1) / np.where(ok, effect, 1.0), 0.0)


# ------------------------------------------------------------------ a rollout ending in the contact state
ROLLOUT_T = 3           # env-steps


def rollout_case(name, n, seed=5):
    """(model, meta, q0 [n, Q], qd0 [n, D], acts [T, n, D]) of golden case 0 (link_util.tether_case with T = ROLLOUT_T)"""
    import wrench_util as W
    model, meta, inp = W.golden_batch(name, n)
    rng = np.random.default_rng(seed)
    acts = np.stack([(inp["act"] * rng.uniform(0.5, 1.5, inp["act"].shape)).astype(np.float32) for _ in range(ROLLOUT_T)])
    return model, meta, inp["q0"], inp["qd0"], acts


def rollout_errors(o, q0, qd0, acts, g, gq, gqd, gact, S, mm, dt, envs):
    """{gq, gqd, gact: worst over environments `envs` of rel_err against the oracle's exact gradient}"""
    err = dict(gq=0.0, gqd=0.0, gact=0.0)
    for e in envs:
        ex = o.rollout_gradient(q0[e], qd0[e], acts[:, e], None, tuple(x[e] for x in g), S, mm, dt)
        for k, got, x in zip(("gq", "gqd", "gact"), (gq[e], gqd[e], gact[:, e]), ex):
            err[k] = max(err[k], rel_err(got, x))
    return err
