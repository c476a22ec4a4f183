"""Single-articulation description ("ModelPack" input) extracted from a finalized Model.

The reference stores every Model tensor tiled over the environments (``dflex/dflex/model.py:1646-1879``:
env ``e``'s links are rows ``e*L .. e*L+L-1``, ``joint_parent`` / ``contact_body0`` /
``contact_material`` / ``muscle_links`` are GLOBAL indices).  All environments of a DFlexEnv are copies
of one articulation (``envs/ant.py:97-124`` with ``env_dist = 0``), so the kernels take the
description of ONE articulation and share it across the batch.  This module slices environment 0 out
of the tiled tensors, makes the indices env-local, and checks that every other environment is
identical (raising otherwise: heterogeneous batches are not supported by the fused kernels).
"""
import ctypes

import numpy as np

_F = ctypes.POINTER(ctypes.c_float)
_I = ctypes.POINTER(ctypes.c_int)


class DfxModelDesc(ctypes.Structure):
    """ctypes mirror of ``DfxModelDesc`` in include/dfx.h (keep field order in sync)."""

    _fields_ = [
        ("link_count", ctypes.c_int), ("dof_count", ctypes.c_int), ("coord_count", ctypes.c_int),
        ("contact_count", ctypes.c_int), ("muscle_count", ctypes.c_int), ("waypoint_count", ctypes.c_int),
        ("shape_count", ctypes.c_int), ("ground", ctypes.c_int), ("gravity", ctypes.c_float * 3),
        ("joint_type", _I), ("joint_parent", _I), ("joint_q_start", _I), ("joint_qd_start", _I),
        ("joint_X_pj", _F), ("joint_X_cm", _F), ("joint_axis", _F), ("body_I_m", _F),
        ("joint_target_ke", _F), ("joint_target_kd", _F), ("joint_limit_ke", _F), ("joint_limit_kd", _F),
        ("joint_target", _F), ("joint_limit_lower", _F), ("joint_limit_upper", _F), ("joint_armature", _F),
        ("contact_body0", _I), ("contact_point0", _F), ("contact_dist", _F), ("contact_material", _I),
        ("shape_materials", _F),
        ("muscle_start", _I), ("muscle_links", _I), ("muscle_points", _F),
    ]


class DfxActionMap(ctypes.Structure):
    """include/dfx.h DfxActionMap: the policy-output -> actuation map folded into dfx_step_*_mapped."""
    _fields_ = [("num_act", ctypes.c_int), ("offset", ctypes.c_int), ("is_muscle", ctypes.c_int),
                ("pre_scale", ctypes.c_float), ("pre_bias", ctypes.c_float), ("drive_scale", ctypes.c_float),
                ("strength", ctypes.c_void_p)]


class DfxExternalWrench(ctypes.Structure):
    """include/dfx.h DfxExternalWrench: per-environment link wrenches [N, L, 6] (torque, force at the centre of mass; world
    axes) for the _ex step entries, and where the adjoint writes their cotangent (NULL: skip)."""
    _fields_ = [("f_ext", ctypes.c_void_p), ("g_f_ext", ctypes.c_void_p)]


class DfxDerived(ctypes.Structure):
    """ctypes mirror of ``DfxDerived`` in include/dfx.h."""

    _fields_ = [(n, ctypes.c_void_p) for n in (
        "body_X_sc", "body_X_sm", "joint_S_s", "body_v_s", "body_a_s", "body_f_s", "body_ft_s",
        "joint_tau", "joint_qdd", "H", "L")]


PER_LINK = ("joint_type", "joint_parent", "joint_X_pj", "joint_X_cm", "joint_axis", "body_I_m",
            "joint_target_ke", "joint_target_kd", "joint_limit_ke", "joint_limit_kd")
PER_COORD = ("joint_target", "joint_limit_lower", "joint_limit_upper")
PER_DOF = ("joint_armature",)


class ArticulationDesc:
    """Host-side numpy arrays of one articulation + the ctypes struct pointing at them."""

    def __init__(self, arrays, counts, gravity, ground):
        self.arrays = arrays          # keeps the numpy buffers alive
        self.counts = counts
        self.gravity = tuple(float(g) for g in gravity)
        self.ground = bool(ground)

    @property
    def L(self):
        return self.counts["link_count"]

    @property
    def D(self):
        return self.counts["dof_count"]

    @property
    def Q(self):
        return self.counts["coord_count"]

    @property
    def C(self):
        return self.counts["contact_count"]

    @property
    def M(self):
        return self.counts["muscle_count"]

    def as_struct(self):
        d = DfxModelDesc()
        for key, value in self.counts.items():
            setattr(d, key, int(value))
        d.ground = int(self.ground)
        d.gravity = (ctypes.c_float * 3)(*self.gravity)
        for name, ctype in DfxModelDesc._fields_:
            if ctype in (_F, _I):
                arr = self.arrays[name]
                want = np.float32 if ctype is _F else np.int32
                assert arr.dtype == want and arr.flags["C_CONTIGUOUS"], name
                setattr(d, name, arr.ctypes.data_as(ctype))
        return d


def _get(model, name):
    """Fetch a Model field as a numpy array (accepts torch tensors, numpy arrays or npz dicts)."""
    value = model[name] if isinstance(model, dict) else getattr(model, name)
    if hasattr(value, "detach"):
        value = value.detach().cpu().numpy()
    return np.asarray(value)


def articulation_from_model(model, num_envs=None, ground=None, gravity=None):
    """Build the ArticulationDesc of environment 0 and verify the batch is homogeneous.

    ``model`` is a finalized Model-like object (attributes) or a dict of arrays whose fields follow
    the reference names.  ``num_envs`` defaults to ``articulation_count``.
    """
    jtype = _get(model, "joint_type").astype(np.int32)
    n_links_total = jtype.shape[0]
    if num_envs is None:
        num_envs = int(_get(model, "articulation_joint_start").shape[0] - 1)
    if num_envs <= 0 or n_links_total % num_envs:
        raise ValueError("link_count %d is not a multiple of the number of articulations %d" % (n_links_total, num_envs))
    L = n_links_total // num_envs
    q_start = _get(model, "joint_q_start").astype(np.int64)
    qd_start = _get(model, "joint_qd_start").astype(np.int64)
    Q = int(q_start[-1]) // num_envs
    D = int(qd_start[-1]) // num_envs
    if int(q_start[-1]) != Q * num_envs or int(qd_start[-1]) != D * num_envs:
        raise ValueError("joint coordinate / dof counts are not multiples of the number of environments")

    def tiled(name, per_env, dtype, local_offset=0, keep_negative=True):
        full = _get(model, name)
        if per_env and full.ndim == 1 and full.shape[0] > num_envs * per_env:
            # the reference indexes per-coordinate arrays by the GLOBAL coordinate index
            # (sim.py:1448-1450), so surplus tail entries (envs/hopper.py:119 grows joint_target
            # by one element per env) are never read
            full = full[: num_envs * per_env]
        full = full.reshape(num_envs, per_env, *full.shape[1:]) if per_env else full.reshape(num_envs, 0)
        first = full[0].copy()
        if local_offset:
            # indices grow by `local_offset` per environment; negatives (-1 parents) stay
            offs = (np.arange(num_envs) * local_offset).reshape((num_envs,) + (1,) * (full.ndim - 1))
            shifted = np.where(full >= 0, full - offs, full) if keep_negative else full - offs
            if not np.array_equal(shifted, np.broadcast_to(first, shifted.shape)):
                raise ValueError("field %s differs between environments (heterogeneous batch)" % name)
        elif not np.array_equal(full, np.broadcast_to(first, full.shape)):
            raise ValueError("field %s differs between environments (heterogeneous batch)" % name)
        return np.ascontiguousarray(first.astype(dtype))

    arrays = {}
    arrays["joint_type"] = tiled("joint_type", L, np.int32)
    arrays["joint_parent"] = tiled("joint_parent", L, np.int32, local_offset=L)
    qs = q_start[: L + 1].astype(np.int32)
    qds = qd_start[: L + 1].astype(np.int32)
    for e in range(num_envs):
        if not (np.array_equal(q_start[e * L:(e + 1) * L + 1] - e * Q, qs) and
                np.array_equal(qd_start[e * L:(e + 1) * L + 1] - e * D, qds)):
            raise ValueError("joint_q_start / joint_qd_start differ between environments")
    arrays["joint_q_start"], arrays["joint_qd_start"] = np.ascontiguousarray(qs), np.ascontiguousarray(qds)
    for name in ("joint_X_pj", "joint_X_cm", "joint_axis", "body_I_m", "joint_target_ke", "joint_target_kd",
                 "joint_limit_ke", "joint_limit_kd"):
        arrays[name] = tiled(name, L, np.float32)
    for name in PER_COORD:
        arrays[name] = tiled(name, Q, np.float32)
    arrays["joint_armature"] = tiled("joint_armature", D, np.float32)

    # contacts (static list made by Model.collide); absent until collide() is called
    try:
        body0 = _get(model, "contact_body0")
    except (AttributeError, KeyError):
        body0 = np.zeros((0,), np.int32)
    c_total = int(body0.shape[0])
    if c_total % num_envs:
        raise ValueError("contact_count is not a multiple of the number of environments")
    C = c_total // num_envs
    shape_mat = _get(model, "shape_materials").astype(np.float32).reshape(-1, 4)
    if shape_mat.shape[0] % num_envs:
        raise ValueError("shape_count is not a multiple of the number of environments")
    S = shape_mat.shape[0] // num_envs
    if C:
        arrays["contact_body0"] = tiled("contact_body0", C, np.int32, local_offset=L)
        arrays["contact_point0"] = tiled("contact_point0", C, np.float32)
        arrays["contact_dist"] = tiled("contact_dist", C, np.float32)
        arrays["contact_material"] = tiled("contact_material", C, np.int32, local_offset=S)
    else:
        arrays["contact_body0"] = np.zeros((0,), np.int32)
        arrays["contact_point0"] = np.zeros((0, 3), np.float32)
        arrays["contact_dist"] = np.zeros((0,), np.float32)
        arrays["contact_material"] = np.zeros((0,), np.int32)
    if S:
        full = shape_mat.reshape(num_envs, S, 4)
        if not np.array_equal(full, np.broadcast_to(full[0], full.shape)):
            raise ValueError("shape_materials differ between environments")
        arrays["shape_materials"] = np.ascontiguousarray(full[0])
    else:
        arrays["shape_materials"] = np.zeros((0, 4), np.float32)

    # muscles
    try:
        mstart = _get(model, "muscle_start").astype(np.int64)
        mlinks = _get(model, "muscle_links").astype(np.int64)
        mpoints = _get(model, "muscle_points").astype(np.float32).reshape(-1, 3)
    except (AttributeError, KeyError):
        mstart, mlinks, mpoints = np.zeros((1,), np.int64), np.zeros((0,), np.int64), np.zeros((0, 3), np.float32)
    m_total = int(mstart.shape[0] - 1)
    if m_total % num_envs or mlinks.shape[0] % num_envs:
        raise ValueError("muscle counts are not multiples of the number of environments")
    M, W = m_total // num_envs, mlinks.shape[0] // num_envs
    if M:
        ms = mstart[: M + 1]
        for e in range(num_envs):
            if not np.array_equal(mstart[e * M:(e + 1) * M + 1] - e * W, ms):
                raise ValueError("muscle_start differs between environments")
        ml = mlinks.reshape(num_envs, W) - (np.arange(num_envs) * L)[:, None]
        mp = mpoints.reshape(num_envs, W, 3)
        if not (np.array_equal(ml, np.broadcast_to(ml[0], ml.shape)) and np.array_equal(mp, np.broadcast_to(mp[0], mp.shape))):
            raise ValueError("muscle way-points differ between environments")
        arrays["muscle_start"] = np.ascontiguousarray(ms.astype(np.int32))
        arrays["muscle_links"] = np.ascontiguousarray(ml[0].astype(np.int32))
        arrays["muscle_points"] = np.ascontiguousarray(mp[0])
    else:
        arrays["muscle_start"] = np.zeros((1,), np.int32)
        arrays["muscle_links"] = np.zeros((0,), np.int32)
        arrays["muscle_points"] = np.zeros((0, 3), np.float32)

    if gravity is None:
        gravity = _get(model, "gravity").astype(np.float32).reshape(3)
    if ground is None:
        ground = bool(model["ground"]) if isinstance(model, dict) else bool(getattr(model, "ground", True))
    counts = dict(link_count=L, dof_count=D, coord_count=Q, contact_count=C, muscle_count=M,
                  waypoint_count=W, shape_count=S)
    return ArticulationDesc(arrays, counts, gravity, ground), num_envs
