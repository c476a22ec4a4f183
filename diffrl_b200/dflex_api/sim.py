"""``dflex.sim``: the drop-in boundary.

``SemiImplicitIntegrator().forward(model, state_in, dt, substeps, mass_matrix_freq) -> State`` has the
signature and semantics of the reference (``dflex/dflex/sim.py:2182-2221``): ``substeps`` symplectic-Euler
substeps of ``dt/substeps`` with the actuation held constant, the joint-space inertia re-factorised
every ``mass_matrix_freq`` substeps, gradients flowing to ``state_in.joint_q / joint_qd / joint_act``
and ``model.muscle_activation``.  Underneath, one fused sm_90a kernel per env-step (and one for its
adjoint) replaces the reference's tape of 10-11 generated kernels per substep.

``state_in.body_f_ext`` (optional, [N*L, 6] or [N, L, 6]): external link wrenches (torque, force at the centre of mass, world
axes; include/dfx.h DfxExternalWrench) held over the env-step's substeps, differentiable.  A returned State carries none.
"""
import torch

from . import config
from .model import (GEO_BOX, GEO_CAPSULE, GEO_MESH, GEO_NONE, GEO_PLANE, GEO_SDF, GEO_SPHERE, JOINT_BALL,  # noqa: F401
                    JOINT_FIXED, JOINT_FREE, JOINT_PRISMATIC, JOINT_REVOLUTE, Mesh, Model, ModelBuilder, State,
                    model_from_articulation)

_DERIVED = ("body_X_sc", "body_X_sm", "joint_S_s", "body_v_s", "body_a_s", "body_f_s", "body_ft_s",
            "joint_tau", "joint_qdd")


def _engine_for(model):
    """The device-resident ModelPack of ``model`` (built on first use, rebuilt after collide())."""
    from ..engine import ArticulationEngine
    from ..modelpack import ArticulationDesc, articulation_from_model  # noqa: F401
    if model._engine is None:
        n = int(model.articulation_count)
        arrays = getattr(model, "_articulation_arrays", None)
        if arrays is not None:
            # tiled from one articulation: the per-env description is already at hand
            import numpy as np
            one = {k: np.asarray(v) for k, v in arrays.items()}
            one["ground"] = bool(model.ground)
            desc, _ = articulation_from_model(one, 1)
            model._engine = ArticulationEngine(desc, n, model.adapter)
        else:
            model._engine = ArticulationEngine.from_model(model, model.adapter, n)
        model._engine_key = None
    g = model.gravity
    key = (id(g), g._version, bool(model.ground))
    if key != model._engine_key:      # envs assign model.gravity / model.ground after finalize()
        model._engine.set_gravity([float(x) for x in g.detach().cpu().tolist()], bool(model.ground))
        model._engine_key = key
    return model._engine


def _derived_getattr(self, name):
    """Derived State fields (values of the LAST substep, reference model.py:375-388) are produced on
    demand by re-running the step with dumps enabled -- rendering/debugging only, never on the hot path."""
    if name == "joint_act" and "_act_proto" in self.__dict__:     # zero actuation, materialised on first use only
        self.__dict__["joint_act"] = torch.zeros_like(self.__dict__["_act_proto"])
        return self.__dict__["joint_act"]
    if name in _DERIVED and "_derive_ctx_mapped" in self.__dict__:
        # the step ran with the action map folded in: form the actuation arrays it used, then fall through
        engine, q, qd, raw, amap, substeps, mm_freq, dt = self.__dict__.pop("_derive_ctx_mapped")
        offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = amap
        from ..env_ops import ActionMapFunction
        width = engine.M if is_muscle else engine.D
        with torch.no_grad():
            _, drive = ActionMapFunction.apply(engine.N, width, offset, pre_scale, pre_bias, drive_scale, strength, raw.view(engine.N, -1))
        act = torch.zeros(engine.N * engine.D, device=q.device) if is_muscle else drive
        self.__dict__["_derive_ctx"] = (engine, q, qd, act, drive if is_muscle else None, substeps, mm_freq, dt)
    if name in _DERIVED and "_derive_ctx" in self.__dict__:
        engine, q, qd, act, musc, substeps, mm_freq, dt = self.__dict__["_derive_ctx"]
        _, _, _, dumps = engine.forward(q, qd, act, musc, substeps, mm_freq, dt, want_tape=False, derived=list(_DERIVED),
                                        f_ext=self.__dict__.get("_derive_f_ext"))
        for key, value in dumps.items():
            self.__dict__[key] = value
        return self.__dict__[name]
    raise AttributeError(name)


State.__getattr__ = _derived_getattr


def _wrench_in(state):
    """``state.body_f_ext`` when set (no derived-field lookup)."""
    return state.__dict__.get("body_f_ext")


def _wrench_args(f_ext):
    return () if f_ext is None else (f_ext,)


def fused_mapped_forward(model, state_in, dt, substeps, mass_matrix_freq, raw_actions, amap):
    """``SemiImplicitIntegrator.forward`` with the env's action map folded into the launch (the env layer's fast path,
    ``envs/base.py:_fused_step``): returns (State, used) where ``used`` are the clipped / affinely mapped actions.
    ``amap`` = (offset, pre_scale, pre_bias, drive_scale, strength, is_muscle).  Reads ``state_in.body_f_ext``."""
    from ..engine import MappedSimStepFunction
    engine = _engine_for(model)
    f_ext = _wrench_in(state_in)
    q_new, qd_new, used = MappedSimStepFunction.apply(engine, int(substeps), int(mass_matrix_freq), float(dt), amap,
                                                      state_in.joint_q, state_in.joint_qd, raw_actions, *_wrench_args(f_ext))
    out = State()
    out.particle_count, out.link_count = model.particle_count, model.link_count
    out.joint_q, out.joint_qd = q_new, qd_new
    out.__dict__["_act_proto"] = model.joint_qd
    out.__dict__["_derive_ctx_mapped"] = (engine, state_in.joint_q.detach(), state_in.joint_qd.detach(), raw_actions.detach(), amap,
                                          int(substeps), int(mass_matrix_freq), float(dt))
    if f_ext is not None:
        out.__dict__["_derive_f_ext"] = f_ext.detach()
    return out, used


def fused_env_step(model, state_in, dt, substeps, mass_matrix_freq, raw_actions, amap, tparams, progress, start_q, start_qd, nan_guard=False):
    """env.step() as one launch (``env_ops.EnvStepFunction`` over ``dfx_env_step_forward / _backward``): the simulation step with
    the action map folded in and the env transition as its epilogue.  Returns (State of the NEXT step's start, (obs_before_reset,
    rew, reset, actions_next, progress_next, obs_next)).  ``nan_guard``: non-finite cotangents of (q, qd, actions) become 0
    (the reference's humanoid.py:196-206 hooks; the wrench's cotangent too).  Reads ``state_in.body_f_ext``."""
    from ..env_ops import EnvStepFunction
    engine = _engine_for(model)
    f_ext = _wrench_in(state_in)
    (obs_before, rew, reset, q_next, qd_next, actions_next, progress_next, obs_next) = EnvStepFunction.apply(
        engine, int(substeps), int(mass_matrix_freq), float(dt), amap, tparams, bool(nan_guard), progress, start_q, start_qd,
        state_in.joint_q, state_in.joint_qd, raw_actions, *_wrench_args(f_ext))
    out = State()
    out.particle_count, out.link_count = model.particle_count, model.link_count
    out.joint_q, out.joint_qd = q_next.view(-1), qd_next.view(-1)
    out.__dict__["_act_proto"] = model.joint_qd
    out.__dict__["_derive_ctx_mapped"] = (engine, state_in.joint_q.detach(), state_in.joint_qd.detach(), raw_actions.detach(), amap,
                                          int(substeps), int(mass_matrix_freq), float(dt))
    if f_ext is not None:
        out.__dict__["_derive_f_ext"] = f_ext.detach()
    return out, (obs_before, rew, reset, actions_next, progress_next, obs_next)


class SemiImplicitIntegrator:
    """Semi-implicit (symplectic) Euler integrator for articulated rigid bodies."""

    def __init__(self):
        pass

    def forward(self, model, state_in, dt, substeps, mass_matrix_freq):
        engine = _engine_for(model)
        musc = model.muscle_activation if engine.M else None
        f_ext = _wrench_in(state_in)
        if config.no_grad:
            with torch.no_grad():
                q = state_in.joint_q if state_in.joint_q.is_contiguous() else state_in.joint_q.contiguous()
                qd = state_in.joint_qd if state_in.joint_qd.is_contiguous() else state_in.joint_qd.contiguous()
                engine.forward(q, qd, state_in.joint_act, musc, substeps, mass_matrix_freq, dt,
                               want_tape=False, out=(q.view(-1), qd.view(-1)), f_ext=f_ext)
                if q is not state_in.joint_q:
                    state_in.joint_q.copy_(q)
                    state_in.joint_qd.copy_(qd)
            return state_in
        from ..engine import SimStepFunction
        q_new, qd_new = SimStepFunction.apply(engine, int(substeps), int(mass_matrix_freq), float(dt),
                                              state_in.joint_q, state_in.joint_qd, state_in.joint_act, musc, *_wrench_args(f_ext))
        out = State()
        out.particle_count, out.link_count = model.particle_count, model.link_count
        out.joint_q, out.joint_qd = q_new, qd_new
        out.__dict__["_act_proto"] = model.joint_qd      # out.joint_act: zeros, created lazily (State.__getattr__)
        out.__dict__["_derive_ctx"] = (engine, state_in.joint_q.detach(), state_in.joint_qd.detach(),
                                       state_in.joint_act.detach(), None if musc is None else musc.detach(),
                                       int(substeps), int(mass_matrix_freq), float(dt))
        if f_ext is not None:
            out.__dict__["_derive_f_ext"] = f_ext.detach()
        if config.verify_fp:
            assert torch.isfinite(q_new).all() and torch.isfinite(qd_new).all(), "non-finite state after integration"
        return out
