"""Fused env epilogue ops (observation + reward + termination flags of the free-root walkers) as ONE
autograd.Function over the C ABI (``dfx_walker_obs_forward / _backward`` in include/dfx.h)."""
import ctypes

import torch

from . import _capi
from .engine import recompute_adjoint


class DfxWalkerParams(ctypes.Structure):
    """ctypes mirror of ``DfxWalkerParams`` in include/dfx.h (keep field order in sync)."""

    _fields_ = [
        ("num_q", ctypes.c_int), ("num_qd", ctypes.c_int), ("num_act", ctypes.c_int), ("num_obs", ctypes.c_int),
        ("obs_has_actions", ctypes.c_int), ("height_mode", ctypes.c_int), ("action_penalty_abs", ctypes.c_int),
        ("early_termination", ctypes.c_int), ("check_invalid", ctypes.c_int), ("zero_reward_on_invalid", ctypes.c_int),
        ("episode_length", ctypes.c_int),
        ("joint_vel_scale", ctypes.c_float), ("termination_height", ctypes.c_float),
        ("termination_tolerance", ctypes.c_float), ("height_rew_scale", ctypes.c_float), ("action_penalty", ctypes.c_float),
        ("target", ctypes.c_float * 3), ("inv_start_rot", ctypes.c_float * 4),
        ("basis_heading", ctypes.c_float * 3), ("basis_up", ctypes.c_float * 3),
    ]


class DfxPlanarParams(ctypes.Structure):
    """ctypes mirror of ``DfxPlanarParams`` in include/dfx.h (keep field order in sync)."""

    _fields_ = [
        ("num_q", ctypes.c_int), ("num_qd", ctypes.c_int), ("num_act", ctypes.c_int), ("num_obs", ctypes.c_int),
        ("kind", ctypes.c_int), ("early_termination", ctypes.c_int), ("zero_actions_on_reset", ctypes.c_int),
        ("episode_length", ctypes.c_int),
        ("termination_height", ctypes.c_float), ("termination_height_tolerance", ctypes.c_float),
        ("termination_angle", ctypes.c_float), ("height_rew_scale", ctypes.c_float), ("action_penalty", ctypes.c_float),
        ("pole_angle_penalty", ctypes.c_float), ("pole_velocity_penalty", ctypes.c_float),
        ("cart_position_penalty", ctypes.c_float), ("cart_velocity_penalty", ctypes.c_float),
    ]


class DfxEnvTransition(ctypes.Structure):
    """ctypes mirror of ``DfxEnvTransition`` in include/dfx.h (keep field order in sync)."""

    _fields_ = [("kind", ctypes.c_int), ("walker", DfxWalkerParams), ("planar", DfxPlanarParams)] + [
        (n, ctypes.c_void_p) for n in ("progress", "start_q", "start_qd", "obs_before", "rew", "reset", "q_next", "qd_next",
                                       "actions_next", "progress_next", "obs_next")]


class DfxEnvTransitionAdj(ctypes.Structure):
    """ctypes mirror of ``DfxEnvTransitionAdj`` in include/dfx.h (keep field order in sync)."""

    _fields_ = [("kind", ctypes.c_int), ("walker", DfxWalkerParams), ("planar", DfxPlanarParams)] + [
        (n, ctypes.c_void_p) for n in ("q_sim", "qd_sim", "used", "reset", "g_obs_before", "g_rew", "g_q_next", "g_qd_next",
                                       "g_actions_next", "g_obs_next", "gq_sim", "gqd_sim", "g_used")]


def _bind(lib):
    if getattr(lib, "_walker_bound", False):
        return
    P = ctypes.POINTER(DfxWalkerParams)
    V = ctypes.c_void_p
    lib.dfx_walker_obs_forward.argtypes = [P, ctypes.c_int, V, V, V, V, V, V, V, V]
    lib.dfx_walker_obs_backward.argtypes = [P, ctypes.c_int, V, V, V, V, V, V, V, V, V]
    lib.dfx_walker_transition_forward.argtypes = [P, ctypes.c_int] + [V] * 15
    lib.dfx_walker_transition_backward.argtypes = [P, ctypes.c_int] + [V] * 14
    PP = ctypes.POINTER(DfxPlanarParams)
    lib.dfx_planar_transition_forward.argtypes = [PP, ctypes.c_int] + [V] * 15
    lib.dfx_planar_transition_backward.argtypes = [PP, ctypes.c_int] + [V] * 14
    I, F = ctypes.c_int, ctypes.c_float
    lib.dfx_action_map_forward.argtypes = [I, I, I, I, F, F, F, V, V, V, V, V]
    lib.dfx_action_map_backward.argtypes = [I, I, I, I, F, F, V, V, V, V, V, V]
    Dbl = ctypes.c_double
    lib.dfx_env_step_forward.argtypes = [V, I, I, I, Dbl, V, V, V, V, V, V, V, V, V, ctypes.POINTER(DfxEnvTransition), V]
    lib.dfx_env_step_backward.argtypes = [V, I, I, I, Dbl, V, V, V, V, ctypes.POINTER(DfxEnvTransitionAdj), V, V, V, V]
    if hasattr(lib, "dfx_env_step_backward_recompute"):
        lib.dfx_env_step_backward_recompute.argtypes = [V, I, I, I, Dbl, V, V, V, V, V, V, ctypes.POINTER(DfxEnvTransitionAdj), V, V, V, V]
    lib._walker_bound = True


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _c(t):
    return t if (t.is_contiguous() and t.dtype == torch.float32) else t.contiguous().float()


class WalkerObsFunction(torch.autograd.Function):
    """(q, qd, actions) -> (obs, rew, reset).  ``want_reward=False`` computes only the observation."""

    @staticmethod
    def forward(ctx, params, n, want_reward, progress, q, qd, actions):
        lib = _capi.lib()
        _bind(lib)
        q, qd, actions = _c(q.detach()), _c(qd.detach()), _c(actions.detach())
        dev = q.device
        obs = torch.empty((n, params.num_obs), dtype=torch.float32, device=dev)
        rew = torch.empty(n, dtype=torch.float32, device=dev) if want_reward else None
        reset = torch.empty(n, dtype=torch.long, device=dev) if want_reward else None
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        with torch.cuda.device(dev):
            code = lib.dfx_walker_obs_forward(ctypes.byref(params), n, _ptr(q), _ptr(qd), _ptr(actions),
                                              _ptr(progress) if want_reward else None, _ptr(obs), _ptr(rew), _ptr(reset), stream)
        _capi.check(code, "dfx_walker_obs_forward")
        ctx.params, ctx.n = params, n
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(q, qd, actions)
        ctx.shapes = None
        if want_reward:
            ctx.mark_non_differentiable(reset)
            return obs, rew, reset
        return obs

    @staticmethod
    def backward(ctx, g_obs, g_rew=None, g_reset=None):
        lib = _capi.lib()
        q, qd, actions = ctx.saved_tensors
        dev = q.device
        gq, gqd = torch.empty_like(q), torch.empty_like(qd)
        gact = torch.empty_like(actions) if ctx.needs_input_grad[6] else None
        g_obs = None if g_obs is None else _c(g_obs)
        g_rew = None if g_rew is None else _c(g_rew)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        with torch.cuda.device(dev):
            code = lib.dfx_walker_obs_backward(ctypes.byref(ctx.params), ctx.n, _ptr(q), _ptr(qd), _ptr(actions),
                                               _ptr(g_obs), _ptr(g_rew), _ptr(gq), _ptr(gqd), _ptr(gact), stream)
        _capi.check(code, "dfx_walker_obs_backward")
        return None, None, None, None, gq, gqd, gact


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


class WalkerTransitionFunction(torch.autograd.Function):
    """Everything env.step() does after the simulation step, in one launch (``dfx_walker_transition_forward``, or
    ``dfx_planar_transition_forward`` when ``params`` is a ``DfxPlanarParams``):
    (q, qd, actions) of the stepped state -> (obs_before_reset, rew, reset, q_next, qd_next, actions_next,
    progress_next, obs_next).  ``progress`` is the counter before the step; ``start_q`` / ``start_qd`` the state a
    terminated environment restarts from (constants for autograd)."""

    @staticmethod
    def forward(ctx, params, n, progress, start_q, start_qd, q, qd, actions):
        lib = _capi.lib()
        _bind(lib)
        q, qd, actions = _c(q.detach()), _c(qd.detach()), _c(actions.detach())
        start_q, start_qd = _c(start_q), _c(start_qd)
        dev = q.device
        f32 = dict(dtype=torch.float32, device=dev)
        obs_before = torch.empty((n, params.num_obs), **f32)
        obs_next = torch.empty((n, params.num_obs), **f32)
        rew = torch.empty(n, **f32)
        reset = torch.empty(n, dtype=torch.long, device=dev)
        progress_next = torch.empty(n, dtype=torch.long, device=dev)
        q_next, qd_next, actions_next = torch.empty_like(q), torch.empty_like(qd), torch.empty_like(actions)
        fwd = lib.dfx_planar_transition_forward if isinstance(params, DfxPlanarParams) else lib.dfx_walker_transition_forward
        with torch.cuda.device(dev):
            code = fwd(
                ctypes.byref(params), n, _ptr(q), _ptr(qd), _ptr(actions), _ptr(progress), _ptr(start_q), _ptr(start_qd),
                _ptr(obs_before), _ptr(rew), _ptr(reset), _ptr(q_next), _ptr(qd_next), _ptr(actions_next),
                _ptr(progress_next), _ptr(obs_next), _stream(dev))
        _capi.check(code, "dfx_*_transition_forward")
        ctx.params, ctx.n = params, n
        ctx.set_materialize_grads(False)      # absent cotangents arrive as None (NULL in the C ABI), not as zero fills
        ctx.save_for_backward(q, qd, actions, reset)
        ctx.mark_non_differentiable(reset, progress_next)
        return obs_before, rew, reset, q_next, qd_next, actions_next, progress_next, obs_next

    @staticmethod
    def backward(ctx, g_obs_before, g_rew, g_reset, g_q_next, g_qd_next, g_actions_next, g_progress, g_obs_next):
        lib = _capi.lib()
        q, qd, actions, reset = ctx.saved_tensors
        dev = q.device
        gq, gqd = torch.empty_like(q), torch.empty_like(qd)
        gact = torch.empty_like(actions) if ctx.needs_input_grad[7] else None
        cot = [None if g is None else _c(g) for g in (g_obs_before, g_rew, g_q_next, g_qd_next, g_actions_next, g_obs_next)]
        bwd = lib.dfx_planar_transition_backward if isinstance(ctx.params, DfxPlanarParams) else lib.dfx_walker_transition_backward
        with torch.cuda.device(dev):
            code = bwd(
                ctypes.byref(ctx.params), ctx.n, _ptr(q), _ptr(qd), _ptr(actions), _ptr(reset),
                *[_ptr(g) for g in cot], _ptr(gq), _ptr(gqd), _ptr(gact), _stream(dev))
        _capi.check(code, "dfx_*_transition_backward")
        return None, None, None, None, None, gq, gqd, gact


class ActionMapFunction(torch.autograd.Function):
    """raw policy output [n, A] -> (used, drive): used = clip(raw, -1, 1) * pre_scale + pre_bias (the env's
    ``actions``), drive [n * width] = zeros with drive[:, offset:offset+A] = (used * drive_scale) * strength (``joint_act`` or the
    muscle activations).  One launch forward, one backward (``dfx_action_map_forward / _backward``)."""

    @staticmethod
    def forward(ctx, n, width, offset, pre_scale, pre_bias, drive_scale, strength, raw):
        lib = _capi.lib()
        _bind(lib)
        raw = _c(raw.detach())
        num_act = raw.shape[-1]
        dev = raw.device
        used = torch.empty_like(raw)
        drive = torch.empty(n * width, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            code = lib.dfx_action_map_forward(n, num_act, width, offset, pre_scale, pre_bias, drive_scale, _ptr(strength), _ptr(raw),
                                              _ptr(used), _ptr(drive), _stream(dev))
        _capi.check(code, "dfx_action_map_forward")
        ctx.cfg = (n, num_act, width, offset, pre_scale, drive_scale)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(strength, raw)
        return used, drive

    @staticmethod
    def backward(ctx, g_used, g_drive):
        lib = _capi.lib()
        strength, raw = ctx.saved_tensors
        n, num_act, width, offset, pre_scale, drive_scale = ctx.cfg
        g_raw = torch.empty_like(raw)
        g_used = None if g_used is None else _c(g_used)
        g_drive = None if g_drive is None else _c(g_drive)
        with torch.cuda.device(raw.device):
            code = lib.dfx_action_map_backward(n, num_act, width, offset, pre_scale, drive_scale, _ptr(strength), _ptr(raw),
                                               _ptr(g_used), _ptr(g_drive), _ptr(g_raw), _stream(raw.device))
        _capi.check(code, "dfx_action_map_backward")
        return None, None, None, None, None, None, None, g_raw


def _addr(t):
    return None if t is None else t.data_ptr()


class EnvStepFunction(torch.autograd.Function):
    """env.step() as ONE launch forward and ONE backward (``dfx_env_step_forward / _backward``): the simulation step with the
    action map folded in (``MappedSimStepFunction``) and the transition (``WalkerTransitionFunction``) as its epilogue --
    (q, qd, raw policy output) -> (obs_before_reset, rew, reset, q_next, qd_next, actions_next, progress_next, obs_next), the same
    values bit for bit.  ``amap`` = (offset, pre_scale, pre_bias, drive_scale, strength, is_muscle); ``params`` a
    ``DfxWalkerParams`` or ``DfxPlanarParams``; ``progress`` the counter before the step; ``start_q`` / ``start_qd`` the state a
    terminated environment restarts from (constants for autograd); ``nan_guard``: non-finite input cotangents become 0 (the
    reference's gradient hooks on the state and the clipped actions, envs/humanoid.py:196-206)."""

    @staticmethod
    def forward(ctx, engine, substeps, mm_freq, dt, amap, params, nan_guard, progress, start_q, start_qd, q, qd, raw):
        from .modelpack import DfxActionMap
        lib = engine.lib
        _bind(lib)
        offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = amap
        dev = engine.device
        q, qd, raw = _c(q.detach()), _c(qd.detach()), _c(raw.detach())
        start_q, start_qd = _c(start_q), _c(start_qd)
        n, A = engine.N, raw.shape[-1]
        m = DfxActionMap(int(A), int(offset), int(bool(is_muscle)), float(pre_scale), float(pre_bias), float(drive_scale), strength.data_ptr())
        f32 = dict(dtype=torch.float32, device=dev)
        q_sim, qd_sim, used = torch.empty_like(q), torch.empty_like(qd), torch.empty_like(raw)
        need = any(ctx.needs_input_grad[10:13])
        ctx.nan_guard = nan_guard
        ctx.recompute = recompute_adjoint()
        tape = torch.empty(engine.tape_floats(substeps, mm_freq), **f32) if (need and not ctx.recompute) else None
        obs_before = torch.empty((n, params.num_obs), **f32)
        obs_next = torch.empty((n, params.num_obs), **f32)
        rew = torch.empty(n, **f32)
        reset = torch.empty(n, dtype=torch.long, device=dev)
        progress_next = torch.empty(n, dtype=torch.long, device=dev)
        q_next, qd_next, actions_next = torch.empty_like(q), torch.empty_like(qd), torch.empty_like(raw)
        planar = isinstance(params, DfxPlanarParams)
        tr = DfxEnvTransition(kind=2 if planar else 1)
        if planar:
            tr.planar = params
        else:
            tr.walker = params
        for name, t in (("progress", progress), ("start_q", start_q), ("start_qd", start_qd), ("obs_before", obs_before), ("rew", rew),
                        ("reset", reset), ("q_next", q_next), ("qd_next", qd_next), ("actions_next", actions_next),
                        ("progress_next", progress_next), ("obs_next", obs_next)):
            setattr(tr, name, t.data_ptr())
        with torch.cuda.device(dev):
            code = lib.dfx_env_step_forward(engine.pack, n, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd), ctypes.byref(m),
                                            _ptr(raw), None, _ptr(used), _ptr(q_sim), _ptr(qd_sim), _ptr(tape), ctypes.byref(tr), _stream(dev))
        _capi.check(code, "dfx_env_step_forward")
        ctx.engine, ctx.cfg, ctx.amap, ctx.params = engine, (substeps, mm_freq, dt), m, params
        ctx.strength = strength                      # keeps the device array the struct points at alive
        ctx.set_materialize_grads(False)             # absent cotangents arrive as None (NULL in the C ABI), not as zero fills
        ctx.shapes = (q.shape, qd.shape)
        # recompute mode: the env-step's input state in place of its tape
        ctx.save_for_backward(raw, tape, q_sim, qd_sim, used, reset, *((q, qd) if ctx.recompute else (None, None)))
        ctx.mark_non_differentiable(reset, progress_next)
        return obs_before, rew, reset, q_next, qd_next, actions_next, progress_next, obs_next

    @staticmethod
    def backward(ctx, g_obs_before, g_rew, g_reset, g_q_next, g_qd_next, g_actions_next, g_progress, g_obs_next):
        raw, tape, q_sim, qd_sim, used, reset, q, qd = ctx.saved_tensors
        engine, (substeps, mm_freq, dt), params = ctx.engine, ctx.cfg, ctx.params
        lib, dev = engine.lib, engine.device
        cot = [None if g is None else _c(g) for g in (g_obs_before, g_rew, g_q_next, g_qd_next, g_actions_next, g_obs_next)]
        planar = isinstance(params, DfxPlanarParams)
        tr = DfxEnvTransitionAdj(kind=2 if planar else 1)
        if planar:
            tr.planar = params
        else:
            tr.walker = params
        # workspace: the cotangents of (q_sim, qd_sim, used) between the transition adjoint and the step adjoint
        gq_sim, gqd_sim, g_used = torch.empty_like(q_sim), torch.empty_like(qd_sim), torch.empty_like(used)
        for name, t in (("q_sim", q_sim), ("qd_sim", qd_sim), ("used", used), ("reset", reset), ("g_obs_before", cot[0]), ("g_rew", cot[1]),
                        ("g_q_next", cot[2]), ("g_qd_next", cot[3]), ("g_actions_next", cot[4]), ("g_obs_next", cot[5]),
                        ("gq_sim", gq_sim), ("gqd_sim", gqd_sim), ("g_used", g_used)):
            setattr(tr, name, _addr(t))
        gq = torch.empty(engine.N * engine.Q, dtype=torch.float32, device=dev)
        gqd = torch.empty(engine.N * engine.D, dtype=torch.float32, device=dev)
        g_raw = torch.empty_like(raw)
        if ctx.recompute:
            workspace = engine.recompute_workspace(substeps, mm_freq)
            with torch.cuda.device(dev):
                code = lib.dfx_env_step_backward_recompute(engine.pack, engine.N, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd),
                                                           ctypes.byref(ctx.amap), _ptr(raw), None, _ptr(workspace), ctypes.byref(tr),
                                                           _ptr(gq), _ptr(gqd), _ptr(g_raw), _stream(dev))
            _capi.check(code, "dfx_env_step_backward_recompute")
        else:
            with torch.cuda.device(dev):
                code = lib.dfx_env_step_backward(engine.pack, engine.N, int(substeps), int(mm_freq), float(dt), ctypes.byref(ctx.amap), _ptr(raw),
                                                 None, _ptr(tape), ctypes.byref(tr), _ptr(gq), _ptr(gqd), _ptr(g_raw), _stream(dev))
            _capi.check(code, "dfx_env_step_backward")
        if ctx.nan_guard:
            for g in (gq, gqd, g_raw):
                torch.nan_to_num(g, nan=0.0, posinf=0.0, neginf=0.0, out=g)
        return None, None, None, None, None, None, None, None, None, None, gq.view(ctx.shapes[0]), gqd.view(ctx.shapes[1]), g_raw
