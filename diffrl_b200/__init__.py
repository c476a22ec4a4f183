import collections


def set_tape_dtype(dtype="fp32"):
    """Storage of the adjoint tape for packs created FROM NOW ON (tile kernels): "fp32" (default) or "bf16" -- link
    velocities, bias accelerations and link wrenches (18 L floats of every row) as bf16, everything that carries
    positions and all arithmetic in fp32 (include/dfx.h dfx_set_tape_dtype; tolerance: tests/tolerances.py)."""
    from . import _capi
    if dtype not in ("fp32", "bf16"):
        raise ValueError("tape dtype must be 'fp32' or 'bf16'")
    _capi.check(_capi.lib().dfx_set_tape_dtype(1 if dtype == "bf16" else 0), "dfx_set_tape_dtype")


def set_adjoint_mode(mode="tape"):
    """How the differentiable step ops (the drop-in ``SemiImplicitIntegrator``, the envs' mapped and single-launch steps) get
    their adjoint, for env-steps run FROM NOW ON:

    - "tape" (default): the forward stores a tape of its intermediates, ``dfx_tape_floats`` per env-step (Ant ~27 KB,
      Humanoid ~182 KB per environment), kept until backward;
    - "recompute": the forward stores no tape and keeps only the env-step's input state, N * (Q + D) floats; the backward
      re-runs each env-step's forward into a one-env-step workspace inside its adjoint launch (include/dfx.h
      dfx_*_backward_recompute).  The recomputed tape is the stored one bit for bit, so gradients do not change; the
      backward costs one more forward per env-step.

    Each op reads the mode when its forward runs, so a graph backpropagates in the mode it was built in and the switch can
    change between rollouts.  Choose "recompute" when the tape of the graph's horizon does not fit in device memory."""
    from . import _capi, engine
    if mode not in engine.ADJOINT_MODES:
        raise ValueError("adjoint mode must be one of %s" % (engine.ADJOINT_MODES,))
    if mode == "recompute" and not hasattr(_capi.lib(), "dfx_step_backward_recompute"):
        raise _capi.DfxError("%s has no recompute adjoint (dfx_step_backward_recompute): rebuild it" % _capi.LIB_PATH)
    engine.adjoint_mode = mode


def link_state(model, joint_q, joint_qd):
    """The pose and velocity of every link of the state (joint_q, joint_qd) of ``model``'s N environments, differentiable:
    ``LinkState(body_X_sc, body_X_sm, body_v_s)`` in the layouts of the reference State fields --

    - ``body_X_sc`` [N, L, 7]: the link frame in world, position then quaternion xyzw;
    - ``body_X_sm`` [N, L, 7]: the centre-of-mass frame X_sc * X_cm (its position is where an external wrench applies its force);
    - ``body_v_s`` [N, L, 6]: the spatial twist (w, v_o) in world axes, v_o the velocity of the body-fixed point at the world
      origin; the centre of mass moves with ``v_o + w x X_sm.p``.

    One kernel launch forward (include/dfx.h dfx_link_state_forward) and one backward, which recomputes the kinematics from
    (joint_q, joint_qd) -- nothing is kept but the inputs, in either adjoint mode.  joint_q [N*Q] or [N, Q], joint_qd [N*D] or
    [N, D], fp32 on the model's device (ValueError otherwise); quaternions are used as given, not renormalised.  Unlike the
    State's derived fields (the start of the last substep of the step that produced a State, no gradient), this is the state
    given, and gradients flow into it."""
    from .dflex_api.sim import _engine_for
    from .engine import LinkStateFunction
    return LinkState(*LinkStateFunction.apply(_engine_for(model), joint_q, joint_qd))


LinkState = collections.namedtuple("LinkState", ["body_X_sc", "body_X_sm", "body_v_s"])


def contact_state(model, joint_q, joint_qd):
    """What the ground does to the links at the state (joint_q, joint_qd) of ``model``'s N environments, differentiable:
    ``ContactState(contact_f, contact_height, body_f_contact)``, fp32, world axes --

    - ``contact_f`` [N, C, 3]: the force the ground exerts on the link at each contact point, in the Model's contact order
      (``contact_body0``); zero for a point that does not penetrate, and for every point when ``model.ground`` is off;
    - ``contact_height`` [N, C]: the point's signed height above the plane, (X_sc p0).y - contact_dist, negative when
      penetrating (computed with the ground on or off);
    - ``body_f_contact`` [N, L, 6]: per link, (torque about its centre of mass, force) summed over its points -- the ``f_ext``
      convention, so it can be passed back as an external wrench.

    This is the step's own penalty contact model at the given state: what the first substep of an env-step from it applies.
    One kernel launch forward (include/dfx.h dfx_contact_state_forward) and one backward, which recomputes the kinematics from
    (joint_q, joint_qd).  The force's gradient flows through penetrating points only, the height's through every point.
    joint_q [N*Q] or [N, Q], joint_qd [N*D] or [N, D], fp32 on the model's device (ValueError otherwise)."""
    from .dflex_api.sim import _engine_for
    from .engine import ContactStateFunction
    return ContactState(*ContactStateFunction.apply(_engine_for(model), joint_q, joint_qd))


ContactState = collections.namedtuple("ContactState", ["contact_f", "contact_height", "body_f_contact"])


def dynamics_state(model, joint_q, joint_qd, joint_act=None, muscle_activation=None, f_ext=None):
    """What the dynamics of the state (joint_q, joint_qd) of ``model``'s N environments produce under the actuation (joint_act,
    muscle_activation) and the external link wrench f_ext, differentiable: ``DynamicsState(joint_qdd, joint_tau, H)``, fp32, in
    the Model's dof order --

    - ``joint_tau`` [N, D]: the generalized joint force, the right-hand side of the solve: -S^T f of each joint's subtree
      (gravity, Coriolis and centrifugal terms, ground contacts, muscles, the external wrench), plus the PD drive to the joint
      target, plus joint_act, plus the joint-limit spring and damper (-f for a free joint).  It is NOT the actuator effort alone;
    - ``H`` [N, D, D]: the joint-space inertia J^T M J, symmetric, without the armature;
    - ``joint_qdd`` [N, D]: the joint accelerations (H + diag(armature))^-1 joint_tau.

    This is what the first substep of an env-step from the state computes before it integrates (H is built from joint_q).  One
    kernel launch forward (include/dfx.h dfx_dynamics_state_forward) and one backward on the tile kernels (two on the lane-group
    kernels), which re-runs a one-substep env-step into a workspace: nothing but the inputs is kept.  Gradients reach joint_q,
    joint_qd, joint_act, muscle_activation and f_ext; only the symmetric part of H's cotangent matters.  joint_act None is zero;
    muscle_activation None is zero (a model with muscles); f_ext [N, L, 6] in the ``DFlexEnv.set_external_wrench`` convention or
    None.  fp32 on the model's device (ValueError otherwise)."""
    import torch
    from .dflex_api.sim import _engine_for
    from .engine import DynamicsStateFunction
    engine = _engine_for(model)
    if joint_act is None:
        joint_act = torch.zeros(engine.N * engine.D, dtype=torch.float32, device=engine.device)
    if muscle_activation is None and engine.M:
        muscle_activation = torch.zeros(engine.N * engine.M, dtype=torch.float32, device=engine.device)
    return DynamicsState(*DynamicsStateFunction.apply(engine, joint_q, joint_qd, joint_act, muscle_activation, f_ext))


DynamicsState = collections.namedtuple("DynamicsState", ["joint_qdd", "joint_tau", "H"])


def jacobian_state(model, joint_q, joint_qd):
    """The link Jacobians and bias accelerations of the state (joint_q, joint_qd) of ``model``'s N environments, differentiable:
    ``JacobianState(J, body_a_s)``, fp32, world axes (semantics in include/dfx.h, dfx_jacobian_state_forward) --

    - ``J`` [N, L, 6, D]: the reference's model.J block per environment.  Column d of link i's 6 rows is the motion subspace
      S_s[d] (spatial (w, v_o), the reference's joint_S_s) when dof d belongs to link i or one of its ancestors, exactly 0
      otherwise; so ``body_v_s = J @ qd`` (``link_state``), and the columns of a free joint are the identity for every link;
    - ``body_a_s`` [N, L, 6]: the reference State's body_a_s, J-dot qd: each link's spatial acceleration with qdd = 0, so the link
      accelerations are ``J @ qdd + body_a_s`` (qdd from ``dynamics_state``).

    Point Jacobians: for a point p fixed to link i (e.g. ``link_state(...).body_X_sm[:, i, :3]``, its centre of mass) with
    (w, v_o) = body_v_s[:, i], dp/dt = (J_v - [p]x J_w) qd, J_w = J[:, i, :3], J_v = J[:, i, 3:]; its bias acceleration is
    body_a_s.v + body_a_s.w x p + w x (v_o + w x p).

    One kernel launch forward (include/dfx.h dfx_jacobian_state_forward) and one backward, which recomputes the kinematics from
    (joint_q, joint_qd).  J depends on joint_q only; body_a_s on both.  joint_q [N*Q] or [N, Q], joint_qd [N*D] or [N, D], fp32 on
    the model's device (ValueError otherwise); quaternions are used as given."""
    from .dflex_api.sim import _engine_for
    from .engine import JacobianStateFunction
    return JacobianState(*JacobianStateFunction.apply(_engine_for(model), joint_q, joint_qd))


JacobianState = collections.namedtuple("JacobianState", ["J", "body_a_s"])
