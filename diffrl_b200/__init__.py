

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
