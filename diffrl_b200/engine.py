"""Host-side engine around the C ABI: one pack per (model, device), one forward and one backward
kernel launch per env-step, exposed to PyTorch as a single ``autograd.Function``.

Replaces the reference's ``SimulateFunc`` + ``Tape`` (``dflex/dflex/sim.py:2086-2154``,
``dflex/dflex/adjoint.py:2114-2216``): instead of recording 10-11 launches per substep and keeping
every State tensor of every substep alive, forward writes one tape ROW per substep -- the (q, qd) entering it plus
the forward intermediates the adjoint needs (X_sc, X_sm, S, v, a, total link wrenches, q'') -- and one H^-1 block
per mass-matrix update; backward is one kernel that streams those rows back (TMA bulk copies in the tile
kernels) and does NOT re-run the forward dynamics.  The tape is an opaque fp32 tensor sized by
``dfx_tape_floats`` (optionally with bf16 (v, a, f_tot): ``diffrl_b200.set_tape_dtype``).  In recompute mode
(``diffrl_b200.set_adjoint_mode("recompute")``) the forward keeps no tape: the backward re-runs the env-step's forward
into a one-env-step workspace inside its adjoint launch.
"""
import ctypes

import torch

from . import _capi
from .modelpack import DfxDerived, DfxExternalWrench, articulation_from_model

_DERIVED_SHAPES = {
    "body_X_sc": ("L", 7), "body_X_sm": ("L", 7), "joint_S_s": ("D", 6), "body_v_s": ("L", 6),
    "body_a_s": ("L", 6), "body_f_s": ("L", 6), "body_ft_s": ("L", 6), "joint_tau": ("D", 0),
    "joint_qdd": ("D", 0), "H": ("DD", 0), "L": ("DD", 0),
}


ADJOINT_MODES = ("tape", "recompute")
adjoint_mode = "tape"        # diffrl_b200.set_adjoint_mode; the step ops read it in forward and keep it on ctx


def recompute_adjoint():
    return adjoint_mode == "recompute"


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _f32c(t, device):
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


def check_wrench(engine, f_ext):
    """``f_ext``: per-environment external link wrenches, [N, L, 6] or [N*L, 6] fp32 on the engine's device -- row (e, i) is
    (torque, force), both in world axes, the force applied at link i's centre of mass (include/dfx.h DfxExternalWrench).
    Returns it detached and contiguous (None stays None); anything else is a ValueError."""
    if f_ext is None:
        return None
    if not isinstance(f_ext, torch.Tensor):
        raise ValueError("f_ext must be a torch.Tensor, got %s" % type(f_ext).__name__)
    if f_ext.dtype != torch.float32:
        raise ValueError("f_ext must be float32, got %s" % f_ext.dtype)
    if f_ext.device != engine.device:
        raise ValueError("f_ext is on %s, the engine on %s" % (f_ext.device, engine.device))
    if tuple(f_ext.shape) not in ((engine.N, engine.L, 6), (engine.N * engine.L, 6)):
        raise ValueError("f_ext has shape %s, expected [%d, %d, 6] or [%d, 6]" % (tuple(f_ext.shape), engine.N, engine.L,
                                                                                  engine.N * engine.L))
    engine.check_wrench_fits()
    return f_ext.detach().contiguous()


def check_link_input(engine, name, t, shapes):
    """``t``: an input of the link state -- fp32 on the engine's device, of one of ``shapes`` (the state: [N*Q] or [N, Q],
    [N*D] or [N, D]; the cotangents: the outputs' shapes).  Returns it detached and contiguous (None stays None); anything else
    is a ValueError, in the style of ``check_wrench``."""
    if t is None:
        return None
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    if t.dtype != torch.float32:
        raise ValueError("%s must be float32, got %s" % (name, t.dtype))
    if t.device != engine.device:
        raise ValueError("%s is on %s, the engine on %s" % (name, t.device, engine.device))
    if tuple(t.shape) not in shapes:
        raise ValueError("%s has shape %s, expected %s" % (name, tuple(t.shape), " or ".join(str(list(s)) for s in shapes)))
    return t.detach().contiguous()


LINK_STATE_FIELDS = ("body_X_sc", "body_X_sm", "body_v_s")
CONTACT_STATE_FIELDS = ("contact_f", "contact_height", "body_f_contact")
DYNAMICS_STATE_FIELDS = ("joint_qdd", "joint_tau", "H")
JACOBIAN_STATE_FIELDS = ("J", "body_a_s")


def wrench_struct(f_ext, g_f_ext=None):
    """The DfxExternalWrench of an _ex entry (by reference), or None: no wrench."""
    if f_ext is None:
        return None
    return ctypes.byref(DfxExternalWrench(f_ext.data_ptr(), None if g_f_ext is None else g_f_ext.data_ptr()))


_GRAVEYARD = []


def _bury():
    """Free the packs of dead engines unless a capture is in progress."""
    try:
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            return
    except Exception:
        return
    while _GRAVEYARD:
        lib, pack = _GRAVEYARD.pop()
        lib.dfx_pack_destroy(pack)


class ArticulationEngine:
    """Device-resident description of one articulation + launchers for N environments."""

    def __init__(self, desc, num_envs, device):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _capi.DfxError("diffrl_b200 runs the simulation step on CUDA devices only (got %s); "
                                 "there is no CPU fallback" % self.device)
        self.lib = _capi.lib()
        self.desc, self.N = desc, int(num_envs)
        index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", index)
        err = ctypes.create_string_buffer(512)
        struct = desc.as_struct()
        _bury()
        self.pack = self.lib.dfx_pack_create(ctypes.byref(struct), index, err, 512)
        if not self.pack:
            raise _capi.DfxError("dfx_pack_create: " + err.value.decode())
        self.L, self.D, self.Q, self.C, self.M = desc.L, desc.D, desc.Q, desc.C, desc.M
        self.tape_bf16 = bool(self.lib.dfx_pack_query(self.pack, 10))
        self._gravity = (desc.gravity, desc.ground)
        self._wrench_fits = False
        self._check_fits()

    def _check_fits(self, wrench=False):
        """The step kernels keep one environment's scratch in shared memory: refuse an articulation whose scratch does not
        fit one CTA (227 KB), instead of failing its first launch with a bare cudaErrorInvalidConfiguration.  ``wrench``: the
        external-wrench kernels, whose scratch holds the wrench and its cotangent as well."""
        if not hasattr(self.lib, "dfx_launch_plan"):      # (older builds loaded through DFX_LIBRARY for A/B timing)
            return
        plan = (ctypes.c_int * 6)()
        for backward, what in ((0, "forward"), (1, "backward")):
            _capi.check(self.lib.dfx_launch_plan(self.pack, backward | (2 if wrench else 0), plan), "dfx_launch_plan")
            if plan[1] == 0:
                floats = self.lib.dfx_pack_query(self.pack, 5 + backward)
                extra = ""
                if wrench:
                    floats = int(plan[4])
                    extra = " with the external wrench and its cotangent staged"
                need = (floats * 4 + plan[5]) / 1024.0
                raise _capi.DfxError(
                    "articulation too large for the step kernels%s: the %s pass of one environment needs %.1f KB of shared "
                    "memory (%d floats of scratch for L=%d links, D=%d dofs, C=%d contacts, plus the model), more than the "
                    "227 KB of one CTA" % (extra, what, need, floats, self.L, self.D, self.C))

    def check_wrench_fits(self):
        """Raise DfxError when the external-wrench kernels of this articulation do not fit one CTA (checked once)."""
        if not self._wrench_fits:
            if not hasattr(self.lib, "dfx_step_forward_ex"):
                raise _capi.DfxError("%s has no external-wrench entries (dfx_*_ex)" % _capi.LIB_PATH)
            self._check_fits(wrench=True)
            self._wrench_fits = True

    @classmethod
    def from_model(cls, model, device, num_envs=None):
        desc, n = articulation_from_model(model, num_envs)
        return cls(desc, n, device)

    def __del__(self):
        # dfx_pack_destroy() is a cudaFree (device-synchronising): it must not run while a CUDA graph is being captured,
        # and the garbage collector can fire at any time -- packs released during a capture wait for the next engine
        try:
            if getattr(self, "pack", None):
                _GRAVEYARD.append((self.lib, self.pack))
                self.pack = None
                _bury()
        except Exception:
            pass

    def set_gravity(self, gravity, ground):
        key = (tuple(float(g) for g in gravity), bool(ground))
        if key != self._gravity:
            _capi.check(self.lib.dfx_pack_set_gravity(self.pack, key[0][0], key[0][1], key[0][2], int(key[1])),
                        "dfx_pack_set_gravity")
            self._gravity = key

    def tape_rows(self, tape, substeps):
        """The [substeps, num_envs, row] view of the tape's per-substep rows as a NEW tensor, whatever the kernel
        family's layout (debugging / tests; the tape is otherwise opaque to callers)."""
        row = int(self.lib.dfx_pack_query(self.pack, 8))
        tile = int(self.lib.dfx_pack_query(self.pack, 9))
        if not tile:
            return tape[: substeps * self.N * row].view(substeps, self.N, row).clone()
        ntiles = (self.N + tile - 1) // tile
        units = int(self.lib.dfx_pack_query(self.pack, 11))       # 4-byte units per row in the tape (< row with a bf16 tape)
        t = tape[: substeps * ntiles * units * tile].view(substeps, ntiles, units, tile)
        if units != row:
            # bf16 tape: [q, qd, X_sc, X_sm, S | (v, a, f_tot) as bf16 pairs | q'', padding]
            mid = 18 * self.L
            head = self.Q + self.D + 14 * self.L + 6 * self.D
            lo = t[:, :, :head]
            halves = t[:, :, head:head + mid // 2].contiguous().view(torch.bfloat16).view(substeps, ntiles, mid, tile).float()
            t = torch.cat([lo, halves, t[:, :, head + mid // 2:]], dim=2)
        return t.permute(0, 1, 3, 2).reshape(substeps, ntiles * tile, row)[:, : self.N].contiguous()

    def tape_hinv(self, tape, substeps, mm_freq):
        """The H^-1 blocks of the tape (every mass-matrix update, every environment slot of the kernel family's layout) as a
        NEW flat tensor (tests)."""
        tile = int(self.lib.dfx_pack_query(self.pack, 9))
        slots = (self.N + tile - 1) // tile * tile if tile else self.N
        end = self.tape_floats(substeps, mm_freq)
        nseg = (substeps + mm_freq - 1) // mm_freq
        return tape[end - nseg * slots * self.D * self.D:end].clone()

    def tape_floats(self, substeps, mm_freq):
        return int(self.lib.dfx_tape_floats(self.pack, self.N, substeps, mm_freq))

    def recompute_workspace(self, substeps, mm_freq):
        """An uninitialised workspace for one recompute adjoint: one env-step's tape + its end state (include/dfx.h)."""
        n = int(self.lib.dfx_recompute_workspace_floats(self.pack, self.N, int(substeps), int(mm_freq)))
        return torch.empty(n, dtype=torch.float32, device=self.device)

    def workspace_end_state(self, workspace, substeps, mm_freq):
        """(q_out, qd_out) of the forward a recompute adjoint re-ran into ``workspace`` (views)."""
        t, nq = self.tape_floats(substeps, mm_freq), self.N * self.Q
        return workspace[t:t + nq], workspace[t + nq:t + nq + self.N * self.D]

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def forward(self, q, qd, act, musc, substeps, mm_freq, dt, want_tape=True, derived=None, out=None, f_ext=None):
        """Returns (q_out, qd_out, tape or None).  ``derived``: optional dict name -> bool of dumps to
        fill (returned as a dict of tensors under key 'derived' attribute of the result tuple).  ``f_ext``: external link
        wrenches [N, L, 6] (``check_wrench``), held over the substeps; the backward must be given the same."""
        dev = self.device
        f_ext = check_wrench(self, f_ext)
        q, qd, act = _f32c(q, dev), _f32c(qd, dev), _f32c(act, dev)
        if q.numel() != self.N * self.Q or qd.numel() != self.N * self.D or act.numel() != self.N * self.D:
            raise ValueError("state tensors do not match num_envs=%d, Q=%d, D=%d" % (self.N, self.Q, self.D))
        if self.M:
            if musc is None:
                raise ValueError("this model has muscles: muscle_activation is required")
            musc = _f32c(musc, dev)
            if musc.numel() != self.N * self.M:
                raise ValueError("muscle_activation has %d entries, expected %d" % (musc.numel(), self.N * self.M))
        else:
            musc = None
        if out is None:
            q_out, qd_out = torch.empty_like(q), torch.empty_like(qd)
        else:
            q_out, qd_out = out
        tape = torch.empty(self.tape_floats(substeps, mm_freq), dtype=torch.float32, device=dev) if want_tape else None
        dv, dumps = None, None
        if derived:
            dv, dumps = DfxDerived(), {}
            dims = {"L": self.L, "D": self.D, "DD": self.D * self.D}
            for name in derived:
                a, b = _DERIVED_SHAPES[name]
                shape = (self.N * dims[a], b) if b else (self.N * dims[a],)
                dumps[name] = torch.zeros(shape, dtype=torch.float32, device=dev)
                setattr(dv, name, dumps[name].data_ptr())
        args = (self.pack, self.N, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(q_out),
                _ptr(qd_out), _ptr(tape), None if dv is None else ctypes.byref(dv), self._stream())
        with torch.cuda.device(dev):
            if f_ext is None:
                code = self.lib.dfx_step_forward(*args)
            else:
                code = self.lib.dfx_step_forward_ex(*args, wrench_struct(f_ext))
        _capi.check(code, "dfx_step_forward")
        return q_out, qd_out, tape, dumps

    def _wrench_grad(self, f_ext, need):
        return torch.empty(f_ext.shape, dtype=torch.float32, device=self.device) if (f_ext is not None and need) else None

    def backward(self, act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt, need=(True, True, True, True), f_ext=None,
                 need_f_ext=True):
        """Cotangents (gq, gqd, gact, gmusc) of the inputs; with ``f_ext`` (the forward's) a fifth, g_f_ext (None unless
        ``need_f_ext``), shaped as ``f_ext``."""
        dev = self.device
        f_ext = check_wrench(self, f_ext)
        g_f_ext = self._wrench_grad(f_ext, need_f_ext)
        act = _f32c(act, dev)
        musc = _f32c(musc, dev) if self.M else None
        gq_out = None if gq_out is None else _f32c(gq_out, dev)
        gqd_out = None if gqd_out is None else _f32c(gqd_out, dev)
        gq = torch.empty(self.N * self.Q, dtype=torch.float32, device=dev) if need[0] else None
        gqd = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[1] else None
        gact = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[2] else None
        gmusc = torch.empty(self.N * self.M, dtype=torch.float32, device=dev) if (need[3] and self.M) else None
        args = (self.pack, self.N, int(substeps), int(mm_freq), float(dt), _ptr(act), _ptr(musc), _ptr(tape), _ptr(gq_out),
                _ptr(gqd_out), _ptr(gq), _ptr(gqd), _ptr(gact), _ptr(gmusc), self._stream())
        with torch.cuda.device(dev):
            if f_ext is None:
                code = self.lib.dfx_step_backward(*args)
            else:
                code = self.lib.dfx_step_backward_ex(*args, wrench_struct(f_ext, g_f_ext))
        _capi.check(code, "dfx_step_backward")
        if f_ext is None:
            return gq, gqd, gact, gmusc
        return gq, gqd, gact, gmusc, g_f_ext

    def backward_recompute(self, q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt, need=(True, True, True, True),
                           workspace=None, f_ext=None, need_f_ext=True):
        """``backward`` without a tape: the env-step's forward from (q, qd, act, musc[, f_ext]) is re-run into a workspace inside
        the adjoint launch (``dfx_step_backward_recompute``).  ``workspace`` (``recompute_workspace()``): used and left readable
        (``tape_rows``, ``tape_hinv``, ``workspace_end_state``); None: one from the caching allocator."""
        dev = self.device
        f_ext = check_wrench(self, f_ext)
        g_f_ext = self._wrench_grad(f_ext, need_f_ext)
        q, qd, act = _f32c(q, dev), _f32c(qd, dev), _f32c(act, dev)
        musc = _f32c(musc, dev) if self.M else None
        gq_out = None if gq_out is None else _f32c(gq_out, dev)
        gqd_out = None if gqd_out is None else _f32c(gqd_out, dev)
        if workspace is None:
            workspace = self.recompute_workspace(substeps, mm_freq)
        gq = torch.empty(self.N * self.Q, dtype=torch.float32, device=dev) if need[0] else None
        gqd = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[1] else None
        gact = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[2] else None
        gmusc = torch.empty(self.N * self.M, dtype=torch.float32, device=dev) if (need[3] and self.M) else None
        args = (self.pack, self.N, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(workspace),
                _ptr(gq_out), _ptr(gqd_out), _ptr(gq), _ptr(gqd), _ptr(gact), _ptr(gmusc), self._stream())
        with torch.cuda.device(dev):
            if f_ext is None:
                code = self.lib.dfx_step_backward_recompute(*args)
            else:
                code = self.lib.dfx_step_backward_recompute_ex(*args, wrench_struct(f_ext, g_f_ext))
        _capi.check(code, "dfx_step_backward_recompute")
        if f_ext is None:
            return gq, gqd, gact, gmusc
        return gq, gqd, gact, gmusc, g_f_ext

    def _link_state_inputs(self, q, qd):
        if not hasattr(self.lib, "dfx_link_state_forward"):
            raise _capi.DfxError("%s has no link-state entries (dfx_link_state_*)" % _capi.LIB_PATH)
        q = check_link_input(self, "q", q, ((self.N * self.Q,), (self.N, self.Q)))
        qd = check_link_input(self, "qd", qd, ((self.N * self.D,), (self.N, self.D)))
        return q, qd

    def link_state(self, q, qd, want=LINK_STATE_FIELDS):
        """(body_X_sc [N, L, 7], body_X_sm [N, L, 7], body_v_s [N, L, 6]) of the state (q, qd) -- ``dfx_link_state_forward``: link
        frame and centre-of-mass frame in world (position, quaternion xyzw), spatial twist (w, v_o) in world axes; the centre of
        mass moves with v_o + w x X_sm.p.  The fields not in ``want`` are None (not computed).  q [N*Q] or [N, Q], qd [N*D] or
        [N, D], fp32 on the engine's device (ValueError otherwise); quaternions are used as given."""
        q, qd = self._link_state_inputs(q, qd)
        dev, N, L = self.device, self.N, self.L
        out = tuple(torch.empty((N, L, 7 if name != "body_v_s" else 6), dtype=torch.float32, device=dev) if name in want else None
                    for name in LINK_STATE_FIELDS)
        with torch.cuda.device(dev):
            code = self.lib.dfx_link_state_forward(self.pack, N, _ptr(q), _ptr(qd), *(_ptr(o) for o in out), self._stream())
        _capi.check(code, "dfx_link_state_forward")
        return out

    def link_state_backward(self, q, qd, g_X_sc, g_X_sm, g_v_s, need=(True, True)):
        """Cotangents (gq [N*Q], gqd [N*D]) of the state from those of (body_X_sc, body_X_sm, body_v_s) (None: zero) --
        ``dfx_link_state_backward``, which recomputes the kinematics of (q, qd).  An output not in ``need`` is None."""
        q, qd = self._link_state_inputs(q, qd)
        N, L = self.N, self.L
        g = [check_link_input(self, "g_" + name, t, ((N, L, w), (N * L, w), (N * L * w,)))
             for name, t, w in zip(LINK_STATE_FIELDS, (g_X_sc, g_X_sm, g_v_s), (7, 7, 6))]
        gq = torch.empty(N * self.Q, dtype=torch.float32, device=self.device) if need[0] else None
        gqd = torch.empty(N * self.D, dtype=torch.float32, device=self.device) if need[1] else None
        with torch.cuda.device(self.device):
            code = self.lib.dfx_link_state_backward(self.pack, N, _ptr(q), _ptr(qd), *(_ptr(x) for x in g), _ptr(gq), _ptr(gqd),
                                                    self._stream())
        _capi.check(code, "dfx_link_state_backward")
        return gq, gqd

    def _contact_state_inputs(self, q, qd):
        if not hasattr(self.lib, "dfx_contact_state_forward"):
            raise _capi.DfxError("%s has no contact-state entries (dfx_contact_state_*)" % _capi.LIB_PATH)
        q = check_link_input(self, "q", q, ((self.N * self.Q,), (self.N, self.Q)))
        qd = check_link_input(self, "qd", qd, ((self.N * self.D,), (self.N, self.D)))
        return q, qd

    def _contact_shapes(self):
        N, C, L = self.N, self.C, self.L
        return {"contact_f": ((N, C, 3), (N * C, 3), (N * C * 3,)), "contact_height": ((N, C), (N * C,)),
                "body_f_contact": ((N, L, 6), (N * L, 6), (N * L * 6,))}

    def contact_state(self, q, qd, want=CONTACT_STATE_FIELDS):
        """(contact_f [N, C, 3], contact_height [N, C], body_f_contact [N, L, 6]) of the state (q, qd) -- ``dfx_contact_state_forward``:
        the force the ground exerts on the link at each contact point (Model contact order; zero when the point does not
        penetrate or the ground is off), the point's signed height above the plane (negative: penetrating), and per link the
        wrench (torque about the centre of mass, force) of its points in world axes -- the ``f_ext`` convention.  The fields not in
        ``want`` are None (not computed).  q [N*Q] or [N, Q], qd [N*D] or [N, D], fp32 on the engine's device (ValueError
        otherwise)."""
        q, qd = self._contact_state_inputs(q, qd)
        shapes = self._contact_shapes()
        out = tuple(torch.empty(shapes[name][0], dtype=torch.float32, device=self.device) if name in want else None
                    for name in CONTACT_STATE_FIELDS)
        with torch.cuda.device(self.device):
            code = self.lib.dfx_contact_state_forward(self.pack, self.N, _ptr(q), _ptr(qd), *(_ptr(o) for o in out), self._stream())
        _capi.check(code, "dfx_contact_state_forward")
        return out

    def contact_state_backward(self, q, qd, g_contact_f, g_contact_height, g_body_f_contact, need=(True, True)):
        """Cotangents (gq [N*Q], gqd [N*D]) of the state from those of (contact_f, contact_height, body_f_contact) (None: zero) --
        ``dfx_contact_state_backward``, which recomputes the kinematics of (q, qd).  An output not in ``need`` is None."""
        q, qd = self._contact_state_inputs(q, qd)
        shapes = self._contact_shapes()
        g = [check_link_input(self, "g_" + name, t, shapes[name])
             for name, t in zip(CONTACT_STATE_FIELDS, (g_contact_f, g_contact_height, g_body_f_contact))]
        gq = torch.empty(self.N * self.Q, dtype=torch.float32, device=self.device) if need[0] else None
        gqd = torch.empty(self.N * self.D, dtype=torch.float32, device=self.device) if need[1] else None
        with torch.cuda.device(self.device):
            code = self.lib.dfx_contact_state_backward(self.pack, self.N, _ptr(q), _ptr(qd), *(_ptr(x) for x in g), _ptr(gq), _ptr(gqd),
                                                       self._stream())
        _capi.check(code, "dfx_contact_state_backward")
        return gq, gqd

    def _jacobian_state_inputs(self, q, qd):
        if not hasattr(self.lib, "dfx_jacobian_state_forward"):
            raise _capi.DfxError("%s has no Jacobian-state entries (dfx_jacobian_state_*)" % _capi.LIB_PATH)
        q = check_link_input(self, "q", q, ((self.N * self.Q,), (self.N, self.Q)))
        qd = check_link_input(self, "qd", qd, ((self.N * self.D,), (self.N, self.D)))
        return q, qd

    def jacobian_state(self, q, qd, want=JACOBIAN_STATE_FIELDS):
        """(J [N, L, 6, D], body_a_s [N, L, 6]) of the state (q, qd) -- ``dfx_jacobian_state_forward`` (semantics in include/dfx.h):
        the link Jacobians, column d of link i's block the motion subspace S_s[d] (spatial (w, v_o), world axes) when dof d moves
        link i and exactly 0 otherwise, so body_v_s = J @ qd; and the bias accelerations J-dot qd, so the link accelerations are
        J @ qdd + body_a_s.  The fields not in ``want`` are None (not computed).  q [N*Q] or [N, Q], qd [N*D] or [N, D], fp32 on the
        engine's device (ValueError otherwise); quaternions are used as given."""
        q, qd = self._jacobian_state_inputs(q, qd)
        N, L, D = self.N, self.L, self.D
        out = (torch.empty((N, L, 6, D), dtype=torch.float32, device=self.device) if "J" in want else None,
               torch.empty((N, L, 6), dtype=torch.float32, device=self.device) if "body_a_s" in want else None)
        with torch.cuda.device(self.device):
            code = self.lib.dfx_jacobian_state_forward(self.pack, N, _ptr(q), _ptr(qd), *(_ptr(o) for o in out), self._stream())
        _capi.check(code, "dfx_jacobian_state_forward")
        return out

    def jacobian_state_backward(self, q, qd, g_J, g_a_s, need=(True, True)):
        """Cotangents (gq [N*Q], gqd [N*D]) of the state from those of (J, body_a_s) (None: zero; g_J as [N, L, 6, D], [N, 6L, D]
        or flat) -- ``dfx_jacobian_state_backward``, which recomputes the kinematics of (q, qd).  J depends on q only.  An output
        not in ``need`` is None."""
        q, qd = self._jacobian_state_inputs(q, qd)
        N, L, D = self.N, self.L, self.D
        g_J = check_link_input(self, "g_J", g_J, ((N, L, 6, D), (N, 6 * L, D), (N * L * 6 * D,)))
        g_a_s = check_link_input(self, "g_body_a_s", g_a_s, ((N, L, 6), (N * L, 6), (N * L * 6,)))
        gq = torch.empty(N * self.Q, dtype=torch.float32, device=self.device) if need[0] else None
        gqd = torch.empty(N * self.D, dtype=torch.float32, device=self.device) if need[1] else None
        with torch.cuda.device(self.device):
            code = self.lib.dfx_jacobian_state_backward(self.pack, N, _ptr(q), _ptr(qd), _ptr(g_J), _ptr(g_a_s), _ptr(gq), _ptr(gqd),
                                                        self._stream())
        _capi.check(code, "dfx_jacobian_state_backward")
        return gq, gqd

    def _dynamics_state_inputs(self, q, qd, act, musc, f_ext):
        if not hasattr(self.lib, "dfx_dynamics_state_forward"):
            raise _capi.DfxError("%s has no dynamics-state entries (dfx_dynamics_state_*)" % _capi.LIB_PATH)
        N, Q, D, M, L = self.N, self.Q, self.D, self.M, self.L
        q = check_link_input(self, "q", q, ((N * Q,), (N, Q)))
        qd = check_link_input(self, "qd", qd, ((N * D,), (N, D)))
        act = check_link_input(self, "act", act, ((N * D,), (N, D)))
        if act is None:
            raise ValueError("act is required (zeros for no actuation)")
        if M:
            musc = check_link_input(self, "musc", musc, ((N * M,), (N, M)))
            if musc is None:
                raise ValueError("this model has muscles: musc is required")
        else:
            musc = None
        f_ext = check_link_input(self, "f_ext", f_ext, ((N, L, 6), (N * L, 6), (N * L * 6,)))
        return q, qd, act, musc, f_ext

    def _dynamics_shapes(self):
        N, D = self.N, self.D
        return {"joint_qdd": ((N, D), (N * D,)), "joint_tau": ((N, D), (N * D,)), "H": ((N, D, D), (N * D, D), (N * D * D,))}

    def dynamics_workspace(self):
        """An uninitialised workspace for ``dynamics_state_backward``: one one-substep env-step's tape + its end state."""
        n = int(self.lib.dfx_dynamics_workspace_floats(self.pack, self.N))
        return torch.empty(n, dtype=torch.float32, device=self.device)

    def dynamics_state(self, q, qd, act, musc=None, f_ext=None, want=DYNAMICS_STATE_FIELDS):
        """(joint_qdd [N, D], joint_tau [N, D], H [N, D, D]) of the state (q, qd) under the actuation (act, musc) and the external
        wrench f_ext (None: none) -- ``dfx_dynamics_state_forward``: what the first substep of an env-step from it computes before it
        integrates.  joint_tau is the right-hand side of the solve (bias, contact, muscle and external forces, PD drive, act, limits),
        not the actuator effort alone; H = J^T M J without the armature; joint_qdd = (H + diag(armature))^-1 joint_tau.  The fields
        not in ``want`` are None (not computed).  q [N*Q] or [N, Q], qd and act [N*D] or [N, D], musc [N*M] or [N, M] (required
        with muscles), f_ext [N, L, 6]; fp32 on the engine's device (ValueError otherwise)."""
        return self._dynamics_state_checked(*self._dynamics_state_inputs(q, qd, act, musc, f_ext), want=want)

    def _dynamics_state_checked(self, q, qd, act, musc, f_ext, want=DYNAMICS_STATE_FIELDS):
        """``dynamics_state`` on inputs ``_dynamics_state_inputs`` has already checked and converted"""
        shapes = self._dynamics_shapes()
        out = tuple(torch.empty(shapes[name][0], dtype=torch.float32, device=self.device) if name in want else None
                    for name in DYNAMICS_STATE_FIELDS)
        with torch.cuda.device(self.device):
            code = self.lib.dfx_dynamics_state_forward(self.pack, self.N, _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(f_ext),
                                                       *(_ptr(o) for o in out), self._stream())
        _capi.check(code, "dfx_dynamics_state_forward")
        return out

    def dynamics_state_backward(self, q, qd, act, musc, f_ext, g_qdd, g_tau, g_H, need=(True, True, True, True, True), workspace=None):
        """Cotangents (gq [N*Q], gqd [N*D], gact [N*D], gmusc [N*M], g_f_ext [N, L, 6]) of the inputs from those of (joint_qdd,
        joint_tau, H) (None: zero; g_H need not be symmetric) -- ``dfx_dynamics_state_backward``, which re-runs a one-substep
        env-step into ``workspace`` (``dynamics_workspace()``; None: one from the caching allocator).  An output not in ``need``,
        gmusc without muscles and g_f_ext without a wrench are None."""
        q, qd, act, musc, f_ext = self._dynamics_state_inputs(q, qd, act, musc, f_ext)
        shapes = self._dynamics_shapes()
        g = [check_link_input(self, "g_" + name, t, shapes[name]) for name, t in zip(DYNAMICS_STATE_FIELDS, (g_qdd, g_tau, g_H))]
        if workspace is None:
            workspace = self.dynamics_workspace()
        dev, N = self.device, self.N
        gq = torch.empty(N * self.Q, dtype=torch.float32, device=dev) if need[0] else None
        gqd = torch.empty(N * self.D, dtype=torch.float32, device=dev) if need[1] else None
        gact = torch.empty(N * self.D, dtype=torch.float32, device=dev) if need[2] else None
        gmusc = torch.empty(N * self.M, dtype=torch.float32, device=dev) if (need[3] and self.M) else None
        g_f_ext = torch.empty((N, self.L, 6), dtype=torch.float32, device=dev) if (need[4] and f_ext is not None) else None
        with torch.cuda.device(dev):
            code = self.lib.dfx_dynamics_state_backward(self.pack, N, _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(f_ext),
                                                        _ptr(workspace), *(_ptr(x) for x in g), _ptr(gq), _ptr(gqd), _ptr(gact),
                                                        _ptr(gmusc), _ptr(g_f_ext), self._stream())
        _capi.check(code, "dfx_dynamics_state_backward")
        return gq, gqd, gact, gmusc, g_f_ext


class MappedSimStepFunction(torch.autograd.Function):
    """(q, qd, raw policy output) -> (q', qd', used): the env-step with the action map folded into the simulation launch
    (``dfx_step_forward_mapped`` / ``dfx_step_backward_mapped``): ``used = clip(raw, -1, 1) * pre_scale + pre_bias`` (the env's
    ``actions``), ``joint_act`` / the muscle activations are formed inside the kernel.  ``amap`` = (offset, pre_scale, pre_bias,
    drive_scale, strength [A], is_muscle).  ``f_ext``: optional external link wrenches [N, L, 6] (``check_wrench``); its
    gradient is returned when it requires one."""

    @staticmethod
    def forward(ctx, engine, substeps, mm_freq, dt, amap, q, qd, raw, f_ext=None):
        from .modelpack import DfxActionMap
        offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = amap
        dev = engine.device
        q, qd = _f32c(q.detach(), dev), _f32c(qd.detach(), dev)
        raw = _f32c(raw.detach(), dev)
        f_ext = check_wrench(engine, f_ext)
        n, A = engine.N, raw.shape[-1]
        m = DfxActionMap(int(A), int(offset), int(bool(is_muscle)), float(pre_scale), float(pre_bias), float(drive_scale), strength.data_ptr())
        need = any(ctx.needs_input_grad[5:9])
        ctx.recompute = recompute_adjoint()
        q_out, qd_out, used = torch.empty_like(q), torch.empty_like(qd), torch.empty_like(raw)
        tape = torch.empty(engine.tape_floats(substeps, mm_freq), dtype=torch.float32, device=dev) if (need and not ctx.recompute) else None
        args = (engine.pack, n, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd), ctypes.byref(m), _ptr(raw), None, _ptr(used),
                _ptr(q_out), _ptr(qd_out), _ptr(tape), engine._stream())
        with torch.cuda.device(dev):
            if f_ext is None:
                code = engine.lib.dfx_step_forward_mapped(*args)
            else:
                code = engine.lib.dfx_step_forward_mapped_ex(*args, wrench_struct(f_ext))
        _capi.check(code, "dfx_step_forward_mapped")
        ctx.engine, ctx.cfg, ctx.amap = engine, (substeps, mm_freq, dt), m
        ctx.strength = strength                      # keeps the device array the struct points at alive
        ctx.set_materialize_grads(False)
        ctx.shapes = (q.shape, qd.shape)
        if ctx.recompute:
            ctx.save_for_backward(raw, f_ext, q, qd)        # the env-step's input state, in place of its tape
        else:
            ctx.save_for_backward(raw, f_ext, tape)
        return q_out, qd_out, used

    @staticmethod
    def backward(ctx, gq_out, gqd_out, g_used):
        engine, (substeps, mm_freq, dt) = ctx.engine, ctx.cfg
        dev = engine.device
        gq_out = None if gq_out is None else _f32c(gq_out, dev)
        gqd_out = None if gqd_out is None else _f32c(gqd_out, dev)
        g_used = None if g_used is None else _f32c(g_used, dev)
        gq = torch.empty(engine.N * engine.Q, dtype=torch.float32, device=dev)
        gqd = torch.empty(engine.N * engine.D, dtype=torch.float32, device=dev)
        cot = (_ptr(gq_out), _ptr(gqd_out), _ptr(g_used), _ptr(gq), _ptr(gqd))
        if ctx.recompute:
            raw, f_ext, q, qd = ctx.saved_tensors
            g_raw = torch.empty_like(raw)
            g_f_ext = engine._wrench_grad(f_ext, ctx.needs_input_grad[8] if f_ext is not None else False)
            workspace = engine.recompute_workspace(substeps, mm_freq)
            args = (engine.pack, engine.N, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd), ctypes.byref(ctx.amap), _ptr(raw), None,
                    _ptr(workspace), *cot, _ptr(g_raw), engine._stream())
            with torch.cuda.device(dev):
                if f_ext is None:
                    code = engine.lib.dfx_step_backward_mapped_recompute(*args)
                else:
                    code = engine.lib.dfx_step_backward_mapped_recompute_ex(*args, wrench_struct(f_ext, g_f_ext))
            _capi.check(code, "dfx_step_backward_mapped_recompute")
        else:
            raw, f_ext, tape = ctx.saved_tensors
            g_raw = torch.empty_like(raw)
            g_f_ext = engine._wrench_grad(f_ext, ctx.needs_input_grad[8] if f_ext is not None else False)
            args = (engine.pack, engine.N, int(substeps), int(mm_freq), float(dt), ctypes.byref(ctx.amap), _ptr(raw), None, _ptr(tape), *cot,
                    _ptr(g_raw), engine._stream())
            with torch.cuda.device(dev):
                if f_ext is None:
                    code = engine.lib.dfx_step_backward_mapped(*args)
                else:
                    code = engine.lib.dfx_step_backward_mapped_ex(*args, wrench_struct(f_ext, g_f_ext))
            _capi.check(code, "dfx_step_backward_mapped")
        return None, None, None, None, None, gq.view(ctx.shapes[0]), gqd.view(ctx.shapes[1]), g_raw, g_f_ext


class LinkStateFunction(torch.autograd.Function):
    """(q, qd) -> (body_X_sc [N, L, 7], body_X_sm [N, L, 7], body_v_s [N, L, 6]): the pose and velocity of every link
    (``ArticulationEngine.link_state``; the centre of mass moves with v_o + w x X_sm.p).  Saves only (q, qd): the backward
    recomputes the kinematics, so it is the same in "tape" and "recompute" adjoint mode."""

    @staticmethod
    def forward(ctx, engine, q, qd):
        qc, qdc = engine._link_state_inputs(q, qd)
        out = engine.link_state(qc, qdc)
        ctx.engine, ctx.shapes = engine, (q.shape, qd.shape)
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_link_state_backward, not a zero fill
        ctx.save_for_backward(qc, qdc)
        return out

    @staticmethod
    def backward(ctx, g_X_sc, g_X_sm, g_v_s):
        q, qd = ctx.saved_tensors
        dev = ctx.engine.device
        g = [None if x is None else _f32c(x, dev) for x in (g_X_sc, g_X_sm, g_v_s)]
        gq, gqd = ctx.engine.link_state_backward(q, qd, *g, need=tuple(ctx.needs_input_grad[1:3]))
        return None, None if gq is None else gq.view(ctx.shapes[0]), None if gqd is None else gqd.view(ctx.shapes[1])


class ContactStateFunction(torch.autograd.Function):
    """(q, qd) -> (contact_f [N, C, 3], contact_height [N, C], body_f_contact [N, L, 6]): what the ground does to the links
    (``ArticulationEngine.contact_state``).  Saves only (q, qd): the backward recomputes the kinematics, so it is the same in
    "tape" and "recompute" adjoint mode."""

    @staticmethod
    def forward(ctx, engine, q, qd):
        qc, qdc = engine._contact_state_inputs(q, qd)
        out = engine.contact_state(qc, qdc)
        ctx.engine, ctx.shapes = engine, (q.shape, qd.shape)
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_contact_state_backward, not a zero fill
        ctx.save_for_backward(qc, qdc)
        return out

    @staticmethod
    def backward(ctx, g_f, g_h, g_body):
        q, qd = ctx.saved_tensors
        dev = ctx.engine.device
        g = [None if x is None else _f32c(x, dev) for x in (g_f, g_h, g_body)]
        gq, gqd = ctx.engine.contact_state_backward(q, qd, *g, need=tuple(ctx.needs_input_grad[1:3]))
        return None, None if gq is None else gq.view(ctx.shapes[0]), None if gqd is None else gqd.view(ctx.shapes[1])


class DynamicsStateFunction(torch.autograd.Function):
    """(q, qd, act, musc, f_ext) -> (joint_qdd [N, D], joint_tau [N, D], H [N, D, D]) (``ArticulationEngine.dynamics_state``).  Saves
    only its inputs: the backward re-runs a one-substep env-step into a workspace it allocates, so it is the same in "tape" and
    "recompute" adjoint mode.  musc and f_ext may be None."""

    @staticmethod
    def forward(ctx, engine, q, qd, act, musc, f_ext):
        ins = engine._dynamics_state_inputs(q, qd, act, musc, f_ext)
        out = engine._dynamics_state_checked(*ins)
        ctx.engine = engine
        ctx.shapes = tuple(None if t is None else t.shape for t in (q, qd, act, musc, f_ext))
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_dynamics_state_backward, not a zero fill
        ctx.save_for_backward(*ins)
        return out

    @staticmethod
    def backward(ctx, g_qdd, g_tau, g_H):
        ins = ctx.saved_tensors
        dev = ctx.engine.device
        g = [None if x is None else _f32c(x, dev) for x in (g_qdd, g_tau, g_H)]
        grads = ctx.engine.dynamics_state_backward(*ins, *g, need=tuple(ctx.needs_input_grad[1:6]))
        return (None,) + tuple(None if x is None else x.view(s) for x, s in zip(grads, ctx.shapes))


class JacobianStateFunction(torch.autograd.Function):
    """(q, qd) -> (J [N, L, 6, D], body_a_s [N, L, 6]): the link Jacobians and bias accelerations
    (``ArticulationEngine.jacobian_state``).  Saves only (q, qd): the backward recomputes the kinematics, so it is the same in
    "tape" and "recompute" adjoint mode."""

    @staticmethod
    def forward(ctx, engine, q, qd):
        qc, qdc = engine._jacobian_state_inputs(q, qd)
        out = engine.jacobian_state(qc, qdc)
        ctx.engine, ctx.shapes = engine, (q.shape, qd.shape)
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_jacobian_state_backward, not a zero fill
        ctx.save_for_backward(qc, qdc)
        return out

    @staticmethod
    def backward(ctx, g_J, g_a_s):
        q, qd = ctx.saved_tensors
        dev = ctx.engine.device
        g = [None if x is None else _f32c(x, dev) for x in (g_J, g_a_s)]
        gq, gqd = ctx.engine.jacobian_state_backward(q, qd, *g, need=tuple(ctx.needs_input_grad[1:3]))
        return None, None if gq is None else gq.view(ctx.shapes[0]), None if gqd is None else gqd.view(ctx.shapes[1])


class SimStepFunction(torch.autograd.Function):
    """(q, qd, act, musc[, f_ext]) -> (q', qd') for one env-step; the drop-in for the reference SimulateFunc.  ``f_ext``: optional
    external link wrenches [N, L, 6] (``check_wrench``); its gradient is returned when it requires one."""

    @staticmethod
    def forward(ctx, engine, substeps, mm_freq, dt, q, qd, act, musc, f_ext=None):
        needs = ctx.needs_input_grad[4:8]
        ctx.need_f_ext = len(ctx.needs_input_grad) > 8 and ctx.needs_input_grad[8]
        ctx.recompute = recompute_adjoint()
        f_ext = check_wrench(engine, f_ext)
        q_out, qd_out, tape, _ = engine.forward(q.detach(), qd.detach(), act.detach(),
                                                None if musc is None else musc.detach(),
                                                substeps, mm_freq, dt, want_tape=(any(needs) or ctx.need_f_ext) and not ctx.recompute,
                                                f_ext=f_ext)
        ctx.engine, ctx.cfg, ctx.needs = engine, (substeps, mm_freq, dt), needs
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_step_backward, not a zero fill
        ctx.shapes = (q.shape, qd.shape, act.shape, None if musc is None else musc.shape)
        musc = musc.detach() if (musc is not None and engine.M) else None
        if ctx.recompute:
            ctx.save_for_backward(act.detach(), musc, f_ext, q.detach(), qd.detach())   # the env-step's input state, in place of its tape
        else:
            ctx.save_for_backward(act.detach(), musc, f_ext, tape)
        return q_out.view(q.shape), qd_out.view(qd.shape)

    @staticmethod
    def backward(ctx, gq_out, gqd_out):
        substeps, mm_freq, dt = ctx.cfg
        wrench = dict(f_ext=None)
        if ctx.recompute:
            act, musc, f_ext, q, qd = ctx.saved_tensors
            if f_ext is not None:
                wrench = dict(f_ext=f_ext, need_f_ext=ctx.need_f_ext)
            g = ctx.engine.backward_recompute(q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt, need=tuple(ctx.needs), **wrench)
        else:
            act, musc, f_ext, tape = ctx.saved_tensors
            if f_ext is not None:
                wrench = dict(f_ext=f_ext, need_f_ext=ctx.need_f_ext)
            g = ctx.engine.backward(act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt, need=tuple(ctx.needs), **wrench)
        gq, gqd, gact, gmusc = g[:4]
        g_f_ext = g[4] if len(g) > 4 else None
        sq, sqd, sact, smusc = ctx.shapes
        return (None, None, None, None,
                None if gq is None else gq.view(sq), None if gqd is None else gqd.view(sqd),
                None if gact is None else gact.view(sact),
                None if (gmusc is None or smusc is None) else gmusc.view(smusc), g_f_ext)
