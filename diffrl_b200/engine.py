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
from .modelpack import DfxDerived, articulation_from_model

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

    def forward(self, q, qd, act, musc, substeps, mm_freq, dt, want_tape=True, derived=None, out=None):
        """Returns (q_out, qd_out, tape or None).  ``derived``: optional dict name -> bool of dumps to
        fill (returned as a dict of tensors under key 'derived' attribute of the result tuple)."""
        dev = self.device
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
        with torch.cuda.device(dev):
            code = self.lib.dfx_step_forward(self.pack, self.N, int(substeps), int(mm_freq), float(dt),
                                             _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(q_out), _ptr(qd_out),
                                             _ptr(tape), None if dv is None else ctypes.byref(dv), self._stream())
        _capi.check(code, "dfx_step_forward")
        return q_out, qd_out, tape, dumps

    def backward(self, act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt, need=(True, True, True, True)):
        dev = self.device
        act = _f32c(act, dev)
        musc = _f32c(musc, dev) if self.M else None
        gq_out = None if gq_out is None else _f32c(gq_out, dev)
        gqd_out = None if gqd_out is None else _f32c(gqd_out, dev)
        gq = torch.empty(self.N * self.Q, dtype=torch.float32, device=dev) if need[0] else None
        gqd = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[1] else None
        gact = torch.empty(self.N * self.D, dtype=torch.float32, device=dev) if need[2] else None
        gmusc = torch.empty(self.N * self.M, dtype=torch.float32, device=dev) if (need[3] and self.M) else None
        with torch.cuda.device(dev):
            code = self.lib.dfx_step_backward(self.pack, self.N, int(substeps), int(mm_freq), float(dt),
                                              _ptr(act), _ptr(musc), _ptr(tape), _ptr(gq_out), _ptr(gqd_out),
                                              _ptr(gq), _ptr(gqd), _ptr(gact), _ptr(gmusc), self._stream())
        _capi.check(code, "dfx_step_backward")
        return gq, gqd, gact, gmusc

    def backward_recompute(self, q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt, need=(True, True, True, True),
                           workspace=None):
        """``backward`` without a tape: the env-step's forward from (q, qd, act, musc) is re-run into a workspace inside the
        adjoint launch (``dfx_step_backward_recompute``).  ``workspace`` (``recompute_workspace()``): used and left readable
        (``tape_rows``, ``tape_hinv``, ``workspace_end_state``); None: one from the caching allocator."""
        dev = self.device
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
        with torch.cuda.device(dev):
            code = self.lib.dfx_step_backward_recompute(self.pack, self.N, int(substeps), int(mm_freq), float(dt),
                                                        _ptr(q), _ptr(qd), _ptr(act), _ptr(musc), _ptr(workspace),
                                                        _ptr(gq_out), _ptr(gqd_out), _ptr(gq), _ptr(gqd), _ptr(gact), _ptr(gmusc),
                                                        self._stream())
        _capi.check(code, "dfx_step_backward_recompute")
        return gq, gqd, gact, gmusc


class MappedSimStepFunction(torch.autograd.Function):
    """(q, qd, raw policy output) -> (q', qd', used): the env-step with the action map folded into the simulation launch
    (``dfx_step_forward_mapped`` / ``dfx_step_backward_mapped``): ``used = clip(raw, -1, 1) * pre_scale + pre_bias`` (the env's
    ``actions``), ``joint_act`` / the muscle activations are formed inside the kernel.  ``amap`` = (offset, pre_scale, pre_bias,
    drive_scale, strength [A], is_muscle)."""

    @staticmethod
    def forward(ctx, engine, substeps, mm_freq, dt, amap, q, qd, raw):
        from .modelpack import DfxActionMap
        offset, pre_scale, pre_bias, drive_scale, strength, is_muscle = amap
        dev = engine.device
        q, qd = _f32c(q.detach(), dev), _f32c(qd.detach(), dev)
        raw = _f32c(raw.detach(), dev)
        n, A = engine.N, raw.shape[-1]
        m = DfxActionMap(int(A), int(offset), int(bool(is_muscle)), float(pre_scale), float(pre_bias), float(drive_scale), strength.data_ptr())
        need = any(ctx.needs_input_grad[5:8])
        ctx.recompute = recompute_adjoint()
        q_out, qd_out, used = torch.empty_like(q), torch.empty_like(qd), torch.empty_like(raw)
        tape = torch.empty(engine.tape_floats(substeps, mm_freq), dtype=torch.float32, device=dev) if (need and not ctx.recompute) else None
        with torch.cuda.device(dev):
            code = engine.lib.dfx_step_forward_mapped(engine.pack, n, int(substeps), int(mm_freq), float(dt), _ptr(q), _ptr(qd),
                                                      ctypes.byref(m), _ptr(raw), None, _ptr(used), _ptr(q_out), _ptr(qd_out),
                                                      _ptr(tape), engine._stream())
        _capi.check(code, "dfx_step_forward_mapped")
        ctx.engine, ctx.cfg, ctx.amap = engine, (substeps, mm_freq, dt), m
        ctx.strength = strength                      # keeps the device array the struct points at alive
        ctx.set_materialize_grads(False)
        ctx.shapes = (q.shape, qd.shape)
        if ctx.recompute:
            ctx.save_for_backward(raw, q, qd)        # the env-step's input state, in place of its tape
        else:
            ctx.save_for_backward(raw, tape)
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
            raw, q, qd = ctx.saved_tensors
            g_raw = torch.empty_like(raw)
            workspace = engine.recompute_workspace(substeps, mm_freq)
            with torch.cuda.device(dev):
                code = engine.lib.dfx_step_backward_mapped_recompute(engine.pack, engine.N, int(substeps), int(mm_freq), float(dt),
                                                                     _ptr(q), _ptr(qd), ctypes.byref(ctx.amap), _ptr(raw), None,
                                                                     _ptr(workspace), *cot, _ptr(g_raw), engine._stream())
            _capi.check(code, "dfx_step_backward_mapped_recompute")
        else:
            raw, tape = ctx.saved_tensors
            g_raw = torch.empty_like(raw)
            with torch.cuda.device(dev):
                code = engine.lib.dfx_step_backward_mapped(engine.pack, engine.N, int(substeps), int(mm_freq), float(dt), ctypes.byref(ctx.amap),
                                                           _ptr(raw), None, _ptr(tape), *cot, _ptr(g_raw), engine._stream())
            _capi.check(code, "dfx_step_backward_mapped")
        return None, None, None, None, None, gq.view(ctx.shapes[0]), gqd.view(ctx.shapes[1]), g_raw


class SimStepFunction(torch.autograd.Function):
    """(q, qd, act, musc) -> (q', qd') for one env-step; the drop-in for the reference SimulateFunc."""

    @staticmethod
    def forward(ctx, engine, substeps, mm_freq, dt, q, qd, act, musc):
        needs = ctx.needs_input_grad[4:8]
        ctx.recompute = recompute_adjoint()
        q_out, qd_out, tape, _ = engine.forward(q.detach(), qd.detach(), act.detach(),
                                                None if musc is None else musc.detach(),
                                                substeps, mm_freq, dt, want_tape=any(needs) and not ctx.recompute)
        ctx.engine, ctx.cfg, ctx.needs = engine, (substeps, mm_freq, dt), needs
        ctx.set_materialize_grads(False)      # a missing cotangent is NULL for dfx_step_backward, not a zero fill
        ctx.shapes = (q.shape, qd.shape, act.shape, None if musc is None else musc.shape)
        musc = musc.detach() if (musc is not None and engine.M) else None
        if ctx.recompute:
            ctx.save_for_backward(act.detach(), musc, q.detach(), qd.detach())   # the env-step's input state, in place of its tape
        else:
            ctx.save_for_backward(act.detach(), musc, tape)
        return q_out.view(q.shape), qd_out.view(qd.shape)

    @staticmethod
    def backward(ctx, gq_out, gqd_out):
        substeps, mm_freq, dt = ctx.cfg
        if ctx.recompute:
            act, musc, q, qd = ctx.saved_tensors
            gq, gqd, gact, gmusc = ctx.engine.backward_recompute(q, qd, act, musc, gq_out, gqd_out, substeps, mm_freq, dt,
                                                                 need=tuple(ctx.needs))
        else:
            act, musc, tape = ctx.saved_tensors
            gq, gqd, gact, gmusc = ctx.engine.backward(act, musc, tape, gq_out, gqd_out, substeps, mm_freq, dt,
                                                       need=tuple(ctx.needs))
        sq, sqd, sact, smusc = ctx.shapes
        return (None, None, None, None,
                None if gq is None else gq.view(sq), None if gqd is None else gqd.view(sqd),
                None if gact is None else gact.view(sact),
                None if (gmusc is None or smusc is None) else gmusc.view(smusc))
