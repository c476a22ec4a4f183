"""Argument refusals of the step, env-step and link-state entries of the C ABI (include/dfx.h), on a real pack.

Every step entry, its ``_ex`` twin and both link-state entries are called with one invalid argument (or several at once) and must
return cudaErrorInvalidValue (1) without a launch: a null required pointer; ``n``, ``substeps`` or ``mm_freq`` <= 0; an external
wrench without ``f_ext``; an action map with no actions, a negative offset, an offset past the actuation width or no strength; a
joint map on a muscle model without ``act_other``; a muscle model without ``musc``; a transition of the wrong kind or sizes, or
with a missing row.  The link-state entries with nothing to compute return 0, also without a launch.  Every pointer that is
present points into one zeroed device buffer large enough for any of these calls."""
import ctypes

import pytest
import torch

from emu_util import load_golden

pytestmark = pytest.mark.gpu

INVALID = 1
N, S, MM, DT = 4, 16, 16, 1.0 / 60.0

# argument names of each entry after (p, n, substeps, mm_freq, dt); the _ex twins append the wrench
STEP_ENTRIES = {
    "dfx_step_forward": "q qd act musc q_out qd_out tape derived stream",
    "dfx_step_backward": "act musc tape gq_out gqd_out gq gqd gact gmusc stream",
    "dfx_step_forward_mapped": "q qd map raw act_other used q_out qd_out tape stream",
    "dfx_step_backward_mapped": "map raw act_other tape gq_out gqd_out g_used gq gqd g_raw stream",
    "dfx_step_backward_recompute": "q qd act musc workspace gq_out gqd_out gq gqd gact gmusc stream",
    "dfx_step_backward_mapped_recompute": "q qd map raw act_other workspace gq_out gqd_out g_used gq gqd g_raw stream",
    "dfx_env_step_forward": "q qd map raw act_other used q_sim qd_sim tape tr stream",
    "dfx_env_step_backward": "map raw act_other tape tra gq gqd g_raw stream",
    "dfx_env_step_backward_recompute": "q qd map raw act_other workspace tra gq gqd g_raw stream",
}
# the pointers each entry requires (musc: on a model with muscles)
REQUIRED = {
    "dfx_step_forward": "q qd act q_out qd_out",
    "dfx_step_backward": "tape act",
    "dfx_step_forward_mapped": "q qd map raw q_out qd_out",
    "dfx_step_backward_mapped": "tape map raw",
    "dfx_step_backward_recompute": "q qd workspace act",
    "dfx_step_backward_mapped_recompute": "q qd workspace map raw",
    "dfx_env_step_forward": "q qd map raw used q_sim qd_sim tr",
    "dfx_env_step_backward": "tape map raw tra",
    "dfx_env_step_backward_recompute": "q qd workspace map raw tra",
}
TR_ROWS = ("progress", "start_q", "start_qd", "obs_before", "rew", "reset", "q_next", "qd_next", "actions_next", "progress_next",
           "obs_next")
TRA_ROWS = ("q_sim", "qd_sim", "used", "reset", "gq_sim", "gqd_sim", "g_used")


@pytest.fixture(scope="module")
def packs():
    from diffrl_b200 import _capi, env_ops
    from diffrl_b200.engine import ArticulationEngine
    lib = _capi.lib()
    env_ops._bind(lib)
    out = {}
    for name in ("AntEnv", "SNUHumanoidEnv"):
        _, model = load_golden(name)
        out[name] = ArticulationEngine.from_model(model, "cuda:0")      # (n = N in the calls: nothing launches)
    buf = torch.zeros(1 << 24, device="cuda:0")
    yield lib, out, buf
    torch.cuda.synchronize()


def _good(lib, eng, buf):
    """valid arguments for every name: the map and the transition match the pack"""
    from diffrl_b200 import env_ops
    from diffrl_b200.modelpack import DfxActionMap
    L, D, Q, M = (lib.dfx_pack_query(eng.pack, k) for k in (0, 1, 2, 4))
    ptr = ctypes.c_void_p(buf.data_ptr())
    na = min(8, D)
    v = dict(p=ctypes.c_void_p(eng.pack), n=N, substeps=S, mm_freq=MM, dt=DT, derived=None, stream=None,
             map=DfxActionMap(num_act=na, offset=D - na, is_muscle=0, pre_scale=1.0, pre_bias=0.0, drive_scale=1.0, strength=ptr.value),
             tr=env_ops.DfxEnvTransition(kind=1), tra=env_ops.DfxEnvTransitionAdj(kind=1))
    for t in (v["tr"], v["tra"]):
        t.walker.num_q, t.walker.num_qd, t.walker.num_act, t.walker.num_obs = Q, D, na, 37
        for row in TR_ROWS if isinstance(t, env_ops.DfxEnvTransition) else TRA_ROWS:
            setattr(t, row, ptr.value)
    for name in set(" ".join(STEP_ENTRIES.values()).split()) - set(v):
        v[name] = ptr
    return v, M


def _call(lib, entry, v, wrench=None):
    names = ["p", "n", "substeps", "mm_freq", "dt"] + STEP_ENTRIES[entry].split()
    args = [ctypes.byref(v[k]) if k in ("map", "tr", "tra") and v[k] is not None else v[k] for k in names]
    if wrench is not None:
        return getattr(lib, entry + "_ex")(*args, ctypes.byref(wrench))
    return getattr(lib, entry)(*args)


def _cases(entry, M):
    """(what, overrides, map edits, transition edits) of one refusal each"""
    req = REQUIRED[entry].split() + (["musc"] if M > 0 and "musc" in STEP_ENTRIES[entry].split() else [])
    cases = [("null p", dict(p=None), {}, {})]
    cases += [("null " + k, {k: None}, {}, {}) for k in req if k not in ("map", "tr", "tra")]
    if "map" in req:
        cases.append(("null map", dict(map=None), {}, {}))
    for k in ("tr", "tra"):
        if k in req:
            cases.append(("null " + k, {k: None}, {}, {}))
    cases += [("n = 0", dict(n=0), {}, {}), ("n < 0", dict(n=-3), {}, {}), ("substeps = 0", dict(substeps=0), {}, {}),
              ("mm_freq = 0", dict(mm_freq=0), {}, {}), ("mm_freq < 0", dict(mm_freq=-1), {}, {}),
              ("n = 0 and null p", dict(n=0, p=None), {}, {})]
    if "map" in req:
        cases += [("map without actions", {}, dict(num_act=0), {}), ("negative map offset", {}, dict(offset=-1), {}),
                  ("map past the actuation width", {}, dict(offset=1 << 20), {}), ("map without strength", {}, dict(strength=None), {}),
                  ("bad map and n = 0", dict(n=0), dict(offset=-1), {})]
        if M > 0:
            cases.append(("joint map without act_other on a muscle model", dict(act_other=None), {}, {}))
    tr = "tr" if "tr" in req else "tra" if "tra" in req else None
    if tr:
        rows = TR_ROWS if tr == "tr" else TRA_ROWS
        cases += [("transition kind 0", {}, {}, dict(kind=0)), ("transition kind 3", {}, {}, dict(kind=3)),
                  ("transition num_q mismatch", {}, {}, dict(num_q=1)), ("transition num_qd mismatch", {}, {}, dict(num_qd=1)),
                  ("transition num_act mismatch", {}, {}, dict(num_act=1)), ("transition without observations", {}, {}, dict(num_obs=0))]
        cases += [("transition without " + r, {}, {}, {r: None}) for r in rows]
    return cases


def _apply(v, over, map_edit, tr_edit):
    v = dict(v)
    v.update(over)
    for k, val in map_edit.items():
        setattr(v["map"], k, val)
    for key in ("tr", "tra"):
        t = v.get(key)
        if t is None:
            continue
        for k, val in tr_edit.items():
            setattr(t if k in ("kind",) + TR_ROWS + TRA_ROWS else t.walker, k, val)
    return v


@pytest.mark.parametrize("model", ["AntEnv", "SNUHumanoidEnv"])
@pytest.mark.parametrize("entry", sorted(STEP_ENTRIES))
@pytest.mark.parametrize("twin", ["plain", "_ex", "_ex without f_ext"])
def test_step_entries_refuse_invalid_arguments(packs, model, entry, twin):
    from diffrl_b200.modelpack import DfxExternalWrench
    lib, engines, buf = packs
    eng = engines[model]
    wrench = None if twin == "plain" else DfxExternalWrench(f_ext=buf.data_ptr(), g_f_ext=None)
    before = lib.dfx_launch_count()
    _, M = _good(lib, eng, buf)
    for what, over, map_edit, tr_edit in _cases(entry, M):
        v, _ = _good(lib, eng, buf)          # fresh structs per case
        got = _call(lib, entry, _apply(v, over, map_edit, tr_edit), wrench)
        assert got == INVALID, (model, entry, twin, what, got)
    if twin == "_ex without f_ext":          # the wrench alone, every other argument valid
        v, _ = _good(lib, eng, buf)
        assert _call(lib, entry, v, DfxExternalWrench(f_ext=None, g_f_ext=buf.data_ptr())) == INVALID, (model, entry)
    torch.cuda.synchronize()
    if entry != "dfx_env_step_backward":     # (its two-launch path runs the transition adjoint before the map is bound)
        assert lib.dfx_launch_count() == before, (model, entry, twin)


@pytest.mark.parametrize("model", ["AntEnv", "SNUHumanoidEnv"])
def test_link_state_entries_refuse_invalid_arguments(packs, model):
    lib, engines, buf = packs
    p, b = ctypes.c_void_p(engines[model].pack), ctypes.c_void_p(buf.data_ptr())
    before = lib.dfx_launch_count()
    fwd, bwd = lib.dfx_link_state_forward, lib.dfx_link_state_backward
    for n, pp, q, qd in ((N, None, b, b), (0, p, b, b), (-1, p, b, b), (N, p, None, b), (N, p, b, None), (0, p, None, None)):
        assert fwd(pp, n, q, qd, b, b, b, None) == INVALID, (model, n, pp, q, qd)
        assert bwd(pp, n, q, qd, b, b, b, b, b, None) == INVALID, (model, n, pp, q, qd)
    assert fwd(p, N, b, b, None, None, None, None) == 0          # nothing to compute
    assert bwd(p, N, b, b, b, b, b, None, None, None) == 0
    torch.cuda.synchronize()
    assert lib.dfx_launch_count() == before, model
