"""ctypes binding of the C ABI in include/dfx.h (``diffrl_b200/libdfx.so``, built by ``__graft_entry__.build()``).

There is NO fallback: if the CUDA library is missing or cannot be loaded this raises, and every
product entry point goes through :func:`lib`.
"""
import ctypes
import os

from .modelpack import DfxActionMap, DfxDerived, DfxModelDesc

_HERE = os.path.dirname(os.path.abspath(__file__))
# DFX_LIBRARY points at another build of the SAME C ABI (same-box A/B timing of two kernel versions); never a fallback
LIB_PATH = os.environ.get("DFX_LIBRARY") or os.path.join(_HERE, "libdfx.so")

_F = ctypes.c_void_p  # raw device pointers
_lib = None


class DfxError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise DfxError(
            "diffrl_b200: CUDA library %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback for the simulation step." % LIB_PATH)
    try:
        L = ctypes.CDLL(LIB_PATH)
    except OSError as exc:  # e.g. libcudart missing
        raise DfxError("diffrl_b200: cannot load %s: %s" % (LIB_PATH, exc))
    L.dfx_version.restype = ctypes.c_char_p
    L.dfx_launch_count.restype = ctypes.c_longlong
    if hasattr(L, "dfx_launch_plan"):   # absent from older builds loaded through DFX_LIBRARY for A/B timing
        L.dfx_launch_plan.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.dfx_set_group_size.argtypes = [ctypes.c_int]
    if hasattr(L, "dfx_set_tile_envs"):
        L.dfx_set_tile_envs.argtypes = [ctypes.c_int]
        L.dfx_set_tape_dtype.argtypes = [ctypes.c_int]
    L.dfx_pack_create.restype = ctypes.c_void_p
    L.dfx_pack_create.argtypes = [ctypes.POINTER(DfxModelDesc), ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    L.dfx_pack_destroy.argtypes = [ctypes.c_void_p]
    L.dfx_pack_query.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.dfx_pack_set_gravity.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int]
    L.dfx_tape_floats.restype = ctypes.c_longlong
    L.dfx_tape_floats.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.dfx_step_forward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                   _F, _F, _F, _F, _F, _F, _F, ctypes.POINTER(DfxDerived), ctypes.c_void_p]
    L.dfx_step_backward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                    _F, _F, _F, _F, _F, _F, _F, _F, _F, ctypes.c_void_p]
    if hasattr(L, "dfx_step_forward_mapped"):
        L.dfx_step_forward_mapped.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                              _F, _F, ctypes.POINTER(DfxActionMap), _F, _F, _F, _F, _F, _F, ctypes.c_void_p]
        L.dfx_step_backward_mapped.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                               ctypes.POINTER(DfxActionMap), _F, _F, _F, _F, _F, _F, _F, _F, _F, ctypes.c_void_p]
    if hasattr(L, "dfx_step_backward_recompute"):     # recompute adjoint (include/dfx.h); env-step entry: env_ops._bind
        L.dfx_recompute_workspace_floats.restype = ctypes.c_longlong
        L.dfx_recompute_workspace_floats.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.dfx_step_backward_recompute.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                                  _F, _F, _F, _F, _F, _F, _F, _F, _F, _F, _F, ctypes.c_void_p]
        L.dfx_step_backward_mapped_recompute.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                                         _F, _F, ctypes.POINTER(DfxActionMap), _F, _F, _F, _F, _F, _F, _F, _F, _F,
                                                         ctypes.c_void_p]
    if os.environ.get("DFX_FLAGS"):      # tuning flags of include/dfx.h (A/B runs of the test-suite)
        L.dfx_set_flags(int(os.environ["DFX_FLAGS"]))
    _lib = L
    return L


def check(code, what):
    if code != 0:
        raise DfxError("%s failed with cudaError %d" % (what, code))
