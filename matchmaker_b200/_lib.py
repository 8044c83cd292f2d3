"""ctypes binding of ``libmatchmaker_b200.so`` (the C ABI declared in ``include/matchmaker_b200.h``).

There is no CPU fallback anywhere in this package: if the shared library is missing or a
kernel cannot run, the call raises.
"""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# MMB200_LIB: load another build of the SAME library (A/B measurements of two kernel versions on one box); the default is
# the in-tree build.  Either way a missing file raises -- there is no fallback implementation behind it.
LIB_PATH = os.environ.get("MMB200_LIB") or os.path.join(_HERE, "csrc", "libmatchmaker_b200.so")

OK = 0
ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED = -1, -2, -3
F16, BF16, F32, F32_SPLIT16, F8E4M3 = 0, 1, 2, 3, 4
MASK_NONE, MASK_U8, MASK_I32, MASK_I64, MASK_F32 = 0, 1, 2, 3, 4
IMPL_AUTO, IMPL_SIMT, IMPL_TCGEN05, IMPL_TCGEN05_DOCM, IMPL_TCGEN05_RAGGED = 0, 1, 2, 3, 4

_c = ctypes
_vp, _i32, _i64, _f32 = _c.c_void_p, _c.c_int32, _c.c_int64, _c.c_float

# name -> (restype, argtypes); must list every symbol of include/matchmaker_b200.h
SIGNATURES = {
    "mmb200_version": (_c.c_int, []),
    "mmb200_last_error": (_c.c_char_p, []),
    "mmb200_device_info": (_c.c_int, [_c.c_int, _c.POINTER(_c.c_int), _c.POINTER(_c.c_int), _c.POINTER(_c.c_int)]),
    "mmb200_maxsim_fwd": (_c.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32,
                                     _i32, _i32, _i32, _i32, _vp]),
    "mmb200_maxsim_bwd": (_c.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32,
                                     _vp]),
    "mmb200_maxsim_allpairs_bwd": (_c.c_int, [_vp] * 6 + [_i64, _i64, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_maxsim_fwd_host": (_c.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32,
                                          _i64]),
    "mmb200_kernel_pool_fwd": (_c.c_int, [_vp] * 12 + [_i64, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _vp]),
    "mmb200_tkl_window_scores": (_c.c_int, [_vp] * 11 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_tkl_bwd": (_c.c_int, [_vp] * 18 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_tkl_top_hills": (_c.c_int, [_vp] * 6 + [_i64, _i32, _vp]),
    "mmb200_tkl_slot_map": (_c.c_int, [_vp, _vp, _i64, _vp]),
    "mmb200_flat_ip_workspace_bytes": (_i64, [_i64, _i64, _i32]),
    "mmb200_flat_ip_plan": (_c.c_int, [_i64, _i64, _i32, _i32, _c.POINTER(_i32)]),
    "mmb200_flat_ip_topk": (_c.c_int, [_vp] * 6 + [_i64, _i64, _i64, _i32, _i32, _i32, _i64, _vp]),
    "mmb200_topk_merge": (_c.c_int, [_vp] * 4 + [_i64, _i32, _i32, _vp]),
    "mmb200_topk_unique": (_c.c_int, [_vp] * 4 + [_i64, _i32, _i32, _vp]),
    "mmb200_ivf_workspace_bytes": (_i64, [_i64, _i32, _i64, _i64, _i32, _i32, _i32]),
    "mmb200_ivf_search": (_c.c_int, [_vp] * 8 + [_i64, _i64, _i32, _i64, _i64, _i64, _i32, _i32, _i32, _vp]),
    "mmb200_ivf_search_gather": (_c.c_int, [_vp] * 9 + [_i64, _i64, _i32, _i64, _i64, _i64, _i32, _i32, _i32, _vp]),
    "mmb200_ivf_list_means": (_c.c_int, [_vp] * 4 + [_i64, _i32, _i32, _vp]),
    "mmb200_residual_encode": (_c.c_int, [_vp] * 5 + [_i64, _i32, _i32, _vp]),
    "mmb200_residual_decode": (_c.c_int, [_vp] * 5 + [_i64, _i32, _i32, _vp]),
    "mmb200_ivf_search_residual": (_c.c_int, [_vp] * 4 + [_i32] + [_vp] * 7 + [_i64, _i64, _i32, _i64, _i64, _i64, _i32,
                                                                                _i32, _vp]),
    "mmb200_maxsim_store_residual_fwd": (_c.c_int, [_vp] * 5 + [_i32] + [_vp] * 4 + [_i64, _i64, _i64, _i64, _i32, _i32,
                                                                                        _i32, _vp]),
    "mmb200_plaid_centroid_scores": (_c.c_int, [_vp] * 4 + [_i64, _i32, _i64, _i32, _f32, _vp]),
    "mmb200_plaid_candidates": (_c.c_int, [_vp] * 5 + [_i64, _i32, _i64, _i64, _i64, _i64, _vp]),
    "mmb200_plaid_interaction": (_c.c_int, [_vp] * 6 + [_i64, _i32, _i64, _i64, _i64, _i64, _i32, _vp]),
    "mmb200_ah_workspace_bytes": (_i64, [_i64, _i32, _i64, _i64, _i32, _i32]),
    "mmb200_ah_search": (_c.c_int, [_vp] * 8 + [_i64, _i64, _i32, _i64, _i64, _i64, _i32, _i32, _vp]),
    "mmb200_ah_reorder": (_c.c_int, [_vp] * 6 + [_i64, _i64, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_graph_prune": (_c.c_int, [_vp, _vp, _i64, _i32, _i32, _vp]),
    "mmb200_graph_hash_slots": (_i64, [_i32, _i32]),
    "mmb200_graph_search": (_c.c_int, [_vp] * 7 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_maxsim_store_fwd": (_c.c_int, [_vp] * 6 + [_i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mmb200_dot_pairs": (_c.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    "mmb200_kernel_pool_bwd": (_c.c_int, [_vp] * 15 + [_i64, _i32, _i32, _i32, _i32, _f32, _i32, _vp]),
    "mmb200_kernel_pool_fwd_ex": (_c.c_int, [_vp] * 13 + [_i64, _i32, _i32, _i32, _i32, _f32, _f32, _f32, _i32, _i32, _vp]),
    "mmb200_kernel_pool_bwd_ex": (_c.c_int, [_vp] * 17 + [_i64, _i32, _i32, _i32, _i32, _f32, _f32, _i32, _vp]),
    "mmb200_kernel_pool_train_tc_supported": (_i32, [_i32, _i32, _i32, _i32]),
    "mmb200_kernel_pool_saved_floats": (_i64, [_i64, _i32]),
    "mmb200_kernel_pool_fwd_train": (_c.c_int, [_vp] * 13 + [_i64, _i32, _i32, _i32, _i32, _f32, _f32, _f32, _i32, _vp]),
    "mmb200_kernel_pool_bwd_saved": (_c.c_int, [_vp] * 18 + [_i64, _i32, _i32, _i32, _i32, _f32, _f32, _i32, _vp]),
    "mmb200_storage_load": (_c.c_int, [_c.POINTER(_c.c_char_p), _c.POINTER(_i64), _c.POINTER(_i64), _i32, _vp, _i64, _vp]),
}


class MatchmakerB200Error(RuntimeError):
    pass


_lock = threading.Lock()
_lib = None


def load() -> ctypes.CDLL:
    """Load the library (once).  Raises if it has not been built -- never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise MatchmakerB200Error(
                f"{LIB_PATH} not found: build it with `python -m matchmaker_b200.build` "
                "(there is no CPU/PyTorch fallback for the interaction kernels)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error() -> str:
    return load().mmb200_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != OK:
        kind = {ERR_INVALID: "invalid argument", ERR_CUDA: "CUDA error", ERR_UNSUPPORTED: "unsupported"}.get(rc, "error")
        raise MatchmakerB200Error(f"{what}: {kind} ({rc}): {last_error()}")
