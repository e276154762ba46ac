"""ctypes binding of libbcone.so (the C ABI declared in include/bcone.h).

There is no CPU fallback: if the CUDA library is missing or no CUDA device is present the
engine raises.  The library is built in-tree by ``cvxpylayers_b200.build`` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
# (BCONE_LIB: a development build of the same library, e.g. one compiled with -DBC_SUBPROF; the product path is the in-tree file)
LIB_PATH = Path(os.environ["BCONE_LIB"]) if os.environ.get("BCONE_LIB") else _PKG / "libbcone.so"

_i32p = C.POINTER(C.c_int32)
_f64p = C.POINTER(C.c_double)

EXPORTS = [
    "bcone_default_settings", "bcone_create", "bcone_destroy", "bcone_last_error", "bcone_set_boundary", "bcone_set_boundary_quad",
    "bcone_ingest", "bcone_emit", "bcone_ingest_pitched", "bcone_emit_pitched", "bcone_peer_alloc", "bcone_peer_open", "bcone_peer_close",
    "bcone_peer_free", "bcone_copy2d_async", "bcone_rows_from_param", "bcone_param_from_rows", "bcone_gather_cols", "bcone_scatter_cols", "bcone_set_param_maps", "bcone_ingest_params", "bcone_emit_params", "bcone_solve", "bcone_solve_warm", "bcone_solve_cached", "bcone_cache_bytes", "bcone_vjp", "bcone_jvp", "bcone_launch_count", "bcone_fallback_count", "bcone_kernel_info", "bcone_path_info", "bcone_small_cta_info", "bcone_memcpy2d", "bcone_set_profile",
    "bcone_solve_shared", "bcone_vjp_shared", "bcone_jvp_shared", "bcone_ingest_params_shared", "bcone_emit_params_shared",
]


class BconeDesc(C.Structure):
    _fields_ = [("n", C.c_int32), ("m", C.c_int32), ("nnzA", C.c_int32), ("nnzP", C.c_int32),
                ("A_indptr", _i32p), ("A_indices", _i32p), ("P_indptr", _i32p), ("P_indices", _i32p),
                ("z", C.c_int32), ("l", C.c_int32), ("nq", C.c_int32), ("ns", C.c_int32),
                ("ep", C.c_int32), ("ed", C.c_int32), ("q", _i32p), ("s", _i32p),
                ("device", C.c_int32), ("max_batch", C.c_int32)]


class BconeSettings(C.Structure):
    _fields_ = [("eps_abs", C.c_double), ("eps_rel", C.c_double), ("eps_infeas", C.c_double),
                ("alpha", C.c_double), ("rho_x", C.c_double), ("scale", C.c_double),
                ("lsqr_atol", C.c_double), ("lsqr_btol", C.c_double), ("lsqr_conlim", C.c_double),
                ("max_iters", C.c_int32), ("normalize", C.c_int32), ("adaptive_scale", C.c_int32),
                ("check_interval", C.c_int32), ("ruiz_passes", C.c_int32), ("lsqr_iter_lim", C.c_int32),
                ("lsqr_precond", C.c_int32), ("adaptive_check", C.c_int32),
                ("acceleration_lookback", C.c_int32), ("acceleration_interval", C.c_int32)]


class EngineUnavailable(RuntimeError):
    """libbcone.so is missing / cannot be loaded. There is deliberately no fallback."""


_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise EngineUnavailable(
            f"{LIB_PATH} not found: build it with `python -m cvxpylayers_b200.build` (nvcc, sm_90a). "
            "The engine has no CPU or PyTorch fallback.")
    try:
        lib = C.CDLL(str(LIB_PATH))
    except OSError as e:  # pragma: no cover
        raise EngineUnavailable(f"cannot load {LIB_PATH}: {e}") from e
    vp = C.c_void_p
    lib.bcone_default_settings.argtypes = [C.POINTER(BconeSettings)]
    lib.bcone_default_settings.restype = None
    lib.bcone_create.argtypes = [C.POINTER(BconeDesc), C.POINTER(vp)]
    lib.bcone_create.restype = C.c_int
    lib.bcone_destroy.argtypes = [vp]
    lib.bcone_destroy.restype = None
    lib.bcone_last_error.argtypes = [vp]
    lib.bcone_last_error.restype = C.c_char_p
    lib.bcone_set_boundary.argtypes = [vp, C.c_int32, _i32p, C.c_int32, _i32p]
    lib.bcone_set_boundary.restype = C.c_int
    lib.bcone_set_boundary_quad.argtypes = [vp, C.c_int32, _i32p]
    lib.bcone_set_boundary_quad.restype = C.c_int
    lib.bcone_ingest.argtypes = [vp, C.c_int32] + [vp] * 8
    lib.bcone_ingest.restype = C.c_int
    lib.bcone_emit.argtypes = [vp, C.c_int32] + [vp] * 8
    lib.bcone_emit.restype = C.c_int
    lib.bcone_ingest_pitched.argtypes = [vp, C.c_int32, C.c_int64] + [vp] * 8
    lib.bcone_ingest_pitched.restype = C.c_int
    lib.bcone_emit_pitched.argtypes = [vp, C.c_int32, C.c_int64] + [vp] * 8
    lib.bcone_emit_pitched.restype = C.c_int
    lib.bcone_peer_alloc.argtypes = [C.c_int32, C.c_int64, C.POINTER(vp), vp]
    lib.bcone_peer_alloc.restype = C.c_int
    lib.bcone_peer_open.argtypes = [C.c_int32, vp, C.POINTER(vp)]
    lib.bcone_peer_open.restype = C.c_int
    lib.bcone_peer_close.argtypes = [vp]
    lib.bcone_peer_close.restype = C.c_int
    lib.bcone_peer_free.argtypes = [vp]
    lib.bcone_peer_free.restype = C.c_int
    lib.bcone_copy2d_async.argtypes = [vp, C.c_int64, vp, C.c_int64, C.c_int64, C.c_int64, vp]
    lib.bcone_copy2d_async.restype = C.c_int
    lib.bcone_rows_from_param.argtypes = [vp, C.c_int64, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.bcone_rows_from_param.restype = C.c_int
    lib.bcone_param_from_rows.argtypes = [vp, vp, C.c_int64, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.bcone_param_from_rows.restype = C.c_int
    lib.bcone_gather_cols.argtypes = [vp, C.c_int64, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.bcone_gather_cols.restype = C.c_int
    lib.bcone_scatter_cols.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    lib.bcone_scatter_cols.restype = C.c_int
    lib.bcone_set_param_maps.argtypes = [vp, C.c_int32] + [_i32p, _i32p, _f64p] * 3
    lib.bcone_set_param_maps.restype = C.c_int
    lib.bcone_ingest_params.argtypes = [vp, C.c_int32] + [vp] * 6
    lib.bcone_ingest_params.restype = C.c_int
    lib.bcone_emit_params.argtypes = [vp, C.c_int32] + [vp] * 6
    lib.bcone_emit_params.restype = C.c_int
    lib.bcone_solve.argtypes = [vp, C.c_int32] + [vp] * 10 + [C.POINTER(BconeSettings), vp]
    lib.bcone_solve.restype = C.c_int
    lib.bcone_solve_warm.argtypes = [vp, C.c_int32] + [vp] * 13 + [C.POINTER(BconeSettings), vp]
    lib.bcone_solve_warm.restype = C.c_int
    lib.bcone_solve_cached.argtypes = [vp, C.c_int32] + [vp] * 13 + [vp, C.c_int32, C.POINTER(BconeSettings), vp]
    lib.bcone_solve_cached.restype = C.c_int
    lib.bcone_cache_bytes.argtypes = [vp, C.c_int32]
    lib.bcone_cache_bytes.restype = C.c_size_t
    lib.bcone_vjp.argtypes = [vp, C.c_int32] + [vp] * 14 + [C.POINTER(BconeSettings), vp]
    lib.bcone_vjp.restype = C.c_int
    lib.bcone_jvp.argtypes = [vp, C.c_int32] + [vp] * 15 + [C.POINTER(BconeSettings), vp]
    lib.bcone_jvp.restype = C.c_int
    lib.bcone_solve_shared.argtypes = [vp, C.c_int32] + [vp] * 13 + [C.POINTER(BconeSettings), vp]
    lib.bcone_solve_shared.restype = C.c_int
    lib.bcone_vjp_shared.argtypes = [vp, C.c_int32] + [vp] * 14 + [C.POINTER(BconeSettings), vp]
    lib.bcone_vjp_shared.restype = C.c_int
    lib.bcone_jvp_shared.argtypes = [vp, C.c_int32] + [vp] * 15 + [C.POINTER(BconeSettings), vp]
    lib.bcone_jvp_shared.restype = C.c_int
    lib.bcone_ingest_params_shared.argtypes = [vp, C.c_int32] + [vp] * 6
    lib.bcone_ingest_params_shared.restype = C.c_int
    lib.bcone_emit_params_shared.argtypes = [vp, C.c_int32] + [vp] * 6
    lib.bcone_emit_params_shared.restype = C.c_int
    lib.bcone_memcpy2d.argtypes = [vp, C.c_int64, vp, C.c_int64, C.c_int64, C.c_int64, C.c_int32, vp]
    lib.bcone_memcpy2d.restype = C.c_int
    lib.bcone_set_profile.argtypes = [vp, C.c_int32, C.POINTER(C.c_uint64)]
    lib.bcone_set_profile.restype = C.c_int
    lib.bcone_launch_count.argtypes = [vp]
    lib.bcone_launch_count.restype = C.c_int64
    lib.bcone_fallback_count.argtypes = [vp, _i32p]
    lib.bcone_fallback_count.restype = C.c_int
    lib.bcone_kernel_info.argtypes = [vp] + [_i32p] * 6
    lib.bcone_kernel_info.restype = C.c_int
    lib.bcone_path_info.argtypes = [vp, _i32p, _i32p]
    lib.bcone_path_info.restype = C.c_int
    lib.bcone_small_cta_info.argtypes = [vp, _i32p, _i32p]
    lib.bcone_small_cta_info.restype = C.c_int
    _lib = lib
    return lib


def default_settings() -> BconeSettings:
    st = BconeSettings()
    load().bcone_default_settings(C.byref(st))
    return st
