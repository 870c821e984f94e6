"""ctypes binding of libccab200.so (the C ABI declared in include/ccab200.h).

The shared library is built in-tree by ``__graft_entry__.build()`` / ``make -C cca_zoo_b200/csrc``.
There is deliberately no fallback: if the library is missing or a call fails, a ``RuntimeError`` /
``ValueError`` is raised before any result is handed back.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libccab200.so")

F32, F64 = 0, 1
PREC_TF32, PREC_TF32X3, PREC_EXACT, PREC_TF32X3B = 0, 1, 2, 3
MAX_VIEWS = 8
# metric ids of ccab_pairwise_kernel (CCAB_KERNEL_* in include/ccab200.h)
KERNEL_METRICS = {"linear": 0, "poly": 1, "polynomial": 1, "rbf": 2, "sigmoid": 3, "cosine": 4, "laplacian": 5,
                  "chi2": 6, "additive_chi2": 7}

_i64p = C.POINTER(C.c_int64)
_vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/ccab200.h one to one
SIGNATURES = {
    "ccab_version": (C.c_int, []),
    "ccab_last_error": (C.c_char_p, []),
    "ccab_launch_count": (C.c_int64, []),
    "ccab_moments_size": (C.c_int64, [C.c_int, _i64p]),
    "ccab_moments_padded_dim": (C.c_int64, [C.c_int, _i64p]),
    "ccab_moments_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, _i64p, C.c_int64]),
    "ccab_moments": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(_vp), _i64p, _i64p, C.c_int64, _vp, _vp,
                               C.c_size_t, _vp]),
    "ccab_moments_packed_size": (C.c_int64, [C.c_int, _i64p]),
    "ccab_moments_pack": (C.c_int, [C.c_int, _i64p, _vp, C.c_double, _vp, _vp]),
    "ccab_moments_unpack": (C.c_int, [C.c_int, _i64p, _vp, _vp, _vp]),
    "ccab_moments_exchange_nvls": (C.c_int, [C.c_int, _i64p, _vp, C.c_double, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int,
                                             C.c_int64, C.c_uint, _vp, _vp]),
    "ccab_column_pilot": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, C.c_int64, _vp, _vp, _vp]),
    "ccab_shift_rows": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, C.c_int64, _vp, _vp, C.c_int64, _vp]),
    "ccab_moments_unshift": (C.c_int, [C.c_int, C.c_int, _i64p, _vp, C.POINTER(_vp), C.c_double, _vp]),
    "ccab_covariance": (C.c_int, [C.c_int, C.c_int, _i64p, _vp, C.c_double, C.c_int, _vp, C.c_int64, _vp, _vp]),
    "ccab_syevj_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ccab_syevj": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, C.c_int64, C.c_double, _vp, _vp, C.c_int64,
                             C.POINTER(C.c_int), C.POINTER(C.c_float), _vp, C.c_size_t, _vp]),
    "ccab_syevj_small": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, _vp, _vp]),
    "ccab_gesvj_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ccab_gesvj": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, _vp, C.c_int64,
                             C.POINTER(C.c_int), C.POINTER(C.c_float), _vp, C.c_size_t, _vp]),
    "ccab_gemm": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, C.c_int64, _vp,
                            C.c_int64, C.c_double, _vp, C.c_int64, _vp]),
    "ccab_gemm_tc": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, C.c_int64, C.c_int64, _vp,
                               C.c_int64, C.c_int64, C.c_double, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int64,
                               C.c_int, C.c_int, _vp]),
    "ccab_whiten_rows": (C.c_int, [C.c_int, C.c_int, _vp, _vp, C.c_int64, C.c_double, C.c_double, _vp, C.c_double,
                                   C.c_double, C.c_int, C.c_double, _vp, C.c_int64, _vp, _vp, _vp]),
    "ccab_ccaloss_small": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, C.c_double, _vp, _vp, _vp, _vp, _vp,
                                     _vp]),
    "ccab_potrf_inv_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "ccab_potrf_inv": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int64,
                                 C.c_double, _vp, _vp, C.c_size_t, _vp]),
    "ccab_rcca_fit_workspace_bytes": (C.c_size_t, [C.c_int, _i64p, C.c_int, C.c_int]),
    "ccab_rcca_fit_result_layout": (C.c_int, [C.c_int, _i64p, C.c_int, C.c_int, _i64p]),
    "ccab_rcca_fit": (C.c_int, [C.c_int, _i64p, _vp, _vp, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int,
                                C.c_int, _vp, C.c_size_t, _vp, C.c_size_t, _vp]),
    "ccab_ccaloss_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "ccab_ccaloss_fwd": (C.c_int, [C.c_int, C.c_int, _vp, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                   C.c_double, _vp, _vp, _vp, _vp, C.c_size_t, _vp]),
    "ccab_ccaloss_bwd": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int, C.c_int, _vp, _vp, _vp,
                                   C.c_int64, _vp, C.c_int64, _vp]),
    "ccab_mcca_fit_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64p, C.c_int, C.c_int]),
    "ccab_mcca_fit_result_layout": (C.c_int, [C.c_int, C.c_int, _i64p, C.c_int, C.c_int, _i64p]),
    "ccab_mcca_fit": (C.c_int, [C.c_int, C.c_int, _i64p, _vp, _vp, C.c_double, C.c_int, C.POINTER(C.c_double),
                                C.c_double, C.c_int, C.c_int, C.c_int, _vp, C.c_size_t, _vp, C.c_size_t, _vp]),
    "ccab_als_fit_workspace_bytes": (C.c_size_t, [C.c_int, _i64p]),
    "ccab_als_regression_workspace_bytes": (C.c_size_t, [C.c_int, _i64p]),
    "ccab_als_fit": (C.c_int, [C.c_int, C.c_int, _i64p, _vp, C.c_double, C.c_double, C.POINTER(C.c_double), C.c_double,
                               _vp, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, C.c_size_t, _vp]),
    "ccab_ey_fit_workspace_bytes": (C.c_size_t, [C.c_int, _i64p, C.c_int, C.c_int]),
    "ccab_ey_fit": (C.c_int, [C.c_int, _i64p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, _vp,
                              C.c_int, C.POINTER(_vp), _i64p, C.c_int, _vp, _vp, _vp, C.c_size_t, _vp]),
    "ccab_gfa_fit_workspace_bytes": (C.c_size_t, [C.c_int, _i64p, C.c_int]),
    "ccab_gfa_fit": (C.c_int, [C.c_int, _i64p, C.c_int, _vp, C.c_double, _vp, C.c_double, C.c_int, C.c_int, _vp, _vp,
                               C.c_size_t, _vp]),
    "ccab_tcca_moment_workspace_bytes": (C.c_size_t, [C.c_int, _i64p, C.c_int64, C.c_int]),
    "ccab_tcca_moment": (C.c_int, [C.c_int, _i64p, C.c_int64, C.POINTER(_vp), _i64p, C.c_double, C.c_int, _vp, _vp,
                                   C.c_size_t, _vp]),
    "ccab_tcca_state_size": (C.c_int64, [C.c_int, _i64p, C.c_int]),
    "ccab_tcca_fit_workspace_bytes": (C.c_size_t, [C.c_int, _i64p, C.c_int]),
    "ccab_tcca_fit": (C.c_int, [C.c_int, _i64p, C.c_int, _vp, C.POINTER(_vp), _vp, _vp, C.c_int, C.c_int, _vp, _vp,
                                C.c_size_t, _vp]),
    "ccab_pairwise_kernel_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64]),
    "ccab_pairwise_kernel": (C.c_int, [C.c_int, C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int,
                                       C.c_double, C.c_double, C.c_double, _vp, C.c_int64, _vp, C.c_size_t, _vp]),
    "ccab_scale": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int64,
                             _vp]),
    "ccab_center_columns": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, _vp]),
    "ccab_frobenius_norm": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int64, _vp, _vp]),
    "ccab_profile_moments": (C.c_int, [C.c_int]),
    "ccab_profile_moments_last_ms": (C.c_double, []),
}

_lib = None


def load():
    """Load (once) and return the ctypes handle; raises if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C cca_zoo_b200/csrc`).  cca_zoo_b200 has no CPU fallback."
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error() -> str:
    return load().ccab_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    """Turn a non-zero return code into an exception (ValueError for argument errors)."""
    if rc == 0:
        return
    msg = f"{what} failed (code {rc}): {last_error()}"
    if rc < 0:
        raise ValueError(msg)
    raise RuntimeError(msg)


def i64_array(values):
    return (C.c_int64 * len(values))(*[int(v) for v in values])
