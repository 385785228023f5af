"""ctypes binding of libb200sparse.so (the C ABI declared in include/b200sparse.h).

This replaces the reference's cffi loader + Legate task launch
(reference legate_sparse/config.py:49-88, runtime.py:96-103): there the
only exported C symbol is ``legate_sparse_perform_registration`` and every
operation travels through a Legate ``TaskContext``; here every operation is a
plain ``extern "C"`` call on raw device pointers.

There is NO CPU fallback: if the shared library or a CUDA device is missing,
every compute entry point raises ``RuntimeError``.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_int, c_int64, c_uint64, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.normpath(os.path.join(_HERE, "..", "lib", "libb200sparse.so"))

# enums (include/b200sparse.h)
B2S_F32, B2S_F64, B2S_C64, B2S_C128 = 0, 1, 2, 3
B2S_I32, B2S_I64 = 0, 1
B2S_SPMV_AUTO, B2S_SPMV_ROWVEC, B2S_SPMV_TILE, B2S_SPMV_PIPE = 0, 1, 2, 3

_lib = None
_load_error = None

# name -> (restype, argtypes).  Keep in sync with include/b200sparse.h; the CPU test
# tests/test_cabi_symbols.py parses the header and checks this table against it.
_P = c_void_p
_I64 = c_int64
SIGNATURES = {
    "b2s_version": (c_int, []),
    "b2s_last_error_string": (c_char_p, []),
    "b2s_launch_count": (_I64, []),
    "b2s_spmv_plan_workspace_bytes": (_I64, [_I64, _I64]),
    "b2s_spmv_plan_create": (c_int, [c_int, _I64, _I64, _I64, _P, _P, _P, _I64, _P, POINTER(_P)]),
    "b2s_spmv_plan_destroy": (None, [_P]),
    "b2s_spmv_plan_info": (c_int, [_P, POINTER(_I64), POINTER(_I64), POINTER(_I64)]),
    "b2s_spmv_csr": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, c_int, _P]),
    "b2s_spmv_csr_bcast": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, c_int, _P, _P]),
    "b2s_spmv_csr_dot": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b2s_csr_colblock_suggest": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, POINTER(c_int)]),
    "b2s_csr_colblock_workspace_bytes": (_I64, [c_int, c_int, _I64, _I64, c_int]),
    "b2s_csr_colblock_create": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, c_int, _P, _I64, _P, POINTER(_P)]),
    "b2s_csr_colblock_destroy": (None, [_P]),
    "b2s_csr_colblock_info": (c_int, [_P, POINTER(c_int), POINTER(_I64), POINTER(_I64)]),
    "b2s_spmv_colblock": (c_int, [_P, _P, _P, _P, _P, _P, c_int, _P]),
    "b2s_spmv_colblock_part": (c_int, [_P, c_int, _P, _P, _P]),
    "b2s_cgs_workspace_bytes": (_I64, []),
    "b2s_cgs_project": (c_int, [c_int, _I64, c_int, _P, _I64, _P, _P, _P, _P]),
    "b2s_cgs_update": (c_int, [c_int, _I64, c_int, _P, _I64, _P, c_int, _P, _P, _P, _P]),
    "b2s_vscale_inv": (c_int, [c_int, _I64, _P, _P, _P, _P]),
    "b2s_axpby": (c_int, [c_int, _I64, _P, _P, _P, _P, c_int, c_int, _P]),
    "b2s_reduce_workspace_bytes": (_I64, []),
    "b2s_dot": (c_int, [c_int, _I64, _P, _P, c_int, _P, _P, _P]),
    "b2s_nrm2": (c_int, [c_int, _I64, _P, _P, _P, _P]),
    "b2s_cg_update": (c_int, [c_int, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b2s_cg_pupdate": (c_int, [c_int, _I64, _P, _P, _P, _P, _P]),
    "b2s_cg_pupdate_bcast": (c_int, [c_int, _I64, _P, _P, _P, _P, _P, c_int, _P]),
    "b2s_cg_pupdate_halo": (c_int, [c_int, _I64, _P, _P, _P, _P, _P, c_int, _P, _P, _P]),
    "b2s_board_bytes": (_I64, []),
    "b2s_allreduce_board": (c_int, [c_int, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    "b2s_cg_update_allreduce": (c_int, [c_int, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    "b2s_spmv_csr_dot_allreduce": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "b2s_spgemm_workspace_bytes": (_I64, [_I64, _I64, _I64]),
    "b2s_spgemm_symbolic": (
        c_int,
        [c_int, _I64, _I64, _I64, _P, _P, _I64, _P, _P, _I64, _P, _P, _I64, POINTER(_I64), POINTER(_I64), _P],
    ),
    "b2s_spgemm_numeric": (
        c_int,
        [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _I64, _P, _P, _P, _I64, _P, _P, _P, _P, _I64, _P],
    ),
    "b2s_csr_diagonal": (c_int, [c_int, c_int, _I64, _P, _P, _P, _P, _P]),
    "b2s_csr_expand_rows": (c_int, [_I64, _I64, _P, _P, _P]),
    "b2s_cast_i64_to_i32": (c_int, [_I64, _P, _P, _P]),
    "b2s_cast_i32_to_i64": (c_int, [_I64, _P, _P, _P]),
    "b2s_csr_to_dense": (c_int, [c_int, c_int, _I64, _I64, _P, _P, _P, _P, _P]),
    "b2s_scan_workspace_bytes": (_I64, [_I64]),
    "b2s_scan_i64": (c_int, [_I64, _P, _P, _I64, _P]),
    "b2s_dense_to_csr_count": (c_int, [c_int, _I64, _I64, _I64, _P, _P, _P]),
    "b2s_dense_to_csr_fill": (c_int, [c_int, c_int, _I64, _I64, _I64, _P, _P, _P, _P, _P]),
    "b2s_dia_to_csr_count": (c_int, [c_int, _I64, _I64, c_int, _I64, _I64, _P, _P, _P, _P, _P]),
    "b2s_dia_to_csr_fill": (c_int, [c_int, c_int, _I64, _I64, c_int, _I64, _I64, _P, _P, _P, _P, _P, _P, _P]),
    "b2s_random_csr_rowptr": (c_int, [_I64, _I64, c_uint64, _I64, _I64, _P, _P]),
    "b2s_random_csr_block_nnz": (_I64, [_I64, _I64, c_uint64, _I64, _I64]),
    "b2s_random_csr_fill": (c_int, [c_int, c_int, _I64, _I64, _I64, c_uint64, _I64, _I64, c_double, c_double, _P, _P, _P]),
}


def lib_path() -> str:
    return os.environ.get("B2S_LIBRARY", _LIB_PATH)


def load() -> ctypes.CDLL:
    """dlopen the library and declare every prototype (no CUDA call is made)."""
    global _lib, _load_error
    if _lib is not None:
        return _lib
    path = lib_path()
    try:
        lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
    except OSError as e:  # loud failure, no fallback
        _load_error = e
        raise RuntimeError(
            f"legate_sparse (b200): cannot load {path}: {e}. Build it with "
            "`python -c 'import __graft_entry__ as g; g.build()'` or `make -C legate-sparse_b200/csrc`."
        ) from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().b2s_last_error_string().decode("utf-8", "replace")


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise RuntimeError(f"libb200sparse {what} failed (code {rc}): {last_error()}")


def launch_count() -> int:
    return int(load().b2s_launch_count())
