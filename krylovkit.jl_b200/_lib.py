"""ctypes binding of libb200krylov.so — the C-ABI declared in include/b200krylov.h.

This module is the *only* way the host code reaches the GPU.  There is no CPU fallback:
if the shared library is missing or a call fails, an exception is raised.

Status codes map to exceptions the way the Julia shim maps them to Julia exceptions
(INTEGRATION.md): B2K_EINVAL -> ValueError (ArgumentError), B2K_EDIM -> DimensionMismatch,
everything else -> B200Error.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200krylov.so")

# status codes / enums (mirror include/b200krylov.h)
OK, EINVAL, EDIM, ECUDA, ENOMEM, ENCCL, ENOTSUP = 0, -1, -2, -3, -4, -5, -6
F64, F32 = 0, 1
CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)


class B200Error(RuntimeError):
    """CUDA / NCCL / resource failure inside libb200krylov."""


class DimensionMismatch(ValueError):
    """Mirror of Julia's DimensionMismatch (src/orthonormal.jl:93,140,158-161)."""


class LibraryMissing(B200Error):
    pass


_lib = None

c_vec = C.c_int32
c_ctx = C.c_void_p
c_op = C.c_void_p
P = C.POINTER

_PROTOS = {
    # name: (restype, [argtypes])
    "b2k_abi_version": (C.c_int32, []),
    "b2k_last_error": (C.c_char_p, [c_ctx]),
    "b2k_ctx_create": (C.c_int32, [P(c_ctx), C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "b2k_ctx_create_dist": (C.c_int32, [P(c_ctx), C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int64]),
    "b2k_nccl_unique_id": (C.c_int32, [C.c_void_p]),
    "b2k_ctx_destroy": (C.c_int32, [c_ctx]),
    "b2k_space_create": (C.c_int32, [c_ctx, C.c_int64, C.c_int32, C.c_int32, P(C.c_int32)]),
    "b2k_ctx_sync": (C.c_int32, [c_ctx]),
    "b2k_ctx_launch_count": (C.c_int64, [c_ctx]),
    "b2k_ctx_stream": (C.c_void_p, [c_ctx]),
    "b2k_prof_enable": (C.c_int32, [c_ctx, C.c_int32]),
    "b2k_prof_reset": (C.c_int32, [c_ctx]),
    "b2k_prof_read": (C.c_int32, [c_ctx, C.c_int32, P(C.c_int64), P(C.c_double), P(C.c_double)]),
    "b2k_timer_start": (C.c_int32, [c_ctx]),
    "b2k_timer_stop": (C.c_int32, [c_ctx, P(C.c_double)]),
    "b2k_pinned_alloc": (C.c_int32, [C.c_size_t, P(C.c_void_p)]),
    "b2k_pinned_free": (C.c_int32, [C.c_void_p]),
    "b2k_device_sync": (C.c_int32, []),
    "b2k_cache_release": (C.c_int32, []),
    "b2k_vec_alloc": (C.c_int32, [c_ctx, C.c_int32, P(c_vec)]),
    "b2k_vec_alloc_range": (C.c_int32, [c_ctx, C.c_int32, C.c_int32, P(c_vec)]),
    "b2k_vec_free": (C.c_int32, [c_ctx, c_vec]),
    "b2k_vec_upload": (C.c_int32, [c_ctx, c_vec, C.c_void_p]),
    "b2k_vec_download": (C.c_int32, [c_ctx, c_vec, C.c_void_p]),
    "b2k_vec_copy": (C.c_int32, [c_ctx, c_vec, c_vec]),
    "b2k_vec_zero": (C.c_int32, [c_ctx, c_vec]),
    "b2k_vec_fill_splitmix": (C.c_int32, [c_ctx, c_vec, C.c_uint64]),
    "b2k_vec_fill": (C.c_int32, [c_ctx, c_vec, C.c_double]),
    "b2k_vec_inner": (C.c_int32, [c_ctx, c_vec, c_vec, P(C.c_double)]),
    "b2k_vec_norm": (C.c_int32, [c_ctx, c_vec, P(C.c_double)]),
    "b2k_vec_axpby": (C.c_int32, [c_ctx, c_vec, c_vec, C.c_double, C.c_double]),
    "b2k_vec_scale": (C.c_int32, [c_ctx, c_vec, c_vec, C.c_double]),
    "b2k_vec_axpy2": (C.c_int32, [c_ctx, c_vec, c_vec, C.c_double, c_vec, C.c_double]),
    "b2k_op_create_csr": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "b2k_op_create_csc": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "b2k_op_create_stencil": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_int64,
                                          P(C.c_double)]),
    "b2k_op_create_stencil_free": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_int64,
                                               P(C.c_double)]),
    "b2k_op_create_dense": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_void_p, C.c_int64]),
    "b2k_op_create_dense_splitmix": (C.c_int32, [c_ctx, P(c_op), C.c_int64, C.c_int64, C.c_uint64]),
    "b2k_op_destroy": (C.c_int32, [c_ctx, c_op]),
    "b2k_op_info": (C.c_int32, [c_op, P(C.c_int64), P(C.c_int64), P(C.c_int64), P(C.c_int32)]),
    "b2k_op_csr_download": (C.c_int32, [c_ctx, c_op, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2k_op_create_transpose": (C.c_int32, [c_ctx, P(c_op), c_op]),
    "b2k_op_apply": (C.c_int32, [c_ctx, c_op, c_vec, c_vec]),
    "b2k_op_apply_shifted": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, C.c_double, C.c_double]),
    "b2k_op_apply_adjoint": (C.c_int32, [c_ctx, c_op, c_vec, c_vec]),
    "b2k_op_apply_normal_gram": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec]),
    "b2k_op_apply_dot": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec, P(C.c_double)]),
    "b2k_cg_step": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec, c_vec, C.c_double, C.c_double, C.c_double,
                                C.c_double, P(C.c_double), P(C.c_double)]),
    "b2k_cg_chain": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec, c_vec, C.c_double, C.c_double, C.c_double,
                                 C.c_double, C.c_double, C.c_int32, P(C.c_double), P(C.c_double), P(C.c_int32)]),
    "b2k_bicgstab_half": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec, c_vec, c_vec, C.c_double, C.c_double,
                                      C.c_double, C.c_double, C.c_double, C.c_int32, P(C.c_double),
                                      P(C.c_double)]),
    "b2k_bicgstab_full": (C.c_int32, [c_ctx, c_op, c_vec, c_vec, c_vec, c_vec, c_vec, c_vec, C.c_double,
                                      C.c_double, C.c_double, P(C.c_double), P(C.c_double), P(C.c_double)]),
    "b2k_bicgstab_chain": (C.c_int32, [c_ctx, c_op] + [c_vec] * 7 + [C.c_double] * 7 +
                           [C.c_int32, P(C.c_double), P(C.c_int32)]),
    "b2k_basis_project": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, c_vec, C.c_double, C.c_double,
                                      P(C.c_double)]),
    "b2k_basis_cross_inner": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(c_vec), C.c_int32, C.c_int32, C.c_int32,
                                          P(C.c_double), C.c_int32]),
    "b2k_basis_unproject": (C.c_int32, [c_ctx, c_vec, P(c_vec), C.c_int32, P(C.c_double), C.c_double,
                                        C.c_double]),
    "b2k_basis_orthogonalize": (C.c_int32, [c_ctx, c_vec, P(c_vec), C.c_int32, P(C.c_double),
                                            C.c_int32, C.c_double, P(C.c_double), P(C.c_int32)]),
    "b2k_vec_orthogonalize": (C.c_int32, [c_ctx, c_vec, c_vec, C.c_int32, C.c_double, P(C.c_double),
                                          P(C.c_double)]),
    "b2k_lanczos_expand": (C.c_int32, [c_ctx, c_op, P(c_vec), C.c_int32, c_vec, c_vec, C.c_double,
                                       C.c_int32, C.c_double, P(C.c_double), P(C.c_double)]),
    "b2k_lanczos_expand_many": (C.c_int32, [c_ctx, c_op, P(c_vec), C.c_int32, C.c_int32, C.c_double,
                                            C.c_double, C.c_int32, C.c_double, P(C.c_double),
                                            P(C.c_double), P(C.c_int32), P(c_vec)]),
    "b2k_basis_transform": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(C.c_double), C.c_int32,
                                        C.c_int32]),
    "b2k_basis_rank1update": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, c_vec, P(C.c_double),
                                          C.c_double, C.c_double]),
    "b2k_basis_givens": (C.c_int32, [c_ctx, c_vec, c_vec, C.c_double, C.c_double]),
    "b2k_basis_householder": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(C.c_double), C.c_double,
                                          c_vec]),
    "b2k_host_lanczos_restart": (C.c_int32, [C.c_int32, C.c_int32, P(C.c_double), P(C.c_double),
                                             P(C.c_double), C.c_int32, P(C.c_double), P(C.c_double)]),
    "b2k_block_inner": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(c_vec), C.c_int32, P(C.c_double)]),
    "b2k_block_axpy": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(c_vec), C.c_int32, P(C.c_double),
                                   C.c_int32]),
    "b2k_block_reorthogonalize": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(c_vec), C.c_int32]),
    "b2k_block_qr": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, C.c_double, P(C.c_double),
                                 P(C.c_int32), P(C.c_int32)]),
    "b2k_op_apply_block": (C.c_int32, [c_ctx, c_op, P(c_vec), P(c_vec), C.c_int32]),
    "b2k_block_orthogonalize": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, P(c_vec), C.c_int32, C.c_int32,
                                            P(C.c_double), P(C.c_double)]),
    "b2k_block_cholqr": (C.c_int32, [c_ctx, P(c_vec), C.c_int32, C.c_double, P(C.c_double), P(C.c_double),
                                     P(C.c_int32)]),
    # debugging knob (not part of the public header): 0 = one launch per phase, 1 = cooperative
    "b2k_debug_set_coop": (C.c_int32, [C.c_int32]),
    "b2k_debug_set_spmv_pipe": (C.c_int32, [C.c_int32]),
    "b2k_debug_set_spmv_variant": (C.c_int32, [C.c_int32]),
    "b2k_debug_set_dmma": (C.c_int32, [C.c_int32]),
    "b2k_debug_set_transform": (C.c_int32, [C.c_int32]),
    "b2k_debug_transform_kernel": (C.c_int32, []),
    "b2k_debug_set_chain": (C.c_int32, [C.c_int32]),
    "b2k_debug_used_columns": (C.c_int32, [c_ctx, C.c_int32]),
    "b2k_debug_set_chain_mode": (C.c_int32, [C.c_int32]),
    "b2k_debug_set_onepass_variant": (C.c_int32, [C.c_int32]),
    "b2k_debug_trace": (C.c_int32, [c_ctx, C.c_int32]),
    "b2k_debug_trace_read": (C.c_int32, [c_ctx, P(C.c_uint64), C.c_int64, P(C.c_int64)]),
}

EXPORTED = tuple(k for k in _PROTOS if not k.startswith("b2k_debug"))


def load():
    """Load the shared library (once) and attach prototypes.  Raises LibraryMissing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found. Build it with `python krylovkit.jl_b200/build.py` "
            "(needs nvcc; cross-compiles for sm_90a without a GPU). "
            "This engine has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, ctx=None):
    """Raise the exception matching a status code."""
    if status == OK:
        return
    lib = load()
    msg = lib.b2k_last_error(ctx)
    msg = msg.decode("utf-8", "replace") if msg else ""
    if status == EINVAL:
        raise ValueError(f"b200krylov: {msg}")
    if status == EDIM:
        raise DimensionMismatch(f"b200krylov: {msg}")
    names = {ECUDA: "CUDA", ENOMEM: "out of memory", ENCCL: "NCCL", ENOTSUP: "not supported"}
    raise B200Error(f"b200krylov [{names.get(status, status)}]: {msg}")
