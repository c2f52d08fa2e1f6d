"""Device-resident linear operators and KrylovKit's `apply` contract (src/apply.jl).

apply(A, x)            -> A*x            (apply.jl:1)
apply(A, x, a0, a1)    -> a1*A*x + a0*x  (apply.jl:4-11)
apply_normal / apply_adjoint            (apply.jl:14-19)

`apply` never mutates x and returns a NEW vector, exactly like the reference.
"""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np

from . import _lib as L
from .vectors import B200Context, B200Vec


class B200Operator:
    kind = "abstract"

    def __init__(self, ctx: B200Context, h):
        self.ctx = ctx
        self.h = h
        self._fin = weakref.finalize(self, _destroy_op, ctx.lib, ctx.h, h, ctx._alive)
        nr, nc, nnz, kind = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
        ctx.lib.b2k_op_info(h, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(kind))
        self.n_rows, self.n_cols, self.nnz = nr.value, nc.value, nnz.value
        self.space_in = 0     # space of x in y = A x
        self.space_out = 0
        self._explicit_spaces = False

    def free(self):
        self._fin()

    def with_spaces(self, space_in: int, space_out: int):
        """Rectangular operators: name the vector spaces of x and y in y = A x."""
        self.space_in, self.space_out = space_in, space_out
        self._explicit_spaces = True
        return self

    # y = A x into an existing vector (y must not alias x)
    def apply_into(self, y: B200Vec, x: B200Vec) -> B200Vec:
        self.ctx.check(self.ctx.lib.b2k_op_apply(self.ctx.h, self.h, x.handle, y.handle))
        return y

    def apply_dot_into(self, y: B200Vec, x: B200Vec, v: B200Vec) -> float:
        """y = A x and <v, y> in the same pass."""
        out = C.c_double()
        self.ctx.check(self.ctx.lib.b2k_op_apply_dot(self.ctx.h, self.h, x.handle, y.handle,
                                                     v.handle, C.byref(out)))
        return out.value

    def __call__(self, x: B200Vec) -> B200Vec:
        return apply(self, x)


def _destroy_op(lib, ctx_h, op_h, alive):
    if alive[0]:
        lib.b2k_op_destroy(ctx_h, op_h)


class B200CSR(B200Operator):
    """CSR sparse matrix in HBM (int32 indices).  Build from scipy.sparse, from Julia's
    SparseMatrixCSC arrays (colptr, rowval, nzval; 1-based Int64) or as a stencil."""

    kind = "csr"

    @classmethod
    def from_scipy(cls, ctx: B200Context, A) -> "B200CSR":
        A = A.tocsr()                      # the caller's own matrix when it is CSR already: never sorted in place
        if not A.has_sorted_indices:
            A = A.sorted_indices()
        n_rows, n_cols = A.shape
        rp = np.ascontiguousarray(A.indptr, dtype=np.int64)
        ci = np.ascontiguousarray(A.indices, dtype=np.int64)
        va = np.ascontiguousarray(A.data, dtype=ctx.np_dtype)
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_csr(ctx.h, C.byref(h), n_rows, n_cols, A.nnz, rp.ctypes.data,
                                            ci.ctypes.data, va.ctypes.data, 8, 0))
        return cls(ctx, h)

    @classmethod
    def from_csr_arrays(cls, ctx: B200Context, n_rows, n_cols, rowptr, colidx, vals,
                        index_base: int = 0) -> "B200CSR":
        rp = np.ascontiguousarray(rowptr)      # no copy when already contiguous (pinned buffers stay pinned)
        ci = np.ascontiguousarray(colidx)
        if rp.dtype != ci.dtype or rp.dtype not in (np.int32, np.int64):
            rp, ci = rp.astype(np.int64), ci.astype(np.int64)
        va = np.ascontiguousarray(vals, dtype=ctx.np_dtype)
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_csr(ctx.h, C.byref(h), n_rows, n_cols, len(va), rp.ctypes.data,
                                            ci.ctypes.data, va.ctypes.data, rp.dtype.itemsize,
                                            index_base))
        return cls(ctx, h)

    @classmethod
    def from_julia_csc(cls, ctx: B200Context, m, n, colptr, rowval, nzval) -> "B200CSR":
        """SparseMatrixCSC fields as Julia stores them (1-based Int64).  nnz is colptr[n] - 1, as Julia's `nnz`:
        rowval and nzval may carry spare capacity past it."""
        cp = np.ascontiguousarray(colptr, dtype=np.int64)
        rv = np.ascontiguousarray(rowval, dtype=np.int64)
        nz = np.ascontiguousarray(nzval, dtype=ctx.np_dtype)
        if n < 0 or len(cp) != n + 1:
            raise L.B200Error(f"from_julia_csc: colptr has {len(cp)} entries, {n} columns need {n + 1}")
        nnz = int(cp[-1]) - 1
        if len(rv) < nnz or len(nz) < nnz:
            raise L.B200Error(f"from_julia_csc: colptr holds {nnz} entries, rowval {len(rv)} and nzval {len(nz)}")
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_csc(ctx.h, C.byref(h), m, n, nnz, cp.ctypes.data,
                                            rv.ctypes.data, nz.ctypes.data, 8, 1))
        return cls(ctx, h)

    @classmethod
    def stencil(cls, ctx: B200Context, nx: int, ny: int, nz: int = 1,
                coeffs=(4.0, -1.0, -1.0, -1.0, -1.0, -1.0, -1.0)) -> "B200CSR":
        """Dirichlet stencil assembled on the device as a real CSR matrix.
        coeffs = (centre, west, east, south, north, down, up)."""
        c = (C.c_double * 7)(*[float(v) for v in coeffs])
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_stencil(ctx.h, C.byref(h), nx, ny, nz, c))
        return cls(ctx, h)

    @classmethod
    def stencil_free(cls, ctx: B200Context, nx: int, ny: int, nz: int = 1,
                     coeffs=(4.0, -1.0, -1.0, -1.0, -1.0, -1.0, -1.0)) -> "B200CSR":
        """The same Dirichlet stencil, MATRIX-FREE: nothing is stored, every apply evaluates the stencil from the
        vector (16 n bytes per apply instead of 12 nnz + 20 n) with the assembled operator's rounding — results are
        bit-identical to `stencil(...)`.  KrylovKit takes any function as its linear map; this is the device form of
        such a function for the grids of the BASELINE configs.  (`to_scipy` is not available.)"""
        c = (C.c_double * 7)(*[float(v) for v in coeffs])
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_stencil_free(ctx.h, C.byref(h), nx, ny, nz, c))
        return cls(ctx, h)

    def transpose(self) -> "B200CSR":
        """A' as a new device CSR operator, built on the device (b2k_op_create_transpose): the arrays of scipy's
        sorted A.T.tocsr(), so products with it are bit-identical to those with the host-built transpose.  Spaces
        given explicitly to A are swapped.  Not for matrix-free stencils or row-sharded contexts."""
        h = L.c_op()
        self.ctx.check(self.ctx.lib.b2k_op_create_transpose(self.ctx.h, C.byref(h), self.h))
        t = B200CSR(self.ctx, h)
        if self._explicit_spaces:
            t.with_spaces(self.space_out, self.space_in)
        return t

    def to_scipy(self):
        import scipy.sparse as sp
        rp = np.empty(self.n_rows + 1, dtype=np.int32)
        ci = np.empty(self.nnz, dtype=np.int32)
        va = np.empty(self.nnz, dtype=self.ctx.np_dtype)
        self.ctx.check(self.ctx.lib.b2k_op_csr_download(self.ctx.h, self.h, rp.ctypes.data,
                                                        ci.ctypes.data, va.ctypes.data))
        return sp.csr_matrix((va, ci, rp), shape=(self.n_rows, max(self.n_cols, int(ci.max(initial=0)) + 1)))


class B200Dense(B200Operator):
    """Dense column-major m x n matrix (rows sharded in dist mode).  x lives in
    `space_in` (length n, replicated), y in space 0 (length m)."""

    kind = "dense"

    @classmethod
    def from_host(cls, ctx: B200Context, A, space_in: int) -> "B200Dense":
        A = np.asfortranarray(A, dtype=ctx.np_dtype)
        m, n = A.shape
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_dense(ctx.h, C.byref(h), m, n, A.ctypes.data, m))
        op = cls(ctx, h)
        op.space_in, op.space_out = space_in, 0
        return op

    @classmethod
    def splitmix(cls, ctx: B200Context, m_local: int, n: int, seed: int, space_in: int) -> "B200Dense":
        h = L.c_op()
        ctx.check(ctx.lib.b2k_op_create_dense_splitmix(ctx.h, C.byref(h), m_local, n, seed))
        op = cls(ctx, h)
        op.space_in, op.space_out = space_in, 0
        return op

    def apply_adjoint_into(self, y: B200Vec, x: B200Vec) -> B200Vec:
        self.ctx.check(self.ctx.lib.b2k_op_apply_adjoint(self.ctx.h, self.h, x.handle, y.handle))
        return y


# ------------------------------------------------------------------ apply contract ----

def apply(op, x: B200Vec, a0: float = 0.0, a1: float = 1.0) -> B200Vec:
    """apply(operator, x[, α₀, α₁]) — src/apply.jl:1-11.  `op` is a B200Operator or any
    callable x -> y on B200Vec (the abstract-linear-map contract)."""
    if isinstance(op, B200Operator):
        # the result lives in the operator's output space when it has one of its own (dense operators, CSR
        # operators given spaces explicitly — also square ones, e.g. the (A, Aᵀ) pair of lssolve), else next to x
        own_space = isinstance(op, B200Dense) or op._explicit_spaces or op.n_rows != op.n_cols
        y = x.ctx.empty(op.space_out if own_space else x.space)
        if a0 != 0.0 or a1 != 1.0:
            x.ctx.check(x.ctx.lib.b2k_op_apply_shifted(x.ctx.h, op.h, x.handle, y.handle,
                                                       float(a0), float(a1)))
        else:
            op.apply_into(y, x)
        return y
    y = op(x)
    if a0 != 0.0 or a1 != 1.0:
        y = y.add_(x, a0, a1)
    return y


class B200Pencil:
    """The pencil (A, B) of a generalized eigenproblem A x = λ B x (geneigsolve): b2k_pencil_*.  A and B are square
    device operators of one context and one size; the pencil holds references to both.  Same-pattern CSR pairs (an
    assembled stencil pair, a stiffness / mass pair of one mesh) are applied by one fused pass over both matrices,
    every other pair by the composition of separate applies; both give the same bits for the vectors.  Calling the
    pencil on x returns (A x, B x): KrylovKit's `genapply(f, x) = f(x)` (apply.jl:23)."""

    def __init__(self, A: B200Operator, B: B200Operator):
        if A.ctx is not B.ctx:
            raise ValueError("B200Pencil: A and B must belong to one context")
        ctx = A.ctx
        h = C.c_void_p()
        ctx.check(ctx.lib.b2k_pencil_create(ctx.h, C.byref(h), A.h, B.h))
        self.ctx, self.A, self.B, self.h = ctx, A, B, h
        self._fin = weakref.finalize(self, _destroy_pencil, ctx.lib, ctx.h, h, ctx._alive)

    def free(self):
        self._fin()

    def apply_into(self, x: B200Vec, w: B200Vec, bx: B200Vec, rho: float, vprev: B200Vec | None = None,
                   beta: float = 0.0, dot: bool = False):
        """bx = B x, w = add!!(A x, bx, -ρ) [then add!!(w, vprev, -β)] — golubye.jl:198-202; returns <x, w> when `dot`
        (b2k_pencil_apply)."""
        out = C.c_double()
        self.ctx.check(self.ctx.lib.b2k_pencil_apply(self.ctx.h, self.h, x.handle, w.handle, bx.handle, float(rho),
                                                     -1 if vprev is None else vprev.handle, float(beta),
                                                     C.byref(out) if dot else None))
        return out.value if dot else None

    def rayleigh_into(self, x: B200Vec, ax: B200Vec, bx: B200Vec, dots: bool = True):
        """ax = A x, bx = B x and, when `dots`, (<x, ax>, <x, bx>) from the same pass (b2k_pencil_rayleigh)."""
        a, b = C.c_double(), C.c_double()
        self.ctx.check(self.ctx.lib.b2k_pencil_rayleigh(self.ctx.h, self.h, x.handle, ax.handle, bx.handle,
                                                        C.byref(a) if dots else None, C.byref(b) if dots else None))
        return (a.value, b.value) if dots else None

    def __call__(self, x: B200Vec):
        ax, bx = x.ctx.empty(x.space), x.ctx.empty(x.space)
        self.rayleigh_into(x, ax, bx, dots=False)
        return ax, bx


def _destroy_pencil(lib, ctx_h, h, alive):
    if alive[0]:
        lib.b2k_pencil_destroy(ctx_h, h)


def genapply(f, x: B200Vec):
    """genapply — src/apply.jl:22-23: (apply(A, x), apply(B, x)) for a tuple (A, B) of operators or callables,
    f(x) -> (A x, B x) for a callable; a B200Pencil forms both products in one call."""
    if isinstance(f, tuple):
        return apply(f[0], x), apply(f[1], x)
    return f(x)


def apply_normal(op, x: B200Vec) -> B200Vec:
    """apply_normal — src/apply.jl:14,16,18."""
    if isinstance(op, B200Operator):
        return apply(op, x)
    if isinstance(op, tuple):
        return op[0](x)
    return op(x, False)


def apply_normal_gram(op: "B200Dense", x: B200Vec):
    """(A x, A'(A x)) from ONE pass over a dense device operator — b2k_op_apply_normal_gram; the flagged
    one-pass mode of the GKL step (factorizations/gkl.py).  Not a reference function."""
    if not isinstance(op, B200Dense):
        raise L.B200Error("apply_normal_gram: dense device operators only")
    y = x.ctx.empty(op.space_out)
    z = x.ctx.empty(op.space_in)
    x.ctx.check(x.ctx.lib.b2k_op_apply_normal_gram(x.ctx.h, op.h, x.handle, y.handle, z.handle))
    return y, z


def apply_adjoint(op, x: B200Vec) -> B200Vec:
    """apply_adjoint — src/apply.jl:15,17,19."""
    if isinstance(op, B200Dense):
        y = x.ctx.empty(op.space_in)
        return op.apply_adjoint_into(y, x)
    if isinstance(op, B200CSR):
        raise L.B200Error("apply_adjoint on B200CSR: pass (A, At) as a tuple of operators")
    if isinstance(op, tuple):
        return op[1](x)
    return op(x, True)
