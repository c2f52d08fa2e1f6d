"""OrthonormalBasis on the device slab — mirror of src/orthonormal.jl.

The basis is a Python list of B200Vec (KrylovKit: `Vector{T}` of independently allocated
vectors, orthonormal.jl:26-28); each operation hands the list of slab-column handles to
one C-ABI call, where the panel is streamed by the fused kernels.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .algorithms import Orthogonalizer
from .vectors import B200Vec, handles


class OrthonormalBasis:
    """src/orthonormal.jl:26-54 (length / getindex / push! / pop! / resize! ...)."""

    def __init__(self, vecs=None):
        self.basis: list[B200Vec] = list(vecs) if vecs else []

    def __len__(self):
        return len(self.basis)

    def __iter__(self):
        return iter(self.basis)

    def __getitem__(self, i):
        return self.basis[i]

    def __setitem__(self, i, q):
        self.basis[i] = q

    def push(self, q: B200Vec):
        self.basis.append(q)
        return self

    def pop(self) -> B200Vec:
        return self.basis.pop()

    def popfirst(self) -> B200Vec:
        return self.basis.pop(0)

    def empty_(self):
        self.basis.clear()
        return self

    def resize_(self, k: int):
        del self.basis[k:]
        return self

    @property
    def ctx(self):
        return self.basis[0].ctx

    def __mul__(self, x):
        """b * x — orthonormal.jl:57-60."""
        y = self.basis[0].zerovector()
        return unproject_(y, self, x)


def _dbl(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _cols(b: OrthonormalBasis, r):
    vecs = b.basis if r is None else [b.basis[i] for i in r]
    return vecs, handles(vecs)


def cross_inner(X, Y, skip=(0, 0), G: np.ndarray | None = None) -> np.ndarray:
    """G[i, j] = <X[i], Y[j]> (host float64, column-major p x q) in one device sweep over both lists —
    b2k_basis_cross_inner.  X and Y are sequences of B200Vec (or OrthonormalBasis), at most 256 each.  The leading
    skip = (p0, q0) block of G is neither computed nor written: pass the G of an earlier call to update only the
    rows and columns added since then."""
    X, Y = list(X), list(Y)
    p, q = len(X), len(Y)
    if G is None:
        G = np.zeros((p, q), order="F")
    if G.dtype != np.float64 or not G.flags.f_contiguous or G.shape[0] < p or G.shape[1] < q:
        raise ValueError("cross_inner: G must be a Fortran-ordered float64 array of at least p x q")
    if p == 0 or q == 0:
        return G
    ctx = X[0].ctx
    ctx.check(ctx.lib.b2k_basis_cross_inner(ctx.h, handles(X), p, handles(Y), q, int(skip[0]), int(skip[1]),
                                            G.ctypes.data_as(C.POINTER(C.c_double)), G.shape[0]))
    return G


def project_(y: np.ndarray, b: OrthonormalBasis, x: B200Vec, alpha: float = 1.0, beta: float = 0.0,
             r=None) -> np.ndarray:
    """project!!(y, b, x, α, β, r): y[j] = β y[j] + α <b[r[j]], x> — orthonormal.jl:88-118.
    y is a HOST float64 vector (mutated and returned)."""
    vecs, hs = _cols(b, r)
    if len(y) != len(vecs):
        raise L.DimensionMismatch("project!!: length(y) != length(r)")
    if not vecs:
        return y
    ctx = x.ctx
    if y.dtype != np.float64 or not y.flags.c_contiguous:
        tmp = _dbl(y)
        ctx.check(ctx.lib.b2k_basis_project(ctx.h, hs, len(vecs), x.handle, alpha, beta,
                                            tmp.ctypes.data_as(C.POINTER(C.c_double))))
        y[:] = tmp
        return y
    ctx.check(ctx.lib.b2k_basis_project(ctx.h, hs, len(vecs), x.handle, alpha, beta,
                                        y.ctypes.data_as(C.POINTER(C.c_double))))
    return y


def unproject_(y: B200Vec, b: OrthonormalBasis, x, alpha: float = 1.0, beta: float = 0.0,
               r=None) -> B200Vec:
    """unproject!!(y, b, x, α, β, r): y = β y + α Σ b[r[i]] x[i] — orthonormal.jl:132-196."""
    vecs, hs = _cols(b, r)
    xs = _dbl(x)
    if len(xs) != len(vecs):
        raise L.DimensionMismatch("unproject!!: length(x) != length(r)")
    ctx = y.ctx
    ctx.check(ctx.lib.b2k_basis_unproject(ctx.h, y.handle, hs, len(vecs),
                                          xs.ctypes.data_as(C.POINTER(C.c_double)), alpha, beta))
    return y


def rank1update_(b: OrthonormalBasis, y: B200Vec, x, alpha: float = 1.0, beta: float = 1.0, r=None):
    """rank1update!(b, y, x, α, β, r): b[r[i]] = β b[r[i]] + α y conj(x[i]) — orthonormal.jl:210-275."""
    vecs, hs = _cols(b, r)
    xs = _dbl(x)
    if len(xs) != len(vecs):
        raise L.DimensionMismatch("rank1update!: length(x) != length(r)")
    ctx = y.ctx
    ctx.check(ctx.lib.b2k_basis_rank1update(ctx.h, hs, len(vecs), y.handle,
                                            xs.ctypes.data_as(C.POINTER(C.c_double)), alpha, beta))
    return b


def basistransform_(b: OrthonormalBasis, U: np.ndarray):
    """basistransform!(b, U): b[j] <- Σ_i b[i] U[i,j] — orthonormal.jl:291-354.
    The first size(U,2) basis vectors are overwritten (in place on the device: the row tile
    is resident on chip, so no second set of vectors is allocated as the reference does)."""
    U = np.asfortranarray(U, dtype=np.float64)
    m, n = U.shape
    if m != len(b):
        raise L.DimensionMismatch("basistransform!: size(U,1) != length(b)")
    ctx = b.ctx
    hs = handles(b.basis)
    ctx.check(ctx.lib.b2k_basis_transform(ctx.h, hs, m, U.ctypes.data_as(C.POINTER(C.c_double)),
                                          m, n))
    return b


def rmul_givens_(b: OrthonormalBasis, i1: int, i2: int, c: float, s: float):
    """rmul!(b, G::Givens) — dense/givens.jl:12-36 (0-based i1, i2 here)."""
    ctx = b.ctx
    ctx.check(ctx.lib.b2k_basis_givens(ctx.h, b[i1].handle, b[i2].handle, c, s))
    return b


def rmul_householder_(b: OrthonormalBasis, beta: float, v, r):
    """rmul!(b, H::Householder) — dense/reflector.jl:143-154; r = 0-based index list."""
    if beta == 0.0:
        return b
    vecs, hs = _cols(b, r)
    vs = _dbl(v)
    ctx = b.ctx
    work = ctx.empty(vecs[0].space)
    try:
        ctx.check(ctx.lib.b2k_basis_householder(ctx.h, hs, len(vecs),
                                                vs.ctypes.data_as(C.POINTER(C.c_double)), beta,
                                                work.handle))
    finally:
        work.free()
    return b


def orthogonalize_(v: B200Vec, b, x=None, alg: Orthogonalizer = None):
    """orthogonalize!!(v, b, [x,] alg) -> (v, x)      — orthonormal.jl:372-452
       orthogonalize!!(v, q, alg)      -> (v, s)      — orthonormal.jl:455-489
    `b` is an OrthonormalBasis or a single normalised B200Vec."""
    ctx = v.ctx
    if isinstance(x, Orthogonalizer) and alg is None:
        x, alg = None, x
    if isinstance(b, B200Vec):
        s, nrm = C.c_double(), C.c_double()
        ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, v.handle, b.handle, alg.tag, alg.eta,
                                                C.byref(s), C.byref(nrm)))
        return v, s.value
    k = len(b)
    if x is None:
        x = np.empty(k, dtype=np.float64)
    if len(x) < k:
        raise L.DimensionMismatch("orthogonalize!!: coefficient vector too short")
    h = np.empty(k, dtype=np.float64)
    nrm = C.c_double()
    passes = C.c_int32()
    ctx.check(ctx.lib.b2k_basis_orthogonalize(ctx.h, v.handle, handles(b.basis), k,
                                              h.ctypes.data_as(C.POINTER(C.c_double)), alg.tag,
                                              alg.eta, C.byref(nrm), C.byref(passes)))
    x[:k] = h
    orthogonalize_.last_norm = nrm.value       # ‖v‖ after orthogonalisation, free by-product
    return v, x


orthogonalize_.last_norm = None


def orthonormalize_(v: B200Vec, b, x=None, alg: Orthogonalizer = None):
    """orthonormalize!!(v, b, [x,] alg) -> (v, β, x) — orthonormal.jl:522-527."""
    if isinstance(x, Orthogonalizer) and alg is None:
        x, alg = None, x
    if isinstance(b, B200Vec):
        ctx = v.ctx
        s, nrm = C.c_double(), C.c_double()
        ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, v.handle, b.handle, alg.tag, alg.eta,
                                                C.byref(s), C.byref(nrm)))
        beta = nrm.value
        v.scale_(1.0 / beta)
        return v, beta, s.value
    v, x = orthogonalize_(v, b, x, alg)
    beta = orthogonalize_.last_norm if len(b) > 0 else v.norm()
    v.scale_(1.0 / beta)
    return v, beta, x
