"""svdsolve with Golub-Kahan-Lanczos bidiagonalisation and thick restart — mirror of
src/eigsolve/svdsolve.jl:144-314."""
from __future__ import annotations

import math
import warnings

import ctypes as C

import numpy as np
import scipy.sparse as sp

from ._lib import B200Error
from .algorithms import ConvergenceInfo, GKL, WARN_LEVEL
from .dense import (bidiagsvd_lower, householder_col, householder_row, lmul_householder,
                    rmul_householder)
from .factorizations import gkl
from .operators import B200CSR, B200Dense
from .orthonormal import basistransform_, rmul_householder_
from .vectors import B200Context, B200Vec

_FORMS = ("svdsolve takes a B200CSR (single-GPU context, stored matrix) or a scipy sparse matrix, a dense numpy "
          "matrix or B200Dense, an (A, At) tuple of operators, or a callable f(x, adjoint)")


def svdsolve(A, u0=None, howmany: int = 1, which: str = "LR", alg: GKL | None = None, **kwargs):
    """svdsolve(A, x₀, howmany, which, alg::GKL).  u0 lives in the codomain (length m).
    Host entries: A = numpy or scipy sparse m x n matrix, u0 = numpy vector (or None: random) -> uploaded, solved,
    downloaded.  A B200CSR takes a device u0; its transpose is built on the device for the call."""
    if which not in ("LR", "SR"):
        raise ValueError(f"invalid specification of which singular values to target: which = {which}")
    if alg is None:
        alg = GKL(**kwargs)
    if u0 is None:
        # svdsolve(A::AbstractMatrix, howmany, which; kwargs...) — svdsolve.jl:123-129: random start vector
        if not hasattr(A, "shape"):
            raise TypeError("svdsolve: a start vector is required unless A is a host matrix")
        dt = (A if sp.issparse(A) else np.asarray(A)).dtype
        u0 = np.random.default_rng().random(A.shape[0]).astype(dt if dt == np.float32 else np.float64)
    if isinstance(u0, B200Vec):
        if isinstance(A, B200CSR):
            return _svdsolve_csr(A, u0, howmany, which, alg)
        return _svdsolve_gkl(A, u0, howmany, which, alg)
    if sp.issparse(A):
        return _svdsolve_sparse_host(A, np.asarray(u0), howmany, which, alg)
    A = np.asarray(A)
    u0 = np.asarray(u0)
    m, n = A.shape
    # every converged triple comes back (up to krylovdim of them): U, the left vectors and their residuals
    # live in space 0, V and the right vectors in the short space
    ctx = B200Context(m, 3 * alg.krylovdim + 12, dtype=A.dtype if A.dtype == np.float32 else np.float64)
    try:
        sv = ctx.add_space(n, (3 if getattr(alg, "onepass", False) else 2) * alg.krylovdim + 14, sharded=False)
        op = B200Dense.from_host(ctx, A, sv)
        S, Uv, Vv, info = _svdsolve_gkl(op, ctx.from_host(u0), howmany, which, alg)
        info.residual = [r.to_host() for r in info.residual]
        return S, [u.to_host() for u in Uv], [v.to_host() for v in Vv], info
    finally:
        ctx.close()


def _svdsolve_sparse_host(A, u0: np.ndarray, howmany: int, which: str, alg: GKL):
    """Host sparse entry: one context (space 0 of length m for U, the left vectors and their residuals, a space of
    length n for V and the right vectors), A uploaded once and transposed on the device, numpy results."""
    m, n = A.shape
    dtype = np.float32 if A.dtype == np.float32 else np.float64
    # a chained call holds one U column and one residual more than the step-by-step loop (b2k_gkl_expand_many)
    ctx = B200Context(m, 3 * alg.krylovdim + 14, dtype=dtype)
    try:
        sv = ctx.add_space(n, 2 * alg.krylovdim + 14, sharded=False)
        op = B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        try:
            S, Uv, Vv, info = _svdsolve_csr(op, ctx.from_host(u0.astype(dtype)), howmany, which, alg)
        finally:
            op.free()
        info.residual = [r.to_host() for r in info.residual]
        return S, [u.to_host() for u in Uv], [v.to_host() for v in Vv], info
    finally:
        ctx.close()


def _svdsolve_csr(A: B200CSR, u0: B200Vec, howmany: int, which: str, alg: GKL):
    """svdsolve on a device CSR matrix: A' is built on the device (B200CSR.transpose()) and freed before returning;
    the steps between two restart decisions are chained on the device (gkl.expand_many_)."""
    if u0.ctx.nranks > 1:
        raise B200Error(f"svdsolve: row-sharded contexts are not supported; {_FORMS}")
    nr, nc, nnz, kind = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    u0.ctx.check(u0.ctx.lib.b2k_op_info(A.h, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(kind)))
    if kind.value == 2:
        raise B200Error(f"svdsolve: a matrix-free stencil has no transpose; {_FORMS}")
    if not A._explicit_spaces and A.n_rows != A.n_cols:
        raise ValueError("svdsolve: a rectangular B200CSR must carry its spaces (A.with_spaces(space_in, space_out))")
    At = A.transpose()
    try:
        return _svdsolve_gkl((A, At), u0, howmany, which, alg, pair=(A, At))
    finally:
        At.free()


def _diverged(fact, alg, what: str, k: int | None = None) -> B200Error:
    k = len(fact) if k is None else k
    return B200Error(
        f"GKL bidiagonalisation diverged at step {k} ({what}; alpha = {fact.alphas[k - 1]:.3g}, "
        f"beta = {fact.betas[k - 1]:.3g}): orthogonality of the Krylov bases was lost with orth = {alg.orth}. "
        "With ClassicalGramSchmidt2 the recurrence reorthogonalises the long side only (gkl.jl:308-323), which is "
        "not enough in Float32 on clustered singular values; use an iterative-refinement orthogonalizer "
        "(ClassicalGramSchmidtIR / ModifiedGramSchmidtIR, as the reference's own Float32 tests do, "
        "test/runtests.jl:18) or ModifiedGramSchmidt2.")


def _check_finite(fact, alg, k: int | None = None) -> None:
    """The reference would carry Inf/NaN coefficients into LAPACK (bdsqr) and fail there; fail here, early
    and with the cause, as soon as a coefficient stops being finite or exceeds any possible ||A||.  Checks step k
    (default: the last one)."""
    k = len(fact) if k is None else k
    a, b = fact.alphas[k - 1], fact.betas[k - 1]
    big = 1.0 / np.finfo(np.float32).eps * max(1.0, abs(fact.alphas[0]))      # >> sigma_max ~ alpha_1
    if not (math.isfinite(a) and math.isfinite(b)):
        raise _diverged(fact, alg, "non-finite coefficient", k)
    if abs(a) > big or abs(b) > big:
        raise _diverged(fact, alg, "coefficient far above any singular value of A", k)


def _svdsolve_gkl(A, u0: B200Vec, howmany: int, which: str, alg: GKL, pair=None):
    krylovdim, maxiter = alg.krylovdim, alg.maxiter
    if howmany > krylovdim:
        raise ValueError(f"krylov dimension {krylovdim} too small to compute {howmany} singular values")
    numiter = 1
    onepass = getattr(alg, "onepass", False)
    # a recycled A'u may carry the rounding of at most 4 direct products, or an absolute error of 1 % of the tolerance
    # asked for (eta counts roundings of size eps ||A||: the iterator divides by its running estimate of ||A||)
    eta_tol = 0.01 * alg.tol / float(np.finfo(u0.ctx.np_dtype).eps)
    it = gkl.GKLIterator(A, u0, alg.orth, onepass=onepass, onepass_eta=4.0, onepass_eta_tol=eta_tol, pair=pair)
    fact = gkl.initialize(it)
    numops = 2
    tol = alg.tol
    HH = np.zeros((krylovdim + 1, krylovdim))
    converged = 0
    P = S = Q = f = None
    while True:
        beta = fact.normres()
        K = len(fact)
        if beta <= tol and K < howmany and alg.verbosity >= WARN_LEVEL:
            warnings.warn(f"Invariant subspace of dimension {K} (up to requested tolerance `tol = {tol}`)")
        if K == krylovdim or beta <= tol or (alg.eager and K >= howmany):
            try:
                P, S, Q = bidiagsvd_lower(fact.alphas[:K], fact.betas[:K - 1])
            except np.linalg.LinAlgError as e:       # LAPACK gives up on a bidiagonal that has blown up
                raise _diverged(fact, alg, f"SVD of the {K}x{K} bidiagonal failed: {e}") from e
            if which == "SR":
                P, S, Q = P[:, ::-1].copy(), S[::-1].copy(), Q[::-1, :].copy()
            f = Q.T[K - 1, :] * beta
            converged = 0
            while converged < K and abs(f[converged]) < tol:
                converged += 1
            if converged >= howmany or beta <= tol:
                break
        if K < krylovdim:
            # the run of expansions up to the next restart decision (K == krylovdim or beta <= tol); eager mode
            # decides after every step.  Chained steps are checked in order after the batch, stepped ones as they come.
            d = gkl.expand_many_(it, fact, 1 if alg.eager else krylovdim - K, tol,
                                 check=lambda f: _check_finite(f, alg))
            numops += 2 * d
            for j in range(K + 1, K + d + 1):
                _check_finite(fact, alg, j)
        else:
            if numiter == maxiter:
                break
            keep = (3 * krylovdim + 2 * converged) // 5
            U, V = fact.basis("U"), fact.basis("V")
            basistransform_(U, P[:, :keep])
            basistransform_(V, Q.T[:, :keep])
            G = fact.G                                            # onepass mode: G = A'U rotates with U
            g_lost = False
            if G is not None:
                basistransform_(G, P[:, :keep])
                fact.eta[:] = [max(fact.eta)] * len(fact.eta)     # an orthogonal mix of the columns and their errors
                if fact.g_next is not None:
                    G[keep], fact.g_next = fact.g_next, None      # the image of U[keep] = r/β below
                    fact.eta[keep] = fact.eta_next
                else:
                    g_lost = True
            r = fact.residual()
            U[keep] = U[keep].scale_(1 / fact.normres(), r)       # U[keep+1] = scale!!(r, 1/β)
            H = HH[: keep + 1, :keep]
            H[:] = 0
            for j in range(keep):
                H[j, j] = S[j]
                H[keep, j] = f[j]
            # restore bidiagonal form in the first keep columns — svdsolve.jl:257-268
            for j in range(keep - 1, -1, -1):
                h, nu = householder_row(H, j + 1, range(0, j + 1), j)
                H[j + 1, j] = nu
                H[j + 1, :j] = 0
                rmul_householder(H, h, slice(0, j + 1))
                rmul_householder_(V, h.beta, h.v, h.r)
                h, nu = householder_col(H, range(0, j + 1), j, j)
                H[j, j] = nu
                H[:j, j] = 0
                lmul_householder(h, H, range(0, j))
                rmul_householder_(U, h.beta, h.v, h.r)
                if G is not None:
                    rmul_householder_(G, h.beta, h.v, h.r)
            for j in range(keep):
                fact.alphas[j] = H[j, j]
                fact.betas[j] = H[j + 1, j]
            fact = gkl.shrink_(fact, keep)
            if g_lost:
                fact.g_next = None                                # the next step forms A'u directly
            numiter += 1
    if converged > howmany:
        howmany = converged
    values = S[:howmany].copy()
    U, V = fact.basis("U"), fact.basis("V")
    left = [U * P[:, i] for i in range(howmany)]
    right = [V * Q[i, :] for i in range(howmany)]
    r = fact.residual()
    residuals = [r.scale(Q[i, -1]) for i in range(howmany)]
    normres = np.abs(f[:howmany])
    if converged < howmany and alg.verbosity >= WARN_LEVEL:
        warnings.warn(f"GKL svdsolve finished without convergence after {numiter} iterations: "
                      f"{converged} singular values converged, normres = {normres}, numops = {numops}")
    info = ConvergenceInfo(converged, residuals, normres, numiter, numops)
    info.passes = fact.passes             # passes over A (numops counts products, as the reference does)
    return values, left, right, info
