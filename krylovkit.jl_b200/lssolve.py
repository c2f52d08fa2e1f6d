"""lssolve with LSMR — mirror of src/lssolve/lsmr.jl (front end: src/lssolve/lssolve.jl).

min_x ‖b − A x‖² + λ²‖x‖² by Golub-Kahan bidiagonalisation; every vector operation is a
VectorInterface call on device vectors, the scalar rotations stay on the host.  The operator is
anything `apply_normal` / `apply_adjoint` accept: a B200Dense, a pair (A, Aᵀ) of B200CSR
operators (rectangular ones carry `space_in` / `space_out`), or a callable f(x, flag).

A B200CSR itself is accepted too: Aᵀ is built on the device for the call, and on one GPU the
iterations are chained on the device (b2k_lsmr_chain, LSMR_CHAIN_LEN per host round trip) when
the reorthogonalisation can be: krylovdim <= 1, or MGS, MGS2, CGS2 or the flagged MGS2B.
"""
from __future__ import annotations

import ctypes as C
import math
import warnings

import numpy as np

from . import _lib as L
from ._lib import B200Error
from .algorithms import ConvergenceInfo, LSMR, WARN_LEVEL
from .operators import B200CSR, B200Dense, apply_adjoint, apply_normal
from .orthonormal import OrthonormalBasis, orthogonalize_
from .vectors import B200Context, B200Vec, handles

USE_LSMR_CHAIN = True    # b2k_lsmr_chain: four launches per iteration (+ the reorthogonalisation), one round trip
LSMR_CHAIN_LEN = 32      # per LSMR_CHAIN_LEN iterations
_FORMS = ("lssolve takes a B200CSR (single-GPU context, stored matrix) or a scipy sparse matrix, a dense numpy "
          "matrix or B200Dense, an (A, At) tuple of operators, or a callable f(x, adjoint)")


def lssolve(A, b, alg: LSMR | None = None, lam: float = 0.0, atol: float | None = None,
            rtol: float | None = None, **kwargs):
    """lssolve(A, b, alg::LSMR, λ).  Host entry: A = numpy m×n array or scipy sparse matrix and
    b = numpy vector -> uploaded, solved, downloaded.  tol = max(atol, rtol*‖Aᴴb‖) when atol/rtol
    are given (lssolve.jl:118-124)."""
    if alg is None:
        alg = LSMR(**kwargs)
    if isinstance(b, B200Vec):
        if isinstance(A, B200CSR):
            return _lssolve_csr(A, b, alg, lam, atol, rtol)
        if atol is not None or rtol is not None:
            alg = _retol(alg, max(atol or 0.0, (rtol or 0.0) * apply_adjoint(A, b).norm()))
        return _lsmr(A, b, alg, lam)
    import scipy.sparse as sp
    b = np.asarray(b)
    m, n = A.shape
    dtype = np.float32 if b.dtype == np.float32 else np.float64
    ctx = B200Context(m, 12, dtype=dtype)
    try:
        sv = ctx.add_space(n, alg.krylovdim + 10, sharded=False)
        if sp.issparse(A):
            op = (B200CSR.from_scipy(ctx, A).with_spaces(sv, 0),
                  B200CSR.from_scipy(ctx, A.T.tocsr()).with_spaces(0, sv))
        else:
            op = B200Dense.from_host(ctx, np.asarray(A), sv)
        x, info = lssolve(op, ctx.from_host(b), alg, lam, atol, rtol)
        info.residual = info.residual.to_host()
        return x.to_host(), info
    finally:
        ctx.close()


def _lssolve_csr(A: B200CSR, b: B200Vec, alg: LSMR, lam: float, atol, rtol):
    """lssolve on a device CSR matrix: Aᵀ is built on the device (B200CSR.transpose()) and freed before returning."""
    ctx = b.ctx
    if ctx.nranks > 1:
        raise B200Error(f"lssolve: row-sharded contexts are not supported; {_FORMS}")
    nr, nc, nnz, kind = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    ctx.check(ctx.lib.b2k_op_info(A.h, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(kind)))
    if kind.value == 2:
        raise B200Error(f"lssolve: a matrix-free stencil has no transpose; {_FORMS}")
    if kind.value != 0:
        raise B200Error(f"lssolve: the operator is not a stored CSR matrix; {_FORMS}")
    if not A._explicit_spaces and A.n_rows != A.n_cols:
        raise ValueError("lssolve: a rectangular B200CSR must carry its spaces (A.with_spaces(space_in, space_out))")
    At = A.transpose()
    try:
        op = (A, At)
        if atol is not None or rtol is not None:
            alg = _retol(alg, max(atol or 0.0, (rtol or 0.0) * apply_adjoint(op, b).norm()))
        K = alg.krylovdim
        # the library refuses what it cannot chain (B2K_ENOTSUP, nothing written): the loop then runs literally
        chain = USE_LSMR_CHAIN and (K <= 1 or alg.orth.tag in (L.MGS, L.MGS2, L.CGS2, L.MGS2B))
        return _lsmr(op, b, alg, lam, chain=chain)
    finally:
        At.free()


def _retol(alg: LSMR, tol: float) -> LSMR:
    return LSMR(orth=alg.orth, maxiter=alg.maxiter, krylovdim=alg.krylovdim, tol=tol, verbosity=alg.verbosity)


def _lsmr(operator, b: B200Vec, alg: LSMR, lam: float, chain: bool = False):
    """lssolve(operator, b, alg::LSMR, λ) — lsmr.jl:1-162.  chain (operator = (A, Aᵀ) of stored CSR matrices on
    one GPU): the iterations run LSMR_CHAIN_LEN at a time in b2k_lsmr_chain, and a beta or alpha breakdown hands
    the state back to the loop below, which completes the solve as the reference does."""
    u = b.copy()
    v = apply_adjoint(operator, b)
    beta = u.norm()
    u = u.scale_(1 / beta)
    v = v.scale_(1 / beta)
    alpha = v.norm()
    v = v.scale_(1 / alpha)

    V = OrthonormalBasis([v])
    K = alg.krylovdim
    Vv = np.zeros(K)                       # storage for the reorthogonalisation coefficients

    alphabar, zetabar = alpha, alpha * beta
    rho, theta, rhobar, cbar, sbar = 1.0, 0.0, 1.0, 1.0, 0.0
    abszetabar = abs(zetabar)

    x = v.zerovector()
    h = v.copy()                           # a copy: v itself sits in the ring and gets replaced
    hbar = v.zerovector()
    r = u.scale(beta)
    Ah = u.zerovector()
    Ahbar = u.zerovector()

    numiter, numops = 0, 1
    maxiter, tol = alg.maxiter, alg.tol
    if abszetabar < tol:
        return x, ConvergenceInfo(1, r, abszetabar, numiter, numops)

    if chain:
        ctx = b.ctx
        R = max(K, 1)
        ring = [v] + [ctx.empty(v.space) for _ in range(R - 1)]
        spare, Av = ctx.empty(v.space), ctx.empty(u.space)
        ring_h = handles(ring)
        state = (C.c_double * 10)()
        state_out = (C.c_double * 10)()
        rec = np.zeros((LSMR_CHAIN_LEN, 16))
        done = C.c_int32()
        while True:
            nsteps = max(1, min(LSMR_CHAIN_LEN, maxiter - numiter))
            state[:] = [alpha, beta, alphabar, rho, rhobar, cbar, sbar, theta, zetabar, lam]
            status = ctx.lib.b2k_lsmr_chain(
                ctx.h, operator[0].h, operator[1].h, x.handle, h.handle, hbar.handle, r.handle, Ah.handle,
                Ahbar.handle, u.handle, Av.handle, ring_h, K, spare.handle, alg.orth.tag, numiter, state, tol,
                nsteps, rec.ctypes.data_as(C.POINTER(C.c_double)), state_out, C.byref(done))
            if status == L.ENOTSUP and numiter == 0:
                # e.g. more ring columns than the cooperative sweep holds, or that sweep switched off
                V = OrthonormalBasis([v])
                del ring, spare, Av
                break
            ctx.check(status)
            d = done.value
            numiter += d
            numops += d + int(rec[:d, 8].sum())
            alpha, beta, alphabar, rho, rhobar, cbar, sbar, theta, zetabar = list(state_out)[:9]
            abszetabar = rec[d - 1, 6]
            code = int(rec[d - 1, 7])
            if code == 1:
                return x, ConvergenceInfo(1, r, abszetabar, numiter, numops)
            if code == 0 and numiter < maxiter:
                continue
            # hand the loop's state to the literal iterations below (include/b200krylov.h: where v is)
            if code == 2:
                v = ring[(numiter - 1) % R]
                V = OrthonormalBasis(ring[:min(K, numiter)] if K > 1 else ring[:1])
            elif code == 3:
                v = spare
                V = OrthonormalBasis(ring[:min(K, numiter)] if K > 1 else ring[:1])
            else:
                v = ring[numiter % R]
                V = OrthonormalBasis(ring[:min(K, numiter + 1)] if K > 1 else ring[:1])
            del ring, spare, Av
            if numiter >= maxiter:
                if alg.verbosity >= WARN_LEVEL:
                    warnings.warn(f"LSMR lssolve stopped without converging after {numiter} iterations: "
                                  f"normres = {abszetabar}, numops = {numops}")
                return x, ConvergenceInfo(0, r, abszetabar, numiter, numops)
            break

    while True:
        numiter += 1
        Av = apply_normal(operator, v)
        numops += 1
        Ah = Ah.add_(Av, 1.0, -theta / rho)

        # β₊ u₊ = A v − α u
        u = Av.add_(u, -alpha)
        del Av
        beta = u.norm()
        if beta > tol:
            u = u.scale_(1 / beta)
            # α₊ v₊ = Aᴴ u₊ − β₊ v
            v = apply_adjoint(operator, u).add_(v, -beta)
            numops += 1
            if K > 1:                      # reorthogonalise against the ring, in slot order
                v, _ = orthogonalize_(v, V, Vv[:min(K, numiter)], alg.orth)
            alpha = v.norm()
            if alpha > tol:
                v = v.scale_(1 / alpha)
                if numiter < K:
                    V.push(v)
                else:
                    V[numiter % K] = v     # mod1(numiter + 1, K) in 1-based terms

        # rotation P̂ (folds the regularisation λ into ᾱ)
        alphahat = math.hypot(alphabar, lam)
        # rotation P: B → R
        rhoold = rho
        rho = math.hypot(alphahat, beta)
        c, s = alphahat / rho, beta / rho
        theta = s * alpha
        alphabar = c * alpha
        # rotation P̄: Rᵀ → R̄
        rhobarold = rhobar
        thetabar = sbar * rho
        cbarrho = cbar * rho
        rhobar = math.hypot(cbarrho, theta)
        cbar = cbarrho / rhobar
        sbar = theta / rhobar
        zeta = cbar * zetabar
        zetabar = -sbar * zetabar

        g = -thetabar * rho / (rhoold * rhobarold)
        hbar = hbar.add_(h, 1.0, g)        # h̄ ← h + g h̄
        Ahbar = Ahbar.add_(Ah, 1.0, g)
        x = x.add_(hbar, zeta / (rho * rhobar))
        r = r.add_(Ahbar, -zeta / (rho * rhobar))
        h = h.add_(v, 1.0, -theta / rho)   # Ah catches up at the top of the next iteration

        abszetabar = abs(zetabar)
        if abszetabar <= tol:
            return x, ConvergenceInfo(1, r, abszetabar, numiter, numops)
        if numiter >= maxiter:
            if alg.verbosity >= WARN_LEVEL:
                warnings.warn(f"LSMR lssolve stopped without converging after {numiter} iterations: "
                              f"normres = {abszetabar}, numops = {numops}")
            return x, ConvergenceInfo(0, r, abszetabar, numiter, numops)
