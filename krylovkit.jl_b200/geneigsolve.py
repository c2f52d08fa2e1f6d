"""geneigsolve with the Golub-Ye algorithm — mirror of src/eigsolve/geneigsolve.jl and src/eigsolve/golubye.jl.

A x = λ B x with A symmetric and B symmetric positive definite, without ever inverting B: a Lanczos process on
A - ρ B around the current Rayleigh quotient ρ, restarted from the best Ritz vector and extended by the previous
iterate's direction (the LOPCG correction of Money and Ye).  All n-length work runs on the device: the products, one
per step, through a pencil (B200Pencil: one fused pass over both matrices when their patterns are equal); the
three-term recurrence and its reorthogonalisation; the border of the projected A at a process step (one
b2k_basis_project call); the projected B (one b2k_basis_cross_inner call); the Ritz vectors (b2k_basis_unproject).
The projected pencil is solved on the host with LAPACK's sygvd, the routine of the reference's geneigh!.
"""
from __future__ import annotations

import math
import warnings

import numpy as np
import scipy.linalg

from . import _lib as L
from .algorithms import ConvergenceInfo, GolubYe, WARN_LEVEL, cgs, mgs
from .dense import eigsort
from .operators import B200CSR, B200Operator, B200Pencil, genapply
from .orthonormal import OrthonormalBasis, cross_inner, orthogonalize_, orthonormalize_, project_, unproject_
from .vectors import B200Context, B200Vec

_SELECTOR_ERROR = ("Only symmetric or hermitian generalized eigenvalue problems with positive definite `B` matrix are "
                   "currently supported.")
MAX_HB_COLUMNS = 256        # the widest column lists b2k_basis_cross_inner takes


def geneigsolve(AB, x0=None, howmany: int = 1, which="LM", alg: GolubYe | None = None, device: int = 0, **kwargs):
    """geneigsolve(AB, x₀, howmany, which, alg::GolubYe) — eigsolve/geneigsolve.jl:148-196, golubye.jl:1-194.

    AB is one of
      * a B200Pencil;
      * a tuple (A, B) of two B200CSR: a pencil is made of them and freed before returning;
      * a tuple (A, B) of other device operators or callables on B200Vec, or a callable f(x) -> (A x, B x): the
        products are formed separately (genapply, apply.jl:22-23);
      * a tuple (A, B) of scipy sparse matrices or numpy arrays on the host: x₀ is then a host array (drawn uniformly
        from [0, 1) when omitted), A and B are uploaded once, and the vectors come back as numpy arrays.
    The device forms take a B200Vec x₀.  Keyword arguments (krylovdim, maxiter, tol, orth, verbosity and the
    selector's issymmetric, ishermitian, isposdef) choose the algorithm as geneigselector does; device operators and
    callables must be declared `ishermitian=True, isposdef=True`, as Julia functions must.
    Scalars (ρ, α, β, the projected matrices) are float64 on the host for Float32 vectors as well, as in the Lanczos
    driver; a Float32 kernel rounds a coefficient to Float32 where it uses it.
    Returns (values, vectors, ConvergenceInfo).
    """
    if alg is None:
        alg = geneigselector(AB, **kwargs)
    elif kwargs:
        raise TypeError(f"geneigsolve: keyword arguments {sorted(kwargs)} only apply when no algorithm is passed")
    if which in ("LI", "SI"):                    # geneigsolve.jl:192-194
        raise ValueError(f"Eigenvalue selector which = {which} invalid: real eigenvalues expected with Lanczos "
                         "algorithm")
    eigsort(which)                               # an unknown selector fails before any work
    if _is_host_pair(AB):
        return _geneigsolve_host(AB, x0, howmany, which, alg, device)
    if not isinstance(x0, B200Vec):
        raise TypeError("geneigsolve: device operators need a device start vector x0 (B200Vec)")
    if x0.ctx.nranks > 1:
        raise L.B200Error("geneigsolve: row-sharded contexts are not supported")
    own = None
    if isinstance(AB, B200Pencil):
        f = AB
    elif isinstance(AB, tuple) and len(AB) == 2:
        if all(isinstance(M, B200CSR) for M in AB):
            f = own = B200Pencil(*AB)
        else:
            f = AB
    elif callable(AB) and not isinstance(AB, B200Operator):
        f = AB
    else:
        raise TypeError(f"geneigsolve: unsupported linear map {type(AB).__name__}")
    try:
        return geneigsolve_golubye(f, x0, howmany, which, alg)
    finally:
        if own is not None:
            own.free()


def _is_host_matrix(M) -> bool:
    import scipy.sparse as sp
    return sp.issparse(M) or (isinstance(M, np.ndarray) and M.ndim == 2)


def _is_host_pair(AB) -> bool:
    return isinstance(AB, tuple) and len(AB) == 2 and all(_is_host_matrix(M) for M in AB)


def _host_isposdef(B) -> bool:
    """LinearAlgebra.isposdef(B) for a symmetric host matrix.  A numpy array takes a dense Cholesky factorization.  A
    sparse B takes the sufficient Gershgorin test (positive diagonal, strictly diagonally dominant) where Julia runs
    CHOLMOD; a B that fails it is not declared indefinite, the caller is asked to state isposdef=True instead."""
    import scipy.sparse as sp
    if sp.issparse(B):
        B = sp.csr_matrix(B)
        d = B.diagonal()
        off = np.asarray(abs(B).sum(axis=1)).ravel() - np.abs(d)
        if np.all(d > 0) and np.all(d > off):
            return True
        raise ValueError("geneigsolve: positive definiteness of a sparse B is only certified here when B has a positive "
                         "diagonal and is strictly diagonally dominant; this B is not, so pass isposdef=True if it "
                         "is positive definite")
    try:
        np.linalg.cholesky(B)
    except np.linalg.LinAlgError:
        return False
    return True


def geneigselector(AB, issymmetric: bool | None = None, ishermitian: bool | None = None,
                   isposdef: bool | None = None, **kwargs) -> GolubYe:
    """geneigselector — eigsolve/geneigsolve.jl:198-223.  Host matrices are tested (symmetry as eigselector does,
    B's definiteness by _host_isposdef); device operators and callables default to issymmetric = ishermitian =
    isposdef = false, like a Julia function.  Real scalars: ishermitian defaults to issymmetric."""
    from .eigsolve import _host_issymmetric
    if _is_host_pair(AB):
        if issymmetric is None:
            issymmetric = all(_host_issymmetric(M) for M in AB)
        if ishermitian is None:
            ishermitian = issymmetric
        if isposdef is None:
            isposdef = bool(ishermitian) and _host_isposdef(AB[1])
    else:
        issymmetric = bool(issymmetric)
        ishermitian = issymmetric if ishermitian is None else bool(ishermitian)
        isposdef = bool(isposdef)
    if (issymmetric or ishermitian) and isposdef:
        return GolubYe(**kwargs)
    raise ValueError(_SELECTOR_ERROR)


def _geneigsolve_host(AB, x0, howmany, which, alg, device=0):
    """Host-matrix entry: upload A and B once, solve on a pencil, download the vectors and residuals.  The slab holds
    the most the reference keeps alive at once: V and BV (up to krylovdim + 1 columns each in a process step), the
    Ritz vectors and residuals of a process step (up to as many), r, vold and one work vector."""
    import scipy.sparse as sp
    A, B = AB
    n = A.shape[0]
    if not (A.shape == (n, n) and B.shape == (n, n)):
        raise L.DimensionMismatch("Matrices `A` and `B` should be square and have matching size")
    if x0 is None:
        dtype = np.float32 if (A.dtype == np.float32 and B.dtype == np.float32) else np.float64
        x0 = np.random.default_rng().random(n).astype(dtype)
    x0 = np.asarray(x0)
    dtype = np.float32 if x0.dtype == np.float32 else np.float64
    ctx = B200Context(n, 4 * (alg.krylovdim + 1) + 3, dtype=dtype, device=device)
    try:
        P = B200Pencil(B200CSR.from_scipy(ctx, sp.csr_matrix(A)), B200CSR.from_scipy(ctx, sp.csr_matrix(B)))
        try:
            values, vectors, info = geneigsolve_golubye(P, ctx.from_host(x0.astype(dtype)), howmany, which, alg)
            vecs_h = [v.to_host() for v in vectors]
            res_h = [r.to_host() for r in info.residual]
            return values, vecs_h, ConvergenceInfo(info.converged, res_h, info.normres, info.numiter, info.numops)
        finally:
            P.free()
    finally:
        ctx.close()


# ---------------------------------------------------------------- golubye.jl ----

def _checkhermitian(z, n=None):
    """checkhermitian(z, n) — KrylovKit.jl:149-153: real scalars pass unchanged."""
    return float(z)


def _checkposdef(z):
    """checkposdef — KrylovKit.jl:143-148."""
    r = _checkhermitian(z)
    if not r > 0:
        raise ValueError(f"operator does not appear to be positive definite: diagonal element {z}")
    return r


def _rayleigh(f, x: B200Vec):
    """ax, bx = genapply(f, x) with inner(x, ax) and inner(x, bx) — golubye.jl:9,13-14 and :112,114."""
    if isinstance(f, B200Pencil):
        ax, bx = x.ctx.empty(x.space), x.ctx.empty(x.space)
        xax, xbx = f.rayleigh_into(x, ax, bx)
        return ax, bx, xax, xbx
    ax, bx = genapply(f, x)
    return ax, bx, x.inner(ax), x.inner(bx)


def _shifted(f, v: B200Vec, rho: float):
    """av, bv = genapply(f, v); av = add!!(av, bv, -ρ) — golubye.jl:65-67, 80-82."""
    if isinstance(f, B200Pencil):
        w, bv = v.ctx.empty(v.space), v.ctx.empty(v.space)
        f.apply_into(v, w, bv, rho)
        return w, bv
    av, bv = genapply(f, v)
    return av.add_(bv, -rho), bv


def golubyerecurrence(f, rho: float, V: OrthonormalBasis, beta: float, orth):
    """golubyerecurrence ×6 (+ the flagged mgs2b) — golubye.jl:196-284.  A pencil forms the product, the shift, the
    MGS-order `add!!(w, V[end-1], -β)` and the first inner product in one call (b2k_pencil_apply); the MGS family's
    `orthogonalize!!(w, v, ModifiedGramSchmidt())` is then `add!!(w, v, -s)` with that s.  Other forms take the
    literal genapply / add!! / inner sequence.  Returns (w, α, β, bv)."""
    t = orth.tag
    v = V[-1]
    mgs_family = t in (L.MGS, L.MGS2, L.MGSIR, L.MGS2B)
    if isinstance(f, B200Pencil):
        w, bv = v.ctx.empty(v.space), v.ctx.empty(v.space)
        if mgs_family:
            alpha = f.apply_into(v, w, bv, rho, V[-2], beta, dot=True)
        else:
            alpha = f.apply_into(v, w, bv, rho, dot=True)
    else:
        av, bv = genapply(f, v)
        w = av.add_(bv, -rho)
        if mgs_family:
            w = w.add_(V[-2], -beta)
        alpha = v.inner(w)
    if not mgs_family:
        w = w.add_(V[-2], -beta)
    w = w.add_(v, -alpha)
    eps = float(np.finfo(v.ctx.np_dtype).eps)
    if t in (L.CGS, L.MGS):
        return w, alpha, w.norm(), bv
    if t == L.CGS2:
        w, s = orthogonalize_(w, V, cgs)
        alpha += s[len(V) - 1]
        return w, alpha, w.norm(), bv
    if t == L.MGS2:
        s = alpha
        for q in V:
            w, s = orthogonalize_(w, q, mgs)
        alpha += s
        return w, alpha, w.norm(), bv
    if t == L.MGS2B:
        # flagged: MGS2 with its second sweep over V applied as one classical block (algorithms.py)
        w, s = orthogonalize_(w, V, cgs)
        alpha += s[len(V) - 1]
        return w, alpha, w.norm(), bv
    if t in (L.CGSIR, L.MGSIR):
        ab2 = alpha * alpha + beta * beta
        beta = w.norm()
        nold = math.sqrt(beta * beta + ab2)
        while eps < beta < orth.eta * nold:
            nold = beta
            if t == L.CGSIR:
                w, s = orthogonalize_(w, V, cgs)
                alpha += s[len(V) - 1]
            else:
                s = 0.0
                for q in V:
                    w, s = orthogonalize_(w, q, mgs)
                alpha += s
            beta = w.norm()
        return w, alpha, beta, bv
    raise ValueError(f"unknown orthogonalizer {orth}")


def _border(HHA: np.ndarray, V: OrthonormalBasis, av: B200Vec, K: int):
    """HHA[i, K + 1] = inner(V[i], av), HHA[K + 1, i] = its conjugate, i in 1:K (golubye.jl:68-71, 83-86), as one
    project!! call."""
    col = project_(np.zeros(K), V, av)
    HHA[:K, K] = col
    HHA[K, :K] = col


def buildHB_(HB: np.ndarray, V: OrthonormalBasis, BV: list):
    """buildHB! — golubye.jl:286-295, from one b2k_basis_cross_inner call: G = V'(BV), the lower triangle with the
    diagonal, mirrored; checkposdef on the diagonal."""
    m = len(V)
    if m > MAX_HB_COLUMNS:
        raise ValueError(f"geneigsolve: the projected B would have {m} columns; at most {MAX_HB_COLUMNS} are supported "
                         "(krylovdim + 1 + converged)")
    G = cross_inner(V, BV)
    for j in range(m):
        HB[j, j] = _checkposdef(G[j, j])
        HB[j + 1:m, j] = G[j + 1:m, j]
        HB[j, j + 1:m] = G[j + 1:m, j]


def geneigh_(HA: np.ndarray, HB: np.ndarray):
    """geneigh! — dense/linalg.jl:118-120, LAPACK.sygvd!(1, 'V', 'U', A, B).  Like the reference it overwrites HA
    (a view of HHA) with the eigenvectors; that matters when the iteration expands again after a process step."""
    D, Z = scipy.linalg.eigh(HA, HB, lower=False, driver="gvd")
    HA[:, :] = Z
    return D, HA


def geneigsolve_golubye(f, x0: B200Vec, howmany: int, which, alg: GolubYe):
    """geneigsolve(f, x₀, howmany, which, alg::GolubYe) — golubye.jl:1-194, step for step.  The vector objects alias
    as the reference's do: `vold` is the first basis vector of the first cycle and is orthonormalized in place and
    pushed into V in every later cycle (:30, :64); the restart scales the last Ritz triple of the loop in place, which
    may be vectors already returned in `vectors` / `residuals` (:165-168)."""
    krylovdim, maxiter = alg.krylovdim, alg.maxiter
    if howmany > krylovdim:
        raise ValueError(f"krylov dimension {krylovdim} too small to compute {howmany} eigenvalues")
    numiter = 1
    ax0, bx0, xax, xbx = _rayleigh(f, x0)
    numops = 1
    beta0 = x0.norm()
    if beta0 == 0:
        raise ValueError("initial vector should not have norm zero")
    xax, xbx = xax / beta0 ** 2, xbx / beta0 ** 2
    invbeta0 = 1.0 / beta0
    v = x0.scale(invbeta0)
    av = ax0.scale_(invbeta0)        # scale!!(zerovector(v), ax₀, invβ₀): ax₀ is not used again
    bv = bx0.scale_(invbeta0)
    rho = _checkhermitian(xax) / _checkposdef(xbx)
    r = av.add_(bv, -rho)
    tol = alg.tol
    HHA = np.zeros((krylovdim + 1, krylovdim + 1), order="F")
    HHB = np.zeros((krylovdim + 1, krylovdim + 1), order="F")
    vold = v
    V = OrthonormalBasis([v])
    BV = [bv]
    r, alpha = orthogonalize_(r, v, alg.orth)
    beta = r.norm()
    converged = 0
    values, vectors, residuals, normresiduals = [], [], [], []
    K = 1
    HHA[K - 1, K - 1] = alpha
    while True:
        beta = r.norm()
        if beta <= tol and K < howmany:
            if alg.verbosity >= WARN_LEVEL:
                warnings.warn(f"Invariant subspace of dimension {K} (up to requested tolerance `tol = {tol}`), which "
                              f"is smaller than the number of requested eigenvalues (i.e. `howmany == {howmany}`);"
                              f"setting `howmany = {K}`.")
            howmany = K
        if K == krylovdim - converged or beta <= tol:       # process
            if numiter > 1:
                v, _, _ = orthonormalize_(vold, V, alg.orth)     # in place: v is vold
                av, bv = _shifted(f, v, rho)
                numops += 1
                _border(HHA, V, av, K)
                K += 1
                HHA[K - 1, K - 1] = _checkhermitian(v.inner(av))
                V.push(v)
                BV.append(bv)
            for i in range(converged):
                v, _, _ = orthonormalize_(vectors[i].copy(), V, alg.orth)
                av, bv = _shifted(f, v, rho)
                numops += 1
                _border(HHA, V, av, K)
                K += 1
                HHA[K - 1, K - 1] = _checkhermitian(v.inner(av))
                V.push(v)
                BV.append(bv)
            av = None
            HA, HB = HHA[:K, :K], HHB[:K, :K]
            buildHB_(HB, V, BV)
            HA += rho * HB
            D, Z = geneigh_(HA, HB)
            p = eigsort(which)(D)
            converged = 0
            values, vectors, residuals, normresiduals = [], [], [], []
            for k in range(K):
                z = Z[:, p[k]].copy()
                v = unproject_(vold.zerovector(), V, z)
                av, bv, vav, vbv = _rayleigh(f, v)
                numops += 1
                rho = _checkhermitian(vav) / _checkposdef(vbv)
                r = av.add_(bv, -rho)
                beta = r.norm()
                if beta < tol * float(np.linalg.norm(z)):
                    converged += 1
                elif numiter < maxiter:
                    break       # in the last iteration, keep adding unconverged vectors up to howmany
                values.append(rho)
                vectors.append(v)
                residuals.append(r)
                normresiduals.append(beta)
                if k + 1 == howmany and numiter == maxiter:
                    break
            av = None
            if converged >= howmany:
                howmany = converged
                break
        if K < krylovdim - converged:       # expand
            v = r.scale_(1 / beta)
            V.push(v)
            HHA[K, K - 1] = beta
            HHA[K - 1, K] = beta
            betaold = beta
            r, alpha, beta, bv = golubyerecurrence(f, rho, V, betaold, alg.orth)
            numops += 1
            K += 1
            n = math.hypot(alpha, beta, betaold)
            HHA[K - 1, K - 1] = _checkhermitian(alpha, n)
            BV.append(bv)
        else:                               # restart
            if numiter == maxiter:
                break
            V.resize_(0)
            BV.clear()
            HHA[:] = 0
            HHB[:] = 0
            K = 1
            invbeta = 1 / v.norm()
            v = v.scale_(invbeta)
            bv = bv.scale_(invbeta)
            r = r.scale_(invbeta)
            r, alpha = orthogonalize_(r, v, alg.orth)
            beta = r.norm()
            V.push(v)
            HHA[K - 1, K - 1] = alpha
            BV.append(bv)
            numiter += 1
    normres = np.array(normresiduals)
    if converged < howmany and alg.verbosity >= WARN_LEVEL:
        warnings.warn(f"Golub-Ye geneigsolve stopped without convergence after {numiter} iterations: {converged} "
                      f"eigenvalues converged, norm of residuals = {normres}, number of operations = {numops}")
    return np.array(values), vectors, ConvergenceInfo(converged, residuals, normres, numiter, numops)
