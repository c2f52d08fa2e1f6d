"""bieigsolve with the BiArnoldi (two-sided Krylov-Schur) algorithm — mirror of src/eigsolve/biarnoldi.jl.

Left and right eigenvectors of a real, non-symmetric operator, biorthogonal to each other: the right ones from an
Arnoldi factorization of A, the left ones from one of A', tied together through the oblique projection
M = W'V (W, V the two Krylov bases).  All n-length work runs on the device: the two Arnoldi expansions, the
oblique corrections of the residuals, one basistransform! per side and restart, the eigenvector combinations, and
M itself (b2k_basis_cross_inner); the projected problems are handled on the host as in the reference.
"""
from __future__ import annotations

import warnings

import numpy as np
from scipy.linalg import lu_factor, lu_solve

from . import _lib as L
from .algorithms import BiArnoldi, ConvergenceInfo, KrylovDefaults, WARN_LEVEL
from .dense import eigsort_complex, hidx, hschur, permuteschur, restore_arnoldi_form, schur2eigvals, schur2eigvecs
from .factorizations import biarnoldi as ba
from .operators import B200CSR, B200Dense, B200Operator, apply_adjoint, apply_normal
from .orthonormal import basistransform_, cross_inner, unproject_
from .schursolve import ComplexVec
from .vectors import B200Context, B200Vec


def bieigsolve(A, v0=None, w0=None, howmany: int = 1, which="LM", alg: BiArnoldi | None = None, device: int = 0,
               **kwargs):
    """bieigsolve(A, v₀, w₀, howmany, which, alg::BiArnoldi) — eigsolve/biarnoldi.jl:104-200.

    A is one of
      * a B200CSR: A' is built on the device (B200CSR.transpose()) and freed before returning;
      * a B200Dense (square, x and y in the same space);
      * a tuple (A, At) of device operators or callables on B200Vec;
      * a callable f(x, adjoint: bool);
      * a scipy sparse matrix or a numpy array on the host: v₀ and w₀ are then host arrays (drawn uniformly from
        [0, 1) when omitted), A is uploaded once and transposed on the device, and the vectors come back as
        complex numpy arrays.
    Keyword arguments (krylovdim, maxiter, tol, orth, eager, verbosity) build a BiArnoldi as the reference's keyword
    method does.  Returns (values, (vectorsV, vectorsW), (infoV, infoW)); complex eigenvectors of the device
    paths are ComplexVec pairs.
    """
    from .eigsolve import checkwhich
    if alg is None:
        kw = dict(krylovdim=KrylovDefaults.krylovdim, maxiter=KrylovDefaults.maxiter, tol=KrylovDefaults.tol,
                  orth=KrylovDefaults.orth, eager=False, verbosity=KrylovDefaults.verbosity)
        unknown = set(kwargs) - set(kw)
        if unknown:
            raise TypeError(f"bieigsolve: unknown keyword arguments {sorted(unknown)}")
        kw.update(kwargs)
        alg = BiArnoldi(**kw)
    elif kwargs:
        raise TypeError(f"bieigsolve: keyword arguments {sorted(kwargs)} only apply when no algorithm is passed")
    checkwhich(which, alg)
    if _is_host_matrix(A):
        return _bieigsolve_host(A, v0, w0, howmany, which, alg, device)
    if not isinstance(v0, B200Vec) or not isinstance(w0, B200Vec):
        raise TypeError("bieigsolve: device operators need device start vectors v0 and w0 (B200Vec)")
    if v0.ctx.nranks > 1:
        raise L.B200Error("bieigsolve: row-sharded contexts are not supported")
    At = None
    if isinstance(A, B200CSR):
        At = A.transpose()
        normal, adjoint = A, At
    elif isinstance(A, B200Dense):
        normal, adjoint = (lambda x: apply_normal(A, x)), (lambda x: apply_adjoint(A, x))
    elif isinstance(A, tuple) and len(A) == 2:
        normal, adjoint = A
    elif callable(A) and not isinstance(A, B200Operator):
        normal, adjoint = (lambda x: A(x, False)), (lambda x: A(x, True))
    else:
        raise TypeError(f"bieigsolve: unsupported linear map {type(A).__name__}")
    try:
        return bieigsolve_biarnoldi(normal, adjoint, v0, w0, howmany, which, alg)
    finally:
        if At is not None:
            At.free()


def _is_host_matrix(A) -> bool:
    import scipy.sparse as sp
    return sp.issparse(A) or (isinstance(A, np.ndarray) and A.ndim == 2)


def _bieigsolve_host(A, v0, w0, howmany, which, alg, device=0):
    """Host-matrix entry: upload A once, transpose it on the device, solve, download complex numpy vectors.  The
    slab holds both bases with their residuals and expansion work vectors, the two residual copies of a process
    step and the Ritz vectors being formed."""
    import scipy.sparse as sp
    n = A.shape[0]
    if A.shape != (n, n):
        raise L.DimensionMismatch(f"bieigsolve: A must be square, got {A.shape}")
    rng = np.random.default_rng()
    v0 = rng.random(n) if v0 is None else np.asarray(v0)
    w0 = rng.random(n) if w0 is None else np.asarray(w0)
    dtype = np.float32 if v0.dtype == np.float32 else np.float64
    ctx = B200Context(n, 2 * alg.krylovdim + 24, dtype=dtype, device=device)
    try:
        op = B200CSR.from_scipy(ctx, sp.csr_matrix(A))
        At = op.transpose()
        try:
            return bieigsolve_biarnoldi(op, At, ctx.from_host(v0.astype(dtype)), ctx.from_host(w0.astype(dtype)),
                                        howmany, which, alg, to_host=True)
        finally:
            At.free()
            op.free()
    finally:
        ctx.close()


def _bischursolve(normal, adjoint, v0: B200Vec, w0: B200Vec, howmany: int, which, alg: BiArnoldi):
    """_bischursolve — eigsolve/biarnoldi.jl:202-455, step for step, with one structural difference: where M = W'V
    comes from.  The reference adds a border of M with 2L + 1 inner products after every expansion and takes
    W' r_V and V' r_W with 2L more at every process step.  Here M's leading k_known x k_known block is known (0 at
    the start, `keep` after a restart: Zₖ' M Qₖ on the host as in the reference); expansions take no inner products,
    and each process step makes ONE b2k_basis_cross_inner call with X = [W₁ … W_L, r̂_W], Y = [V₁ … V_L, r̂_V]
    that skips the known block.  r̂ is the residual already scaled by 1/β, as the reference scales it first.  These
    are the reference's own entries ⟨W_i, V_j⟩, ⟨W_i, r̂_V⟩, ⟨V_j, r̂_W⟩, formed later: the vectors do not change
    between their creation and the next restart.  With eager = true a process step therefore computes only the
    rows and columns added since the previous one."""
    krylovdim, maxiter = alg.krylovdim, alg.maxiter
    if howmany > krylovdim:
        raise ValueError(f"krylov dimension {krylovdim} too small to compute {howmany} eigenvalues")
    sort = eigsort_complex(which)
    numiter = 1
    it = ba.BiArnoldiIterator(normal, adjoint, v0, w0, alg.orth)
    fact = ba.initialize(it)
    numops = 1
    tol = alg.tol
    MM = np.zeros((krylovdim + 1, krylovdim + 1), order="F")     # M = MM[:L, :L]; row / column L: the projections
    k_known = 0
    converged = 0
    S = T = Q = Z = rV = rW = h = k = M = None
    MWv = MVw = None
    while True:
        bv, bw = fact.normres()
        Lk = len(fact)
        if (bv <= tol or bw <= tol) and Lk < howmany and alg.verbosity >= WARN_LEVEL:
            warnings.warn(f"Invariant subspace of dimension {Lk} (up to requested tolerance `tol = {tol}`), "
                          f"which is smaller than the number of requested eigenvalues (i.e. `howmany == {howmany}`).")
        if Lk == krylovdim or (bv <= tol and bw <= tol) or (alg.eager and Lk >= howmany):     # process
            H, K = fact.rayleighquotient()
            # Step 1: the residuals, normalised to the next Arnoldi vectors
            rV, rW = fact.residual()
            if Lk < krylovdim:           # a copy: later expansions continue from the unnormalised residual
                rV, rW = rV.scale(1 / bv), rW.scale(1 / bw)
            else:
                rV, rW = rV.scale_(1 / bv), rW.scale_(1 / bw)
            # Steps 2-3: the oblique projection, with M and both projections from one sweep
            V, W = fact.basis()
            cross_inner(list(W.basis) + [rW], list(V.basis) + [rV], skip=(k_known, k_known), G=MM)
            k_known = Lk
            M = MM[:Lk, :Lk].copy()
            Wv = MM[:Lk, Lk].copy()          # ⟨W_i, r̂_V⟩
            Vw = MM[Lk, :Lk].copy()          # ⟨r̂_W, V_i⟩ = ⟨V_i, r̂_W⟩
            luM = lu_factor(M, check_finite=False)
            MWv = lu_solve(luM, Wv)
            MVw = lu_solve(luM, Vw, trans=1)
            H[:, Lk - 1] += bv * MWv         # H̃ = H + (M \ (W' v)) h'
            K[:, Lk - 1] += bw * MVw         # K̃ = K + (M' \ (V' w)) k'
            rV = unproject_(rV, V, MWv, -1.0, 1.0)      # ṽ = v − V M⁻¹W'v (the reference's chain of add!!)
            rW = unproject_(rW, W, MVw, -1.0, 1.0)
            brV, brW = rV.norm(), rW.norm()
            # Steps 5-6: Schur forms, ordered (the left side by the conjugate values)
            S, Q, valuesH = hschur(H)
            T, Z, valuesK = hschur(K)
            S, Q, _ = permuteschur(S, Q, sort(valuesH))
            T, Z, _ = permuteschur(T, Z, sort(np.conj(valuesK)))
            # Steps 7-8 (partly): h̃ = Q' h, k̃ = Z' k
            h = Q[Lk - 1, :] * bv
            k = Z[Lk - 1, :] * bw
            converged = 0
            while converged < Lk:
                if max(brV * abs(h[converged]), brW * abs(k[converged])) <= tol:
                    converged += 1
                else:
                    break
            if 0 < converged < Lk and S[converged, converged - 1] != 0:
                converged -= 1
            if converged >= howmany or (bv <= tol and bw <= tol):
                break
        if Lk < krylovdim:               # expand
            fact = ba.expand_(it, fact)
            numops += 2
        else:                            # shrink
            if numiter == maxiter:
                break
            keep = (3 * krylovdim + 2 * converged) // 5
            H, K = S, T                  # hschur! / permuteschur! work in place in the reference
            while H[keep, keep - 1] != 0 or K[keep, keep - 1] != 0:
                # in the middle of a 2x2 block: shrink by one more, but never to zero
                if keep > 1:
                    keep -= 1
                else:
                    keep += 1
                    if krylovdim == 2:
                        if alg.verbosity >= WARN_LEVEL:
                            warnings.warn("Arnoldi iteration got stuck in a 2x2 block, consider increasing the "
                                          "Krylov dimension")
                        break
            # Steps 10-11: Ĥ = Sₖₖ − Qₖ' M⁻¹W'v h̃ₖ', K̂ likewise, and the residuals
            VQv = -(Q[:, :keep].T @ MWv)
            WZw = -(Z[:, :keep].T @ MVw)
            H[:keep, :keep] += np.outer(VQv, h[:keep])
            K[:keep, :keep] += np.outer(WZw, k[:keep])
            V, W = fact.basis()
            rV = unproject_(rV, V, Q[:, :keep] @ VQv, -1.0, 1.0)
            rW = unproject_(rW, W, Z[:, :keep] @ WZw, -1.0, 1.0)
            brV, brW = rV.norm(), rW.norm()
            rV = rV.scale_(1 / brV)
            rW = rW.scale_(1 / brW)
            h = h * brV
            k = k * brW
            restore_arnoldi_form(Q, H, h, keep)
            restore_arnoldi_form(Z, K, k, keep)
            for side, Hs in ((fact.VH, H), (fact.WK, K)):      # copy!(rayleighquotient(fact), (H, K))
                for j in range(1, Lk + 1):
                    for i in range(1, min(j + 1, Lk) + 1):
                        side.H[hidx(i, j)] = float(Hs[i - 1, j - 1])
            basistransform_(V, Q[:, :keep])
            V[keep] = rV
            basistransform_(W, Z[:, :keep])
            W[keep] = rW
            # Step 9: M of the new bases, Zₖ' M Qₖ
            MM[:keep, :keep] = Z[:, :keep].T @ (M @ Q[:, :keep])
            k_known = keep
            fact = ba.shrink_(fact, keep)
            numiter += 1
    V, W = fact.basis()
    return (S, T), (Q, Z), (V, W), (rV, rW), (h, k), M, converged, numiter, numops


def _isapprox(x, y, dtype) -> bool:
    """Base.isapprox for arrays: norm(x − y) <= sqrt(eps) max(norm(x), norm(y)), eps of the problem's scalar type
    (the reference's dense matrices have the element type of the vectors)."""
    rtol = np.sqrt(np.finfo(dtype).eps)
    return np.linalg.norm(x - y) <= rtol * max(np.linalg.norm(x), np.linalg.norm(y))


def bieigsolve_biarnoldi(normal, adjoint, v0: B200Vec, w0: B200Vec, howmany: int, which, alg: BiArnoldi,
                         to_host: bool = False):
    """bieigsolve(f, v₀, w₀, howmany, which, alg::BiArnoldi) — eigsolve/biarnoldi.jl:135-200, on the operators of
    the two sides.  `to_host` streams every vector out as a complex numpy array as soon as it is formed."""
    (S, T), (Q, Z), (V, W), (rV, rW), (h, k), M, converged, numiter, numops = \
        _bischursolve(normal, adjoint, v0, w0, howmany, which, alg)
    hm = howmany
    if howmany < T.shape[0] and T[howmany, howmany - 1] != 0:
        hm += 1
    elif T.shape[0] < howmany:
        hm = T.shape[0]
    if converged > howmany:
        hm = converged
    SS, TT = S[:hm, :hm], T[:hm, :hm]
    valuesS = schur2eigvals(SS)
    vecsS = schur2eigvecs(SS)
    # the left eigenvectors from ZᴴMQ S = T' ZᴴMQ: biorthogonal to the right ones by construction
    ZMQ = Z[:, :hm].T @ M @ Q[:, :hm]
    vecsT = np.linalg.inv((ZMQ @ vecsS).conj().T)
    valuesT = np.conj(valuesS)
    if not _isapprox(TT @ vecsT, vecsT @ np.diag(valuesT), v0.ctx.np_dtype) and alg.verbosity >= WARN_LEVEL:
        warnings.warn("Unexpected relation between S and T in BiArnoldi eigsolve: left eigenvectors might not be "
                      "correctly computed")

    fS =np.array([np.dot(h[:hm], vecsS[:, i]) for i in range(hm)])        # hᴴ vecsS (h real)
    fT = np.array([np.dot(k[:hm], vecsT[:, i]) for i in range(hm)])
    vectorsS, residualsS = _combine(V, rV, Q[:, :hm] @ vecsS, fS, to_host)
    vectorsT, residualsT = _combine(W, rW, Z[:, :hm] @ vecsT, fT, to_host)
    normresS = rV.norm() * np.abs(fS)
    normresT = rW.norm() * np.abs(fT)
    if converged < howmany and alg.verbosity >= WARN_LEVEL:
        warnings.warn(f"BiArnoldi eigsolve stopped without convergence after {numiter} iterations: {converged} "
                      f"eigenvalues converged, norm of residuals = {normresS}, number of operations = {numops}")
    infoS = ConvergenceInfo(converged, residualsS, normresS, numiter, numops)
    infoT = ConvergenceInfo(converged, residualsT, normresT, numiter, numops)
    return valuesS, (vectorsS, vectorsT), (infoS, infoT)


def _combine(B, r: B200Vec, C: np.ndarray, f: np.ndarray, to_host: bool):
    """[B * C[:, i]] and the residuals [f[i] r] as complex vectors (device ComplexVec or host arrays)."""
    vecs, res = [], []
    for i in range(C.shape[1]):
        c = C[:, i]
        vec = ComplexVec(B * np.ascontiguousarray(c.real), B * np.ascontiguousarray(c.imag))
        vecs.append(vec.to_host() if to_host else vec)
        del vec
        rr = ComplexVec(r.scale(float(f[i].real)), r.scale(float(f[i].imag)))
        res.append(rr.to_host() if to_host else rr)
        del rr
    return vecs, res
