"""Numpy restatement of bieigsolve with BiArnoldi (src/eigsolve/biarnoldi.jl) for the tests: two Arnoldi
factorizations of the oracle (oracle/krylov_oracle.py), one of A and one of A', and the oblique projection
M = W'V grown the reference's way — after every expansion the 2L + 1 inner products of the new border, at every
process step 2L more for W'r_V and V'r_W — so that the library's deferred M (one cross Gram sweep per process
step) is checked against the literal one.  `inner_calls` counts those inner products."""
from __future__ import annotations

import math

import numpy as np
from scipy.linalg import lu_factor, lu_solve

from oracle import krylov_oracle as ko

inner_calls = [0]


def _inner(x, y):
    inner_calls[0] += 1
    return ko.inner(x, y)


def _sorter(which):
    if hasattr(which, "permutation"):                    # EigSorter
        return which.permutation
    return ko.eigsort_complex(which)


def _isapprox(x, y):
    return np.linalg.norm(x - y) <= math.sqrt(np.finfo(float).eps) * max(np.linalg.norm(x), np.linalg.norm(y))


def bischursolve(A, At, v0, w0, howmany, which, krylovdim, maxiter, tol, orth, eager, warn):
    if howmany > krylovdim:
        raise ValueError("krylov dimension too small")
    sort = _sorter(which)
    normal = (lambda x: A @ x) if not callable(A) else A
    adjoint = (lambda x: At @ x) if not callable(At) else At
    numiter = 1
    fV = ko.arnoldi_initialize(normal, v0, orth)
    fW = ko.arnoldi_initialize(adjoint, w0, orth)
    numops = 1
    MM = np.zeros((krylovdim, krylovdim))
    MM[0, 0] = _inner(fW.V[0], fV.V[0])
    converged = 0
    S = T = Q = Z = rV = rW = h = k = M = MWv = MVw = None
    while True:
        bv, bw = fV.normres(), fW.normres()
        Lk = fV.k
        if (bv <= tol or bw <= tol) and Lk < howmany:
            warn("Invariant subspace")
        if Lk == krylovdim or (bv <= tol and bw <= tol) or (eager and Lk >= howmany):
            H, K = ko.arnoldi_rayleighquotient(fV), ko.arnoldi_rayleighquotient(fW)
            M = MM[:Lk, :Lk].copy()
            rV, rW = fV.r * (1 / bv), fW.r * (1 / bw)
            Wv = np.array([_inner(fW.V[i], rV) for i in range(Lk)])
            Vw = np.array([_inner(fV.V[i], rW) for i in range(Lk)])
            luM = lu_factor(M)
            MWv, MVw = lu_solve(luM, Wv), lu_solve(luM, Vw, trans=1)
            H[:, Lk - 1] += bv * MWv
            K[:, Lk - 1] += bw * MVw
            for i in range(Lk):
                rV = rV - MWv[i] * fV.V[i]
                rW = rW - MVw[i] * fW.V[i]
            brV, brW = ko.norm(rV), ko.norm(rW)
            S, Q, valsH = ko.hschur(H)
            T, Z, valsK = ko.hschur(K)
            S, Q, _ = ko.permuteschur(S, Q, sort(valsH))
            T, Z, _ = ko.permuteschur(T, Z, sort(np.conj(valsK)))
            h, k = Q[Lk - 1, :] * bv, Z[Lk - 1, :] * bw
            converged = 0
            while converged < Lk and max(brV * abs(h[converged]), brW * abs(k[converged])) <= tol:
                converged += 1
            if 0 < converged < Lk and S[converged, converged - 1] != 0:
                converged -= 1
            if converged >= howmany or (bv <= tol and bw <= tol):
                break
        if Lk < krylovdim:
            fV = ko.arnoldi_expand(normal, fV, orth)
            fW = ko.arnoldi_expand(adjoint, fW, orth)
            for i in range(Lk):
                MM[i, Lk] = _inner(fW.V[i], fV.V[Lk])
                MM[Lk, i] = _inner(fW.V[Lk], fV.V[i])
            MM[Lk, Lk] = _inner(fW.V[Lk], fV.V[Lk])
            numops += 2
        else:
            if numiter == maxiter:
                break
            keep = (3 * krylovdim + 2 * converged) // 5
            H, K = np.array(S), np.array(T)
            while H[keep, keep - 1] != 0 or K[keep, keep - 1] != 0:
                if keep > 1:
                    keep -= 1
                else:
                    keep += 1
                    if krylovdim == 2:
                        warn("stuck in a 2x2 block")
                        break
            VQv = -(Q[:, :keep].T @ MWv)
            WZw = -(Z[:, :keep].T @ MVw)
            H[:keep, :keep] += np.outer(VQv, h[:keep])
            K[:keep, :keep] += np.outer(WZw, k[:keep])
            QVQv, ZWZw = Q[:, :keep] @ VQv, Z[:, :keep] @ WZw
            for i in range(Lk):
                rV = rV - QVQv[i] * fV.V[i]
                rW = rW - ZWZw[i] * fW.V[i]
            brV, brW = ko.norm(rV), ko.norm(rW)
            rV, rW = rV * (1 / brV), rW * (1 / brW)
            h, k = h * brV, k * brW
            ko.restore_arnoldi_form(Q, H, h, keep)
            ko.restore_arnoldi_form(Z, K, k, keep)
            for f, Hs in ((fV, H), (fW, K)):
                for j in range(1, Lk + 1):
                    for i in range(1, min(j + 1, Lk) + 1):
                        f.H[ko.hidx(i, j)] = Hs[i - 1, j - 1]
            ko.basistransform(fV.V, Q[:, :keep])
            fV.V[keep] = rV
            ko.basistransform(fW.V, Z[:, :keep])
            fW.V[keep] = rW
            MM[:keep, :keep] = Z[:, :keep].T @ (M @ Q[:, :keep])
            fV = ko.arnoldi_shrink(fV, keep)
            fW = ko.arnoldi_shrink(fW, keep)
            S, T = H, K
            numiter += 1
    return (S, T), (Q, Z), (fV.V, fW.V), (rV, rW), (h, k), M, converged, numiter, numops


def bieigsolve_biarnoldi(A, At, v0, w0, howmany=1, which="LM", krylovdim=30, maxiter=100, tol=1e-12,
                         orth: ko.Orth = ko.Orth(ko.MGS2), eager=False):
    """(values, (vectorsV, vectorsW), (infoV, infoW), warnings) with the infos as dicts."""
    msgs = []
    (S, T), (Q, Z), (V, W), (rV, rW), (h, k), M, converged, numiter, numops = bischursolve(
        A, At, np.asarray(v0, dtype=np.float64), np.asarray(w0, dtype=np.float64), howmany, which, krylovdim,
        maxiter, tol, orth, eager, msgs.append)
    hm = howmany
    if howmany < T.shape[0] and T[howmany, howmany - 1] != 0:
        hm += 1
    elif T.shape[0] < howmany:
        hm = T.shape[0]
    if converged > howmany:
        hm = converged
    SS, TT = S[:hm, :hm], T[:hm, :hm]
    values = ko.schur2eigvals(SS)
    vecsS = ko.schur2eigvecs(SS)
    ZMQ = Z[:, :hm].T @ M @ Q[:, :hm]
    vecsT = np.linalg.inv((ZMQ @ vecsS).conj().T)
    if not _isapprox(TT @ vecsT, vecsT @ np.diag(np.conj(values))):
        msgs.append("Unexpected relation between S and T")
    Vm, Wm = np.column_stack(V[:len(Q)]), np.column_stack(W[:len(Z)])
    VS, VT = Q[:, :hm] @ vecsS, Z[:, :hm] @ vecsT
    fS = np.array([np.dot(h[:hm], vecsS[:, i]) for i in range(hm)])
    fT = np.array([np.dot(k[:hm], vecsT[:, i]) for i in range(hm)])
    infoV = dict(converged=converged, residual=[rV * s for s in fS], normres=ko.norm(rV) * np.abs(fS),
                 numiter=numiter, numops=numops)
    infoW = dict(converged=converged, residual=[rW * s for s in fT], normres=ko.norm(rW) * np.abs(fT),
                 numiter=numiter, numops=numops)
    if converged < howmany:
        msgs.append("stopped without convergence")
    return values, ([Vm @ VS[:, i] for i in range(hm)], [Wm @ VT[:, i] for i in range(hm)]), (infoV, infoW), msgs
