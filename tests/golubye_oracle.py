"""TEST INFRASTRUCTURE ONLY — a numpy restatement of KrylovKit's Golub-Ye geneigsolve (src/eigsolve/golubye.jl:1-295),
in float64, with the reference's literal per-step inner products: the border of HHA one inner product at a time
(:68-71, 83-86), buildHB! entry by entry (:286-295).  The projected pencil is solved by LAPACK's sygvd, the routine of
geneigh! (scipy.linalg.eigh(HA, HB, lower=False, driver="gvd")).

Vectors are numpy arrays and alias as the reference's objects do: `vold` is orthonormalized in place in every cycle
after the first (:30, :64); the restart scales the last Ritz triple in place (:165-168).  `alias=False` copies instead,
so that a test can show the aliasing matters.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg

from oracle import krylov_oracle as ko

CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)


class Result:
    def __init__(self, values, vectors, residuals, normres, converged, numiter, numops, warnings):
        self.values, self.vectors, self.residuals, self.normres = values, vectors, residuals, normres
        self.converged, self.numiter, self.numops, self.warnings = converged, numiter, numops, warnings


def _vec_orth(w, q, tag, eta):
    """orthogonalize!!(w, q, alg) against one vector (MGS2B: the reference's MGS2)."""
    return ko.orthogonalize_vec(w, q, ko.Orth(MGS2 if tag == MGS2B else tag, eta))


def _orthonormalize(v, V, tag, eta):
    """orthonormalize!!(v, V, alg) (MGS2B: two classical sweeps, as the library's blocked form)."""
    w, _ = ko.orthogonalize(v, list(V), np.zeros(len(V)), ko.Orth(CGS2 if tag == MGS2B else tag, eta))
    return w / ko.norm(w)


def recurrence(A, B, rho, V, beta, tag, eta):
    """golubyerecurrence — golubye.jl:196-284 (mgs2b: MGS's first part, then one classical sweep over V)."""
    v = V[-1]
    av, bv = A @ v, B @ v
    w = av + (-rho) * bv
    if tag in (CGS, CGS2, CGSIR):
        alpha = ko.inner(v, w)
        w = w + (-beta) * V[-2]
        w = w + (-alpha) * v
    else:
        w = w + (-beta) * V[-2]
        alpha = ko.inner(v, w)
        w = w + (-alpha) * v
    if tag in (CGS, MGS):
        return w, alpha, ko.norm(w), bv
    if tag in (CGS2, MGS2B):
        w, s = ko.orthogonalize(w, list(V), np.zeros(len(V)), ko.Orth(CGS))
        return w, alpha + s[-1], ko.norm(w), bv
    if tag == MGS2:
        s = alpha
        for q in V:
            s = ko.inner(q, w)
            w = w + (-s) * q
        return w, alpha + s, ko.norm(w), bv
    ab2 = alpha * alpha + beta * beta
    beta = ko.norm(w)
    nold = math.sqrt(beta * beta + ab2)
    while np.finfo(np.float64).eps < beta < eta * nold:
        nold = beta
        if tag == CGSIR:
            w, s = ko.orthogonalize(w, list(V), np.zeros(len(V)), ko.Orth(CGS))
            alpha += s[-1]
        else:
            s = 0.0
            for q in V:
                s = ko.inner(q, w)
                w = w + (-s) * q
            alpha += s
        beta = ko.norm(w)
    return w, alpha, beta, bv


def golubye(A, B, x0, howmany, which="LM", krylovdim=30, maxiter=100, tol=1e-12, orth=MGS2, eta=1 / math.sqrt(2),
            alias=True):
    """geneigsolve(f, x₀, howmany, which, alg::GolubYe) — golubye.jl:1-194."""
    if howmany > krylovdim:
        raise ValueError(f"krylov dimension {krylovdim} too small to compute {howmany} eigenvalues")
    warns = []
    x0 = np.asarray(x0, dtype=np.float64)
    numiter = 1
    ax0, bx0 = A @ x0, B @ x0
    numops = 1
    beta0 = ko.norm(x0)
    if beta0 == 0:
        raise ValueError("initial vector should not have norm zero")
    xax = ko.inner(x0, ax0) / beta0 ** 2
    xbx = ko.inner(x0, bx0) / beta0 ** 2
    inv0 = 1.0 / beta0
    v = x0 * inv0
    av = ax0 * inv0
    bv = bx0 * inv0
    assert xbx > 0
    rho = xax / xbx
    r = av + (-rho) * bv
    HHA = np.zeros((krylovdim + 1, krylovdim + 1), order="F")
    HHB = np.zeros((krylovdim + 1, krylovdim + 1), order="F")
    vold = v
    V, BV = [v], [bv]
    r, alpha = _vec_orth(r, v, orth, eta)
    beta = ko.norm(r)
    converged = 0
    values, vectors, residuals, normres = [], [], [], []
    K = 1
    HHA[0, 0] = alpha
    sort = {"SR": lambda d: np.argsort(d, kind="stable"), "LR": lambda d: np.argsort(-d, kind="stable"),
            "LM": lambda d: np.argsort(-np.abs(d), kind="stable")}[which]
    while True:
        beta = ko.norm(r)
        if beta <= tol and K < howmany:
            warns.append("invariant")
            howmany = K
        if K == krylovdim - converged or beta <= tol:
            extra = []
            if numiter > 1:
                new = _orthonormalize(vold, V, orth, eta)
                if alias:
                    vold[:] = new
                    extra.append(vold)
                else:
                    extra.append(new)
            extra += [("conv", i) for i in range(converged)]      # orthonormalize(vectors[i], V): copies
            for item in extra:
                if isinstance(item, tuple):
                    v = _orthonormalize(vectors[item[1]].copy(), V, orth, eta)
                else:
                    v = item
                av, bv = A @ v, B @ v
                numops += 1
                av = av + (-rho) * bv
                for i in range(K):
                    HHA[i, K] = ko.inner(V[i], av)
                    HHA[K, i] = HHA[i, K]
                K += 1
                HHA[K - 1, K - 1] = ko.inner(v, av)
                V.append(v)
                BV.append(bv)
            HA, HB = HHA[:K, :K], HHB[:K, :K]
            for j in range(K):                                  # buildHB!
                HB[j, j] = ko.inner(V[j], BV[j])
                assert HB[j, j] > 0
                for i in range(j + 1, K):
                    HB[i, j] = ko.inner(V[i], BV[j])
                    HB[j, i] = HB[i, j]
            HA += rho * HB
            D, Z = scipy.linalg.eigh(HA, HB, lower=False, driver="gvd")
            HA[:, :] = Z
            Z = HA
            p = sort(D)
            converged = 0
            values, vectors, residuals, normres = [], [], [], []
            for k in range(K):
                z = Z[:, p[k]].copy()
                v = np.zeros_like(vold)
                for i in range(K):
                    v = v + z[i] * V[i]
                av, bv = A @ v, B @ v
                numops += 1
                vbv = ko.inner(v, bv)
                assert vbv > 0
                rho = ko.inner(v, av) / vbv
                r = av + (-rho) * bv
                beta = ko.norm(r)
                if beta < tol * ko.norm(z):
                    converged += 1
                elif numiter < maxiter:
                    break
                values.append(rho)
                vectors.append(v)
                residuals.append(r)
                normres.append(beta)
                if k + 1 == howmany and numiter == maxiter:
                    break
            if converged >= howmany:
                howmany = converged
                break
        if K < krylovdim - converged:
            r *= 1 / beta                      # scale!!(r, 1/β): v is r
            v = r
            V.append(v)
            HHA[K, K - 1] = beta
            HHA[K - 1, K] = beta
            betaold = beta
            r, alpha, beta, bv = recurrence(A, B, rho, V, betaold, orth, eta)
            numops += 1
            K += 1
            HHA[K - 1, K - 1] = alpha
            BV.append(bv)
        else:
            if numiter == maxiter:
                break
            V, BV = [], []
            HHA[:] = 0
            HHB[:] = 0
            K = 1
            invb = 1 / ko.norm(v)
            if alias:
                v *= invb
                bv *= invb
                r *= invb
            else:
                v, bv, r = v * invb, bv * invb, r * invb
            r, alpha = _vec_orth(r, v, orth, eta)
            beta = ko.norm(r)
            V.append(v)
            HHA[0, 0] = alpha
            BV.append(bv)
            numiter += 1
    if converged < howmany:
        warns.append("noconv")
    return Result(np.array(values), vectors, residuals, np.array(normres), converged, numiter, numops, warns)
