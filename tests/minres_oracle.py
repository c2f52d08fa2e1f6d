"""TEST INFRASTRUCTURE ONLY — float64 numpy restatement of linsolve(A, b, x₀, MINRES, a₀, a₁) as
krylovkit.jl_b200/linsolve.py::_minres defines it (the reference declares MINRES and has no driver): Paige & Saunders
(1975), unpreconditioned Lanczos + Givens QR, in the literal operation order of the VectorInterface sequence, with the
stopping rules of cg.jl:69-73 (explicit residual before convergence is reported, restart from x if it disagrees).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np


def fresh_state(beta1: float):
    """[β_k, 1/β_k, 1/β_{k-1}, c, s, δ̄, ε, φ̄] of a process started from a residual of norm β₁"""
    return [beta1, 1.0 / beta1, 0.0, -1.0, 0.0, 0.0, 0.0, beta1]


def givens_step(st, alpha: float, beta_new: float):
    """One step of the scalar recurrence; advances st in place and returns
    (α, β_{k+1}, γ, φ, |φ̄|, γ == 0, δ, ε_k)."""
    c0, s0, dbar, eps, phibar = st[3], st[4], st[5], st[6], st[7]
    delta = c0 * dbar + s0 * alpha
    gbar = s0 * dbar - c0 * alpha
    gamma = math.sqrt(gbar * gbar + beta_new * beta_new)
    if gamma == 0.0:
        c = s = phi = 0.0
        phibar_n = phibar
    else:
        c, s = gbar / gamma, beta_new / gamma
        phi, phibar_n = c * phibar, s * phibar
    st[2], st[0], st[1] = st[1], beta_new, (1.0 / beta_new if beta_new != 0.0 else math.inf)
    st[3], st[4], st[5], st[6], st[7] = c, s, -(c0 * beta_new), s0 * beta_new, phibar_n
    return alpha, beta_new, gamma, phi, abs(phibar_n), gamma == 0.0, delta, eps


@dataclass
class Result:
    x: np.ndarray
    converged: int
    residual: np.ndarray
    normres: float
    numiter: int
    numops: int
    phibars: list = field(default_factory=list)     # |φ̄| after every iteration
    iterates: list = field(default_factory=list)    # x after every iteration (keep_iterates)
    restarts: int = 0
    singular: bool = False


def minres(A, b, x0=None, a0=0.0, a1=1.0, tol=1e-12, maxiter=100, keep_iterates=False) -> Result:
    b = np.asarray(b, dtype=np.float64)
    x = np.zeros_like(b) if x0 is None else np.array(x0, dtype=np.float64)

    def op(v):
        y = A @ v
        return a1 * y + a0 * v if (a0 != 0 or a1 != 1) else y

    r = b - a0 * x - a1 * (A @ x) if a0 != 0 else b - a1 * (A @ x)
    normr = float(np.sqrt(np.dot(r, r)))
    out = Result(x, 0, r, normr, 0, 1)
    if normr < tol:
        out.converged = 1
        return out
    v, v_prev = r * (1.0 / normr), np.zeros_like(b)
    d1, d2 = np.zeros_like(b), np.zeros_like(b)
    st = fresh_state(normr)
    while True:
        q = op(v)
        alpha = float(np.dot(v, q))
        q = q - alpha * v
        q = q - st[0] * v_prev
        _, beta_new, gamma, phi, phibar, sing, delta, eps = givens_step(st, alpha, float(np.sqrt(np.dot(q, q))))
        if not sing:
            d = ((v - delta * d1) - eps * d2) * (1.0 / gamma)
            x = x + phi * d
        else:
            d = np.zeros_like(b)
        d1, d2, v_prev = d, d1, v
        if beta_new != 0.0:
            v = q * st[1]
        out.numiter += 1
        out.numops += 1
        out.phibars.append(phibar)
        if keep_iterates:
            out.iterates.append(x.copy())
        hit = phibar < tol or beta_new == 0.0
        if sing or hit or out.numiter >= maxiter:
            r = b - op(x)
            out.numops += 1
            out.x, out.residual, out.normres = x, r, float(np.sqrt(np.dot(r, r)))
            if sing:
                out.singular = True
                return out
            if hit and (out.normres < tol or out.normres == 0.0):      # (tol = 0: an exact solution still ends it)
                out.converged = 1
                return out
            if out.numiter >= maxiter:
                return out
            out.restarts += 1
            v, v_prev = r * (1.0 / out.normres), np.zeros_like(b)
            d1, d2 = np.zeros_like(b), np.zeros_like(b)
            st = fresh_state(out.normres)
