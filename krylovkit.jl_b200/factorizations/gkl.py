"""Golub-Kahan-Lanczos bidiagonalisation — mirror of src/factorizations/gkl.jl.

Flagged mode `onepass` (SURVEY §8f-4; not a reference mode): the reference's step reads A twice — `apply_adjoint` for
A'u_k, then `apply_normal` for A v_k (gkl.jl:308-323).  For a dense device operator `b2k_op_apply_normal_gram` returns
z = A'(A v_k) from the SAME pass that forms A v_k, and since u_{k+1} = (A v_k - sum_j c_j u_j) / beta_k — c = alpha_k
on u_k plus whatever the reorthogonalisation removed —

    A'u_{k+1} = (z - sum_j c_j G_j) / beta_k,        G_j = A'u_j   (short vectors, kept next to U)

needs no second pass.  G is carried through the thick restart with U's own rotations (svdsolve.py).

The recursion is not unconditionally stable: an error e_j in G_j comes back multiplied by c_j / beta_k, i.e. the image
of u_{k+1} inherits (alpha_k / beta_k) e_k + ... plus the rounding of z itself, ~ eps ||A||^2 / beta_k.  Where the
bidiagonal has alpha_k << beta_k (config 4: a tall matrix with a flat spectrum and a start vector mostly outside its
range) errors die out; where alpha_k > beta_k (a recurrence that is converging to the top of a spread spectrum) they
grow geometrically — measured on the simulator: a factor ~5 per step after the first restart of a 3001 x 120 Gaussian
matrix.  So every recycled image carries an error estimate eta (in units of one direct product's rounding):

    eta_{k+1} = ( sum_j |c_j| eta_j + 2 ||B|| ) / beta_k,       ||B|| = max_k hypot(alpha_k, beta_k) <= ||A||

and an image whose estimate exceeds max(`onepass_eta` = 4, 0.01 tol / (eps ||B||)) — four roundings of a direct product,
or an absolute error of 1 % of the caller's tolerance — is thrown away: that step forms A'u directly (eta = 1), exactly
like the reference.  One pass where it is safe, two where it is not; `passes` counts what was actually streamed,
`numops` keeps counting both products per step, like the reference.  With the estimate in place the results differ
from the two-pass step by rounding at the level of the tolerance asked for (tools/onepass_gkl_study.py, DESIGN.md §6)."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from .. import _lib as L
from ..algorithms import Orthogonalizer, cgs, mgs
from ..operators import B200Dense, apply_adjoint, apply_normal, apply_normal_gram
from ..orthonormal import OrthonormalBasis, orthogonalize_, unproject_
from ..vectors import B200Vec

# columns the cooperative Gram-Schmidt sweep of a chained step holds (U and the new residual after the last step):
# its panel ring, include/b200krylov.h b2k_gkl_expand_many
CHAIN_COLS = {8: 96, 4: 192}       # by element size: Float64, Float32


class GKLIterator:
    """GKLIterator(f, u₀, orth, keepvecs) — gkl.jl:123-139.  u₀ lives in the codomain."""

    def __init__(self, operator, u0: B200Vec, orth: Orthogonalizer, keepvecs: bool = True, onepass: bool = False,
                 onepass_eta: float = 4.0, onepass_eta_tol: float = 0.0, pair=None):
        if not keepvecs and (orth.is_reorth2 or orth.is_ir):
            raise ValueError("Cannot use reorthogonalization without keeping all Krylov vectors")
        if onepass and not isinstance(operator, B200Dense):
            raise TypeError("GKL onepass mode needs a dense device operator (B200Dense)")
        if onepass and not keepvecs:
            raise ValueError("GKL onepass mode keeps all Krylov vectors")
        self.operator, self.u0, self.orth, self.keepvecs, self.onepass = operator, u0, orth, keepvecs, onepass
        # largest error estimate a recycled A'u may carry (module doc): onepass_eta roundings of a direct product, or
        # an absolute error onepass_eta_tol * eps (= a fraction of the caller's tolerance), whichever is larger
        self.onepass_eta, self.onepass_eta_tol = float(onepass_eta), float(onepass_eta_tol)
        # (A, A') as B200CSR operators, A' the exact device transpose of A: expand_many_ may chain the steps on the
        # device (b2k_gkl_expand_many).  A user's (A, At) tuple is not known to be an exact transpose: None.
        self.pair = pair

    def eta_max(self, anorm: float) -> float:
        return max(self.onepass_eta, self.onepass_eta_tol / anorm if anorm > 0 else 0.0)


class GKLFactorization:
    """{k, U, V, αs, βs, r} — gkl.jl:31-38; rayleighquotient = Bidiagonal(αs, βs, :L)."""

    def __init__(self, k, U: OrthonormalBasis, V: OrthonormalBasis, alphas, betas, r: B200Vec,
                 G: OrthonormalBasis | None = None, g_next: B200Vec | None = None, passes: int = 2):
        self.k, self.U, self.V, self.alphas, self.betas, self.r = k, U, V, alphas, betas, r
        # onepass mode only: G[j] = A'U[j] as it was used, g_next = A'(r / beta) for the residual r; else None
        self.G, self.g_next = G, g_next
        self.eta = [1.0] * (len(G) if G is not None else 0)     # error estimates of G[j] / of g_next (module doc)
        self.eta_next = 0.0
        self.anorm = 0.0
        self.passes = passes              # passes over A so far (the reference's step: two per expansion)

    def __len__(self):
        return self.k

    def basis(self, which: str):
        return self.U if which == "U" else self.V

    def residual(self):
        return self.r

    def normres(self):
        return self.betas[-1]


def _eps(v):
    return float(np.finfo(v.ctx.np_dtype).eps)


def initialize(it: GKLIterator) -> GKLFactorization:
    """initialize(iter) — gkl.jl:183-215."""
    u0 = it.u0
    beta0 = u0.norm()
    if beta0 == 0:
        raise ValueError("initial vector should not have norm zero")
    v0 = apply_adjoint(it.operator, u0)
    alpha = v0.norm() / beta0
    z = None
    if it.onepass:
        Av0, z = apply_normal_gram(it.operator, v0)          # z = A'(A v0) from the same pass
    else:
        Av0 = apply_normal(it.operator, v0)
    alpha2 = u0.inner(Av0) / (beta0 * beta0)
    if not math.isclose(alpha2, alpha * alpha, rel_tol=math.sqrt(_eps(u0))):
        raise ValueError("operator and its adjoint are not compatible")
    u = u0.scale(1 / beta0)
    v = v0.scale(1 / (alpha * beta0))
    r = Av0.scale_(1 / (alpha * beta0))
    r = r.add_(u, -alpha)
    beta = r.norm()
    if it.onepass:
        # G_1 = A'u_1 = v0 / beta0;  A'(r / beta) = (z / (alpha beta0) - alpha G_1) / beta
        G = OrthonormalBasis([v0.scale_(1 / beta0)])
        anorm = math.hypot(alpha, beta)
        eta_next = (alpha + 2 * anorm) / beta if beta > 0 else math.inf
        g_next = None
        if eta_next <= it.eta_max(anorm):
            g_next = unproject_(z, G, [alpha], -1 / beta, 1 / (alpha * beta0 * beta))
        else:
            z.free()
        fact = GKLFactorization(1, OrthonormalBasis([u]), OrthonormalBasis([v]), [alpha], [beta], r, G, g_next)
        fact.anorm, fact.eta_next = anorm, eta_next
        return fact
    v0.free()
    return GKLFactorization(1, OrthonormalBasis([u]), OrthonormalBasis([v]), [alpha], [beta], r)


def gklrecurrence(operator, U: OrthonormalBasis, V: OrthonormalBasis, beta: float,
                  orth: Orthogonalizer, state: GKLFactorization | None = None, eta_max=None):
    """gklrecurrence ×5 — gkl.jl:294-404.  `state` (onepass mode): its G / g_next are consumed and renewed."""
    t = orth.tag
    u = U[-1]
    onepass = state is not None and state.G is not None
    if onepass and state.g_next is not None:
        v, state.g_next = state.g_next, None     # A'u recovered from the previous step's pass over A
        eta_k = state.eta_next
    else:
        v = apply_adjoint(operator, u)
        eta_k = 1.0
        if state is not None:
            state.passes += 1
    if onepass:
        state.G.push(v.copy())                   # G_k = A'u_k as it is used (v is modified in place below)
        state.eta.append(eta_k)
    v = v.add_(V[-1], -beta)
    if t == L.MGS2:
        for q in V:
            v, _ = orthogonalize_(v, q, mgs)
    elif t == L.MGS2B:                          # flagged: the same sweep as one classical block
        v, _ = orthogonalize_(v, V, cgs)
    alpha = v.norm()
    if t in (L.CGSIR, L.MGSIR):
        nold = math.sqrt(alpha * alpha + beta * beta)
        while (alpha < orth.eta * nold) if t == L.CGSIR else (_eps(v) < alpha < orth.eta * nold):
            nold = alpha
            if t == L.CGSIR:
                v, _ = orthogonalize_(v, V, cgs)
            else:
                for q in V:
                    v, _ = orthogonalize_(v, q, mgs)
            alpha = v.norm()
    v = v.scale_(1 / alpha)

    z = None
    if onepass:
        r, z = apply_normal_gram(operator, v)   # z = A'(A v) from the same pass over A
    else:
        r = apply_normal(operator, v)
    if state is not None:
        state.passes += 1
    r = r.add_(u, -alpha)
    c = np.zeros(len(U))                        # everything removed from A v: r = A v - sum_j c_j u_j
    c[-1] = alpha
    beta_known = None
    if t == L.CGS2:
        r, x = orthogonalize_(r, U, cgs)        # only the long (U) side is reorthogonalised, :320
        c += x[:len(U)]
        beta_known = orthogonalize_.last_norm
    elif t == L.MGS2:
        for j, q in enumerate(U):
            r, sj = orthogonalize_(r, q, mgs)
            c[j] += sj
    elif t == L.MGS2B:
        r, x = orthogonalize_(r, U, cgs)
        c += x[:len(U)]
        beta_known = orthogonalize_.last_norm
    beta = beta_known if beta_known is not None else r.norm()
    if t in (L.CGSIR, L.MGSIR):
        nold = math.sqrt(alpha * alpha + beta * beta)
        while _eps(r) < beta < orth.eta * nold:
            nold = beta
            if t == L.CGSIR:
                r, x = orthogonalize_(r, U, cgs)
                c += x[:len(U)]
            else:
                for j, q in enumerate(U):
                    r, sj = orthogonalize_(r, q, mgs)
                    c[j] += sj
            beta = r.norm()
    if onepass:
        state.anorm = max(state.anorm, math.hypot(alpha, beta))
        ok = beta > 0 and math.isfinite(beta) and math.isfinite(alpha)
        state.eta_next = (float(np.dot(np.abs(c), state.eta)) + 2 * state.anorm) / beta if ok else math.inf
        if state.eta_next <= (eta_max(state.anorm) if callable(eta_max) else 4.0):
            state.g_next = unproject_(z, state.G, c, -1 / beta, 1 / beta)     # A'(r / beta)
        else:
            z.free()                              # too much inherited error: the next step forms A'u directly
    return v, r, alpha, beta


def expand_(it: GKLIterator, state: GKLFactorization) -> GKLFactorization:
    """expand!(iter, state) — gkl.jl:246-269."""
    betaold = state.normres()
    U, V, r = state.U, state.V, state.r
    U.push(r.scale_(1 / betaold))
    v, r, alpha, beta = gklrecurrence(it.operator, U, V, betaold, it.orth, state, it.eta_max)
    V.push(v)
    state.alphas.append(alpha)
    state.betas.append(beta)
    state.k += 1
    state.r = r
    return state


def expand_many_(it: GKLIterator, state: GKLFactorization, nsteps: int, tol: float, check=None) -> int:
    """Up to `nsteps` consecutive expand! steps, stopping after the first one with normres <= tol or a non-finite
    coefficient; returns the number of steps done.  With `it.pair` and ClassicalGramSchmidt2 or the flagged
    ModifiedGramSchmidt2Blocked they are chained on the device in one C-ABI call (b2k_gkl_expand_many, one host
    synchronisation); every other iterator steps through gklrecurrence, calling `check(state)` after each step.
    The chained steps are committed before an error is raised, like lanczos.expand_many_."""
    if nsteps <= 0:
        return 0
    U, V, r = state.U, state.V, state.r
    k = len(U)
    chained = it.pair is not None and it.orth.tag in (L.CGS2, L.MGS2B)
    if not chained or k + nsteps > CHAIN_COLS[r.ctx.np_dtype.itemsize]:
        done = 0
        for _ in range(nsteps):
            expand_(it, state)
            done += 1
            if check is not None:
                check(state)
            a, b = state.alphas[-1], state.betas[-1]
            if b <= tol or not (math.isfinite(a) and math.isfinite(b)):
                break
        return done
    A, At = it.pair
    ctx = r.ctx
    ucols = (L.c_vec * (k + nsteps + 1))(*[u.handle for u in U.basis], r.handle)
    vcols = (L.c_vec * (k + nsteps))(*[v.handle for v in V.basis])
    al = (C.c_double * nsteps)()
    be = (C.c_double * nsteps)()
    done, rout = C.c_int32(), L.c_vec()
    status = ctx.lib.b2k_gkl_expand_many(ctx.h, A.h, At.h, ucols, vcols, k, nsteps, state.normres(), tol,
                                         it.orth.tag, al, be, C.byref(done), C.byref(rout))
    d = done.value
    if d > 0:
        r.disown()                                  # released (and possibly reused) inside the library
        for i in range(d):
            U.push(B200Vec(ctx, ucols[k + i]))      # columns allocated by the library
            V.push(B200Vec(ctx, vcols[k + i]))
        state.r = B200Vec(ctx, rout.value)
        state.alphas.extend(al[:d])
        state.betas.extend(be[:d])
        state.k += d
        state.passes += 2 * d
    ctx.check(status)
    return d


def shrink_(state: GKLFactorization, k: int) -> GKLFactorization:
    """shrink!(state, k) — gkl.jl:270-291."""
    if state.k != len(state.V):
        raise RuntimeError("we cannot shrink GKLFactorization without keeping vectors")
    if state.k <= k:
        return state
    U, V = state.U, state.V
    while len(V) > k + 1:
        U.pop()
        V.pop()
    V.pop()
    r = U.pop()
    if state.G is not None:
        # G follows U: the vector that becomes the residual direction is U[k], and its image is G[k]  (the thick
        # restart of svdsolve.py has put r / beta into U[k] and A'(r / beta) into G[k] before it shrinks)
        while len(state.G) > k + 1:
            state.G.pop()
            state.eta.pop()
        state.g_next, state.eta_next = state.G.pop(), state.eta.pop()      # (every estimate kept passed the check when it was made)
    del state.alphas[k:]
    del state.betas[k:]
    state.k = k
    state.r = r.scale_(state.normres())
    return state
