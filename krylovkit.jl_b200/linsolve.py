"""linsolve with restarted GMRES — mirror of src/linsolve/gmres.jl (and the tolerance
resolution of src/linsolve/linsolve.jl:123-180)."""
from __future__ import annotations

import math
import warnings

import numpy as np

from .algorithms import BiCGStab, CG, ConvergenceInfo, GMRES, MINRES, WARN_LEVEL
from .dense import givens, ldiv_upper
from .factorizations import arnoldi as ar
from .operators import B200CSR, apply
from .orthonormal import rmul_givens_, unproject_
from .vectors import B200Context, B200Vec

# gmres.jl:112-117 rotates the WHOLE basis with k Givens sweeps only to read column k+1.
# True = do exactly that (k two-column sweeps); False = obtain the same column as one
# linear combination with host-accumulated coefficients (rounding differs at the 1e-16 level).
LITERAL_GIVENS_RESTART = False


def linsolve(A, b, x0=None, alg: GMRES | None = None, a0: float = 0.0, a1: float = 1.0,
             atol: float | None = None, rtol: float | None = None, **kwargs):
    """linsolve(A, b, x₀, alg::GMRES, a₀, a₁): solve (a₀ + a₁ A) x = b.
    `tol` of the algorithm is the absolute residual tolerance; pass atol/rtol to get
    KrylovKit's tol = max(atol, rtol*‖b‖) (linsolve.jl:159-161)."""
    if alg is None:
        alg = linselector(A, b, atol=atol, rtol=rtol, **kwargs)
        atol = rtol = None                              # already folded into alg.tol
    elif kwargs:
        raise TypeError(f"linsolve: keyword arguments {sorted(kwargs)} only apply when no algorithm is passed")
    if isinstance(alg, (CG, BiCGStab, MINRES)) and not isinstance(b, B200Vec):
        return _linsolve_host(A, b, x0, alg, a0, a1, atol, rtol)
    if isinstance(alg, CG):
        if not isinstance(b, B200Vec):
            raise TypeError("linsolve(CG): pass device vectors (B200Vec)")
        if atol is not None or rtol is not None:
            alg = CG(maxiter=alg.maxiter, tol=max(atol or 0.0, (rtol or 0.0) * b.norm()), verbosity=alg.verbosity)
        return _cg(A, b, x0 if x0 is not None else b.zerovector(), alg, a0, a1)
    if isinstance(alg, MINRES):
        if atol is not None or rtol is not None:
            alg = MINRES(maxiter=alg.maxiter, tol=max(atol or 0.0, (rtol or 0.0) * b.norm()), verbosity=alg.verbosity)
        return _minres(A, b, x0 if x0 is not None else b.zerovector(), alg, a0, a1)
    if isinstance(alg, BiCGStab):
        if not isinstance(b, B200Vec):
            raise TypeError("linsolve(BiCGStab): pass device vectors (B200Vec)")
        if atol is not None or rtol is not None:
            alg = BiCGStab(maxiter=alg.maxiter, tol=max(atol or 0.0, (rtol or 0.0) * b.norm()),
                           verbosity=alg.verbosity)
        return _bicgstab(A, b, x0 if x0 is not None else b.zerovector(), alg, a0, a1)
    if not isinstance(b, B200Vec):
        return _linsolve_host(A, b, x0, alg, a0, a1, atol, rtol)
    if atol is not None or rtol is not None:
        tol = max(atol or 0.0, (rtol or 0.0) * b.norm())
        alg = GMRES(orth=alg.orth, maxiter=alg.maxiter, krylovdim=alg.krylovdim, tol=tol,
                    verbosity=alg.verbosity)
    if x0 is None:
        x0 = b.zerovector()
    return _gmres(A, b, x0, alg, a0, a1)


def linselector(A, b, issymmetric: bool | None = None, ishermitian: bool | None = None,
                isposdef: bool = False, krylovdim: int | None = None, maxiter: int | None = None,
                rtol: float | None = None, atol: float | None = None, tol: float | None = None, orth=None,
                verbosity: int | None = None):
    """linselector — src/linsolve/linsolve.jl:123-180: CG for symmetric positive definite problems (the
    caller asserts `isposdef`; the reference only tests it for an AbstractMatrix), GMRES otherwise;
    tol = max(atol, rtol·‖b‖) with both defaulting to KrylovDefaults.tol."""
    from .algorithms import KrylovDefaults
    from .eigsolve import _host_issymmetric
    if issymmetric is None:
        issymmetric = _host_issymmetric(A)
    if ishermitian is None:
        ishermitian = issymmetric
    kd = KrylovDefaults.krylovdim if krylovdim is None else krylovdim
    mi = KrylovDefaults.maxiter if maxiter is None else maxiter
    vb = KrylovDefaults.verbosity if verbosity is None else verbosity
    if tol is None:
        nb = b.norm() if isinstance(b, B200Vec) else float(np.linalg.norm(np.asarray(b, dtype=np.float64)))
        tol = max(KrylovDefaults.tol if atol is None else atol, (KrylovDefaults.tol if rtol is None else rtol) * nb)
    if (issymmetric or ishermitian) and isposdef:
        return CG(maxiter=kd * mi, tol=tol, verbosity=vb)
    return GMRES(krylovdim=kd, maxiter=mi, tol=tol, orth=KrylovDefaults.orth if orth is None else orth, verbosity=vb)


def _linsolve_host(A, b, x0, alg, a0, a1, atol, rtol):
    import scipy.sparse as sp
    b = np.asarray(b)
    n = b.shape[0]
    ctx = B200Context(n, getattr(alg, "krylovdim", 0) + 16, dtype=np.float32 if b.dtype == np.float32 else np.float64)
    try:
        if not sp.issparse(A):
            raise TypeError("linsolve: host-side A must be a scipy sparse matrix")
        op = B200CSR.from_scipy(ctx, A)
        bv = ctx.from_host(b)
        xv = ctx.from_host(x0) if x0 is not None else None
        x, info = linsolve(op, bv, xv, alg, a0, a1, atol, rtol)
        info.residual = info.residual.to_host()
        return x.to_host(), info
    finally:
        ctx.close()


def _gmres(operator, b: B200Vec, x0: B200Vec, alg: GMRES, a0: float, a1: float):
    y0 = apply(operator, x0)
    r = b.copy()                               # scale(b, one(T))
    if a0 != 0:
        r = r.add_(x0, -a0)
    r = r.add_(y0, -a1)
    x = x0.copy()                              # scale!!(zerovector(r), x₀, 1)
    beta = r.norm()
    maxiter, krylovdim, tol = alg.maxiter, alg.krylovdim, alg.tol
    if beta < tol:
        return x, ConvergenceInfo(1, r, beta, 0, 1)
    y = np.zeros(krylovdim + 1)
    gs = [None] * krylovdim
    R = np.zeros((krylovdim, krylovdim))
    numiter, numops = 0, 1
    it = ar.ArnoldiIterator(operator, r, alg.orth)
    fact = ar.initialize(it)
    numops += 1
    while True:
        numiter += 1
        y[0] = beta
        k = 1
        R[0, 0] = a0 + a1 * fact.h(1, 1)
        c, s, rr = givens(R[0, 0], a1 * fact.normres())
        gs[0] = (c, s)
        R[0, 0] = rr
        y[1] = 0.0
        y[0], y[1] = c * y[0] + s * y[1], -s * y[0] + c * y[1]
        beta = abs(y[1])
        while R[k - 1, k - 1] != 0 and beta > tol and len(fact) < krylovdim:
            fact = ar.expand_(it, fact)
            numops += 1
            k = len(fact)
            for i in range(1, k):
                R[i - 1, k - 1] = a1 * fact.h(i, k)
            R[k - 1, k - 1] = a0 + a1 * fact.h(k, k)
            for i in range(k - 1):
                c, s = gs[i]
                R[i, k - 1], R[i + 1, k - 1] = (c * R[i, k - 1] + s * R[i + 1, k - 1],
                                                -s * R[i, k - 1] + c * R[i + 1, k - 1])
            if math.hypot(R[k - 1, k - 1], a1 * fact.normres()) < tol:
                if alg.verbosity >= WARN_LEVEL:
                    warnings.warn(f"GMRES linsolve in iteration {numiter}; step {k}: linear operator is "
                                  "singular in Krylov subspace")
                # rotate all the weight into y[k+1] — gmres.jl:84-86: gs[k] = Givens(k+1, k, c, s)
                c, s, rr = givens(0.0, y[k - 1])
                gs[k - 1] = ("swap", c, s)
                y[k] = rr
                y[k - 1] = 0.0
                R[k - 1, k - 1] = 0.0
            else:
                c, s, rr = givens(R[k - 1, k - 1], a1 * fact.normres())
                gs[k - 1] = (c, s)
                R[k - 1, k - 1] = rr
                y[k] = 0.0
                y[k - 1], y[k] = c * y[k - 1] + s * y[k], -s * y[k - 1] + c * y[k]
            beta = abs(y[k])
        if R[k - 1, k - 1] == 0 and y[k - 1] == 0:
            ldiv_upper(R, y, k - 1)
        else:
            ldiv_upper(R, y, k)
        V = fact.basis()
        # x = add!!(x, V[i], y[i]) for i in 1:k — gmres.jl:105-108: one fused lincomb sweep
        x = unproject_(x, V, y[:k], 1.0, 1.0, range(k))
        if beta > tol and numiter < maxiter:
            w = fact.residual()
            V.push(w.scale_(1 / fact.normres()))
            if LITERAL_GIVENS_RESTART:
                for i in range(k):
                    if gs[i][0] == "swap":                    # singular branch: Givens(k+1, k, c, s)
                        rmul_givens_(V, i + 1, i, gs[i][1], -gs[i][2])
                        continue
                    c, s = gs[i]
                    rmul_givens_(V, i, i + 1, c, -s)          # rmul!(V, gs[i]')
                r = r.scale_(y[k], V[k])
            else:
                # column k+1 of V·G₁ᴴ⋯G_kᴴ as coefficients: e_{k+1} pushed back through the rotations
                coef = np.zeros(k + 1)
                coef[k] = 1.0
                for i in range(k - 1, -1, -1):
                    if gs[i][0] == "swap":                    # rotation acting on (i1, i2) = (i+1, i)
                        _, c, s = gs[i]
                        ci1, ci = coef[i + 1], coef[i]
                        coef[i + 1], coef[i] = c * ci1 - s * ci, s * ci1 + c * ci
                        continue
                    c, s = gs[i]
                    ci, ci1 = coef[i], coef[i + 1]
                    coef[i], coef[i + 1] = c * ci - s * ci1, s * ci + c * ci1
                r = unproject_(r, V, coef * y[k], 1.0, 0.0)
        else:
            r = r.scale_(1.0, b)
            r = r.add_(apply(operator, x, a0, a1), -1.0)
            numops += 1
            beta = r.norm()
            if beta < tol:
                return x, ConvergenceInfo(1, r, beta, numiter, numops)
        if numiter >= maxiter:
            if alg.verbosity >= WARN_LEVEL:
                warnings.warn(f"GMRES linsolve stopped without converging after {numiter} iterations: "
                              f"normres = {beta}, numops = {numops}")
            return x, ConvergenceInfo(0, r, beta, numiter, numops)
        it = ar.ArnoldiIterator(operator, r, alg.orth)
        fact = ar.initialize_(it, fact)


USE_FUSED_CG = True      # b2k_cg_step (one host round trip per iteration) for device CSR operators
USE_BICGSTAB_CHAIN = True   # b2k_bicgstab_chain: same for BiCGStab (two device-side convergence tests per iteration)
BICG_CHAIN_LEN = 32
USE_CG_CHAIN = True      # b2k_cg_chain: iterations chained on the device, one host round trip per CG_CHAIN_LEN
CG_CHAIN_LEN = 32


def _cg(operator, b: B200Vec, x0: B200Vec, alg: CG, a0: float, a1: float):
    """linsolve(operator, b, x₀, alg::CG, a₀, a₁) — src/linsolve/cg.jl:1-103 (SURVEY §8f-2)."""
    import ctypes as C
    y0 = apply(operator, x0)
    r = b.copy()
    if a0 != 0:
        r = r.add_(x0, -a0)
    r = r.add_(y0, -a1)
    x = x0.copy()
    normr = r.norm()
    maxiter, tol = alg.maxiter, alg.tol
    numops, numiter = 1, 0
    if normr < tol:
        return x, ConvergenceInfo(1, r, normr, numiter, numops)
    ctx = b.ctx
    fused = USE_FUSED_CG and isinstance(operator, B200CSR)
    rho = normr * normr           # Julia: normr^2 is literal_pow = normr*normr
    p = r.zerovector()
    q = r.zerovector() if fused else None
    beta = 0.0           # first iteration: p = r  (cg.jl:35)
    first = True
    chain = fused and USE_CG_CHAIN and ctx.nranks == 1
    pending: list[float] = []      # ||r|| of iterations the device has already run (b2k_cg_chain), oldest first
    while True:
        if fused and chain and not first:
            if not pending:
                # nothing in the reference's loop needs the host between iterations except the two exit tests;
                # the device applies the ||r|| < tol test itself, the iteration count is bounded here
                m = max(1, min(CG_CHAIN_LEN, maxiter - numiter))
                pqs, nrs, done = (C.c_double * m)(), (C.c_double * m)(), C.c_int32()
                ctx.check(ctx.lib.b2k_cg_chain(ctx.h, operator.h, x.handle, r.handle, p.handle, q.handle, a0, a1,
                                               beta, rho, tol, m, pqs, nrs, C.byref(done)))
                pending = [nrs[i] for i in range(done.value)]
            normr = pending.pop(0)
        elif fused:
            pq, nr = C.c_double(), C.c_double()
            ctx.check(ctx.lib.b2k_cg_step(ctx.h, operator.h, x.handle, r.handle, p.handle, q.handle, a0, a1,
                                          beta, rho, C.byref(pq), C.byref(nr)))
            normr = nr.value
        else:
            p = p.scale_(1.0, r) if first else p.add_(r, 1.0, beta)      # cg.jl:35 / :63
            q = apply(operator, p, a0, a1)
            alpha = rho / p.inner(q)
            x = x.add_(p, alpha)
            r = r.add_(q, -alpha)
            normr = r.norm()
        if not first and normr < tol:
            # recompute to account for buildup of floating point errors — cg.jl:69-73
            r = r.scale_(1.0, b)
            r = r.add_(apply(operator, x, a0, a1), -1.0)
            normr = r.norm()
            rho = normr * normr           # Julia: normr^2 is literal_pow = normr*normr
            beta = 0.0
        else:
            rhoold = rho
            rho = normr * normr           # Julia: normr^2 is literal_pow = normr*normr
            beta = rho / rhoold
        was_first, first = first, False
        numops += 1
        numiter += 1
        if normr < tol:
            return x, ConvergenceInfo(1, r, normr, numiter, numops)
        if not was_first and numiter >= maxiter:     # cg.jl:35-60: the first iteration never looks at maxiter
            if alg.verbosity >= WARN_LEVEL:
                warnings.warn(f"CG linsolve stopped without converging after {numiter} iterations: "
                              f"normres = {normr}, numops = {numops}")
            return x, ConvergenceInfo(0, r, normr, numiter, numops)


USE_FUSED_APPLY_DOT = True   # BiCGStab: take ⟨r̃, A p⟩ and ⟨A s, s⟩ from the SpMV epilogue (b2k_op_apply_dot)


def _apply_and_dot(operator, x: B200Vec, a0: float, a1: float, v: B200Vec):
    """(y, ⟨v, y⟩) with y = apply(operator, x, a₀, a₁).  For an unshifted device CSR operator the inner
    product rides on the SpMV pass (one sweep and one host round trip less); otherwise the two literal
    VectorInterface calls."""
    if USE_FUSED_APPLY_DOT and isinstance(operator, B200CSR) and a0 == 0.0 and a1 == 1.0:
        y = x.ctx.empty(x.space)
        return y, operator.apply_dot_into(y, x, v)
    y = apply(operator, x, a0, a1)
    return y, v.inner(y)


USE_FUSED_BICGSTAB = True    # b2k_bicgstab_half / _full (two host round trips per iteration) for device CSR operators


def _bicgstab(operator, b: B200Vec, x0: B200Vec, alg: BiCGStab, a0: float, a1: float):
    """linsolve(operator, b, x₀, alg::BiCGStab, a₀, a₁) — src/linsolve/bicgstab.jl:1-203
    (SURVEY §8f-2).  Real arithmetic only (the library has no complex dtype).  The reference
    spells its first iteration out ahead of the loop; here one loop serves both, `p is None`
    marking the first pass, including its quirk that `maxiter` is only looked at from the
    second iteration on.  For a device CSR operator every iteration is two fused C-ABI calls
    (b2k_bicgstab_half / _full: 17 vector sweeps + 2 SpMV instead of 28 + 2, two host round trips
    instead of six); any other operator runs the literal VectorInterface sequence."""
    import ctypes as C
    y0 = apply(operator, x0)
    r = b.copy()
    if a0 != 0:
        r = r.add_(x0, -a0)
    r = r.add_(y0, -a1)
    del y0
    x = x0.copy()
    normr = r.norm()
    maxiter, tol = alg.maxiter, alg.tol
    numops, numiter = 1, 0
    if normr < tol:
        return x, ConvergenceInfo(1, r, normr, numiter, numops)
    ctx = b.ctx
    fused = USE_FUSED_BICGSTAB and isinstance(operator, B200CSR)
    r_shadow = r.copy()
    rho = alpha = omega = 1.0
    rho_next = None                              # ⟨r̃, r⟩ delivered by the previous fused full step
    p = v = None
    s, xhalf = r.zerovector(), x.zerovector()
    t = r.zerovector() if fused else None
    chain = fused and USE_BICGSTAB_CHAIN and ctx.nranks == 1
    rec = np.zeros((BICG_CHAIN_LEN, 8)) if chain else None
    while True:
        numiter += 1
        rhoold, rho = rho, (r_shadow.inner(r) if rho_next is None else rho_next)
        rho_next = None
        first = p is None
        half_done = full_done = False
        if chain and not first:
            # iterations 2, 3, ... enqueued back to back (b2k_bicgstab_chain): the scalar recurrences and both
            # convergence tests of each iteration run on the device; the host sees the batch once it stops
            nsteps = max(1, min(BICG_CHAIN_LEN, maxiter - numiter + 1))
            done = C.c_int32()
            ctx.check(ctx.lib.b2k_bicgstab_chain(ctx.h, operator.h, x.handle, r.handle, r_shadow.handle, p.handle,
                                                 v.handle, s.handle, t.handle, a0, a1, rho, rhoold, alpha, omega,
                                                 tol, nsteps, rec.ctypes.data_as(C.POINTER(C.c_double)),
                                                 C.byref(done)))
            d = done.value
            last = rec[d - 1]
            numiter += d - 1
            rho, alpha = float(last[0]), float(last[2])
            half_done = True
            if last[7] == 1.0:                   # ‖s‖ < tol: the full step of the last iteration has not run
                numops += 2 * d - 1
                normr = float(last[3])
            else:
                numops += 2 * d
                omega, normr, rho_next = float(last[4]), float(last[5]), float(last[6])
                full_done = True
        if first:
            if rho == 0.0:                       # `ρ ≈ 0.0` (bicgstab.jl:36): the method breaks down
                if alg.verbosity >= WARN_LEVEL:
                    warnings.warn("BiCGStab linsolve errored after 1 iteration: rho = 0")
                return x, ConvergenceInfo(0, r, normr, numiter, numops)
            beta = 0.0
        else:
            beta = (rho / rhoold) * (alpha / omega)
        if half_done:
            pass
        elif fused:
            if first:
                p, v = r.zerovector(), r.zerovector()
            sg, ns = C.c_double(), C.c_double()
            ctx.check(ctx.lib.b2k_bicgstab_half(ctx.h, operator.h, r_shadow.handle, r.handle, p.handle, v.handle,
                                                s.handle, a0, a1, beta, omega, rho, int(first),
                                                C.byref(sg), C.byref(ns)))
            numops += 1
            alpha = rho / sg.value
            normr = ns.value
        else:
            if first:
                p = r.copy()
            else:
                p = p.add_(v, -omega)
                p = p.add_(r, 1.0, beta)
            v, sigma = _apply_and_dot(operator, p, a0, a1, r_shadow)      # v = (a₀ + a₁A) p, σ = ⟨r̃, v⟩
            numops += 1
            alpha = rho / sigma
            s = s.scale_(1.0, r)
            s = s.add_(v, -alpha)                # half step residual
            xhalf = xhalf.scale_(1.0, x)
            xhalf = xhalf.add_(p, alpha)         # half step iterate
            normr = s.norm()
        if normr < tol and not full_done:
            # replace the recurrence residual by the actual one before trusting it
            if fused:
                xhalf = xhalf.scale_(1.0, x)
                xhalf = xhalf.add_(p, alpha)
            s = s.scale_(1.0, b)
            s = s.add_(apply(operator, xhalf, a0, a1), -1.0)
            numops += 1
            normr_act = s.norm()
            if normr_act < tol:
                return xhalf, ConvergenceInfo(1, s, normr_act, numiter, numops)
        if full_done:
            pass
        elif fused:
            om, nr, rn = C.c_double(), C.c_double(), C.c_double()
            ctx.check(ctx.lib.b2k_bicgstab_full(ctx.h, operator.h, x.handle, r.handle, r_shadow.handle, p.handle,
                                                s.handle, t.handle, a0, a1, alpha, C.byref(om), C.byref(nr),
                                                C.byref(rn)))
            numops += 1
            omega, normr, rho_next = om.value, nr.value, rn.value
        else:
            t, ts = _apply_and_dot(operator, s, a0, a1, s)                # t = (a₀ + a₁A) s, ⟨t, s⟩
            numops += 1
            omega = ts / t.inner(t)
            x = x.scale_(1.0, xhalf)
            x = x.add_(s, omega)                     # full step iterate
            r = r.scale_(1.0, s)
            r = r.add_(t, -omega)                    # full step residual
            del t
            normr = r.norm()
        if normr < tol:
            r = r.scale_(1.0, b)
            r = r.add_(apply(operator, x, a0, a1), -1.0)
            numops += 1
            rho_next = None                      # r changed: ⟨r̃, r⟩ has to be taken again
            normr_act = r.norm()
            if normr_act < tol:
                return x, ConvergenceInfo(1, r, normr_act, numiter, numops)
        if numiter > 1 and numiter >= maxiter:
            if alg.verbosity >= WARN_LEVEL:
                warnings.warn(f"BiCGStab linsolve stopped without converging after {numiter} iterations: "
                              f"normres = {normr}, numops = {numops}")
            return x, ConvergenceInfo(0, r, normr, numiter, numops)


USE_MINRES_CHAIN = True   # b2k_minres_chain: two launches per iteration, one host round trip per MINRES_CHAIN_LEN
MINRES_CHAIN_LEN = 32


def _minres_scalars(st, alpha: float, beta_new: float):
    """The Givens-QR half of one MINRES iteration, in the operation order of k_minres_step's last CTA (plain double
    arithmetic, every product and sum rounded on its own).  st = [β_k, 1/β_k, 1/β_{k-1}, c, s, δ̄, ε, φ̄] is advanced
    in place; returns the record (α, β_{k+1}, γ, φ, |φ̄|, stop code, δ, ε_k)."""
    c0, s0, dbar, eps, phibar = st[3], st[4], st[5], st[6], st[7]
    delta = c0 * dbar + s0 * alpha
    gbar = s0 * dbar - c0 * alpha
    gamma = math.sqrt(gbar * gbar + beta_new * beta_new)
    sing = gamma == 0.0
    c, s = (0.0, 0.0) if sing else (gbar / gamma, beta_new / gamma)
    phi = 0.0 if sing else c * phibar
    phibar_n = phibar if sing else s * phibar
    st[2], st[0], st[1] = st[1], beta_new, (1.0 / beta_new if beta_new != 0.0 else math.inf)
    st[3], st[4], st[5], st[6], st[7] = c, s, -(c0 * beta_new), s0 * beta_new, phibar_n
    return alpha, beta_new, gamma, phi, abs(phibar_n), (2.0 if sing else 0.0), delta, eps


def _minres(operator, b: B200Vec, x0: B200Vec, alg: MINRES, a0: float, a1: float):
    """linsolve(operator, b, x₀, alg::MINRES, a₀, a₁) for a real symmetric operator that need not be definite.  The
    reference declares the algorithm (src/algorithms.jl:397-427) and leaves the driver as a TODO
    (src/linsolve/linsolve.jl:140-141), so the recurrence is fixed here: Paige & Saunders (1975), unpreconditioned
    Lanczos + Givens QR, with the stopping rules of cg.jl:69-73 (a recurrence residual is never trusted: when |φ̄|
    < tol the residual is computed, and if it is not below tol the process restarts from the current x).
    A device CSR operator on one GPU runs b2k_minres_chain (the Lanczos vectors stay unnormalised, two launches
    per iteration, one host round trip per MINRES_CHAIN_LEN iterations); every other operator, and row-sharded
    contexts, run the literal VectorInterface sequence, which produces the same vectors given the same scalars."""
    import ctypes as C
    y0 = apply(operator, x0)
    r = b.copy()
    if a0 != 0:
        r = r.add_(x0, -a0)
    r = r.add_(y0, -a1)
    del y0
    x = x0.copy()
    normr = r.norm()
    maxiter, tol = alg.maxiter, alg.tol
    numops, numiter = 1, 0
    if normr < tol:
        return x, ConvergenceInfo(1, r, normr, numiter, numops)
    ctx = b.ctx
    chain = USE_MINRES_CHAIN and isinstance(operator, B200CSR) and ctx.nranks == 1
    d1, d2 = r.zerovector(), r.zerovector()
    if chain:       # p_cur = p_{k-1}, p_prev = p_{k-2}: the Lanczos vectors before normalisation (v_k = p_{k-1}/β_k)
        p_cur, p_prev, q = r.copy(), r.zerovector(), r.zerovector()
    else:
        v, v_prev = r.scale(1.0 / normr), r.zerovector()
    st = [normr, 1.0 / normr, 0.0, -1.0, 0.0, 0.0, 0.0, normr]
    pending: list = []            # records of iterations the device has already run, oldest first
    while True:
        if chain:
            if not pending:
                m = max(1, min(MINRES_CHAIN_LEN, maxiter - numiter))
                rec, done = np.zeros((m, 8)), C.c_int32()
                sin, sout = (C.c_double * 8)(*st), (C.c_double * 8)()
                ctx.check(ctx.lib.b2k_minres_chain(ctx.h, operator.h, x.handle, p_prev.handle, p_cur.handle, q.handle,
                                                   d1.handle, d2.handle, a0, a1, sin, tol, m,
                                                   rec.ctypes.data_as(C.POINTER(C.c_double)), sout, C.byref(done)))
                st = list(sout)
                if done.value & 1:                                   # the roles rotate once per iteration
                    p_prev, p_cur, d1, d2 = p_cur, p_prev, d2, d1
                pending = [rec[i] for i in range(done.value)]
            _, beta_new, gamma, _, phibar, _, _, _ = pending.pop(0)
        else:
            q = apply(operator, v, a0, a1)
            alpha = v.inner(q)
            q = q.add_(v, -alpha)
            q = q.add_(v_prev, -st[0])
            eps = st[6]
            _, beta_new, gamma, phi, phibar, _, delta, _ = _minres_scalars(st, alpha, q.norm())
            d = v_prev.scale_(1.0, v)                                # v_{k-1} has done its work: d_k takes its storage
            if gamma != 0.0:
                d = d.add_(d1, -delta)
                d = d.add_(d2, -eps)
                d = d.scale_(1.0 / gamma)
                x = x.add_(d, phi)
            else:
                d = d.zerovector_()
            d1, d2, v_prev = d, d1, v
            v = q.scale_(st[1]) if beta_new != 0.0 else q            # v_{k+1} = p_k/β_{k+1}
        numiter += 1
        numops += 1
        hit = phibar < tol or beta_new == 0.0
        if gamma == 0.0 or hit or numiter >= maxiter:
            r = r.scale_(1.0, b)
            r = r.add_(apply(operator, x, a0, a1), -1.0)
            numops += 1
            normr = r.norm()
            if gamma == 0.0:
                if alg.verbosity >= WARN_LEVEL:
                    warnings.warn(f"MINRES linsolve in iteration {numiter}: the operator is singular in the Krylov "
                                  f"subspace: normres = {normr}, numops = {numops}")
                return x, ConvergenceInfo(0, r, normr, numiter, numops)
            if hit and (normr < tol or normr == 0.0):               # (tol = 0: an exact solution still ends it)
                return x, ConvergenceInfo(1, r, normr, numiter, numops)
            if numiter >= maxiter:
                if alg.verbosity >= WARN_LEVEL:
                    warnings.warn(f"MINRES linsolve stopped without converging after {numiter} iterations: "
                                  f"normres = {normr}, numops = {numops}")
                return x, ConvergenceInfo(0, r, normr, numiter, numops)
            # the recurrence reported convergence and the residual does not confirm it: a fresh process from x
            if chain:
                p_cur, p_prev = p_cur.scale_(1.0, r), p_prev.zerovector_()
            else:
                v, v_prev = v.scale_(1.0 / normr, r), v_prev.zerovector_()
            d1, d2 = d1.zerovector_(), d2.zerovector_()
            st = [normr, 1.0 / normr, 0.0, -1.0, 0.0, 0.0, 0.0, normr]
