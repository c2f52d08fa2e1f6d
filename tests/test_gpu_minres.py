"""GPU tests of linsolve(MINRES): the chained driver (b2k_minres_chain) and the literal VectorInterface sequence on
symmetric indefinite systems against the float64 restatement (tests/minres_oracle.py) — convergence, the explicit
residual, the counts — in Float64 and Float32, with a shift, with a starting vector, through the host entry, and one
full-size run."""
import importlib

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from oracle import krylov_oracle as ko

import minres_oracle as mo

ls = importlib.import_module("krylovkit_jl_b200.linsolve")
f64, f32 = np.float64, np.float32


def laplace_shift(nx, ny):
    """σ in the middle of the widest gap between neighbouring eigenvalues in the lower third of the spectrum (past the
    first 50): indefinite, nonsingular, and as well conditioned as a shift inside this spectrum gets"""
    lam = np.unique(np.round(ko.laplace_eigenvalues(nx, ny), 12))
    g = np.diff(lam[:len(lam) // 3])
    j = int(np.argmax(g[50:])) + 50
    return 0.5 * (lam[j] + lam[j + 1])


def random_coupling(n, per_row, seed):
    """n x n sparse matrix with about per_row random entries per row (index pairs drawn directly: scipy.sparse.random
    permutes all n² positions)"""
    rng = np.random.default_rng(seed)
    k = int(per_row * n)
    return sp.coo_matrix((rng.uniform(0.0, 1.0, k), (rng.integers(0, n, k), rng.integers(0, n, k))), shape=(n, n)).tocsr()


def random_indefinite(n, seed=1):
    """diagonal of both signs, |d| in [1, 2], plus a weak symmetric coupling: converges in a few dozen iterations"""
    rng = np.random.default_rng(seed)
    R = random_coupling(n, 2, seed)
    d = rng.uniform(1.0, 2.0, n) * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    A = (sp.diags(d) + 0.05 * (R + R.T)).tocsr()
    A.sort_indices()
    return A, rng.standard_normal(n)


def run(op_of, n, b, dt, tol, maxiter, chain, a0=0.0, a1=1.0, x0=None):
    saved = ls.USE_MINRES_CHAIN
    ls.USE_MINRES_CHAIN = chain
    try:
        ctx = kk.B200Context(n, 12, dtype=dt)
        op = op_of(ctx)
        bv = ctx.from_host(b.astype(dt))
        xv = ctx.from_host(x0.astype(dt)) if x0 is not None else None
        x, info = kk.linsolve(op, bv, xv, kk.MINRES(maxiter=maxiter, tol=tol, verbosity=0), a0, a1)
        out = x.to_host().astype(f64), info.residual.to_host().astype(f64), info
        ctx.close()
        return out
    finally:
        ls.USE_MINRES_CHAIN = saved


@pytest.mark.parametrize("dt,rtol", [(f64, 1e-10), (f32, 1e-4)])
def test_shifted_laplacian(dt, rtol):
    nx, ny = 200, 150
    n = nx * ny
    sigma = laplace_shift(nx, ny)
    A = ko.stencil_matrix(nx, ny)
    b = ko.splitmix_vector(11, n)
    tol = rtol * np.linalg.norm(b)
    res = {}
    for chain in (True, False):
        x, r, info = run(lambda c: kk.B200CSR.stencil(c, nx, ny), n, b, dt, tol, 40000, chain, a0=-sigma)
        assert info.converged == 1 and info.normres < tol
        true = np.linalg.norm(b.astype(dt).astype(f64) - (A @ x - sigma * x))
        assert true < tol * (1.0 + (1e-6 if dt == f64 else 0.5))
        assert np.linalg.norm(r) == pytest.approx(info.normres, rel=1e-5)
        res[chain] = info
    # thousands of iterations on a system this close to singular: the last bits of α and β (per-CTA sums in the
    # fused path) move the count by a little; both drivers solve the same problem in about the same number
    assert abs(res[True].numiter - res[False].numiter) <= 0.05 * res[False].numiter
    assert res[True].numops >= res[True].numiter + 2


@pytest.mark.parametrize("dt,rtol", [(f64, 1e-10), (f32, 1e-4)])
@pytest.mark.parametrize("variant", ["plain", "shift", "x0"])
def test_random_indefinite_counts_match_the_oracle(dt, rtol, variant):
    n = 200000
    A, b = random_indefinite(n)
    a0, a1 = (0.3, -1.7) if variant == "shift" else (0.0, 1.0)
    x0 = np.random.default_rng(9).standard_normal(n) if variant == "x0" else None
    Ad, bd = A.astype(dt), b.astype(dt).astype(f64)
    tol = rtol * np.linalg.norm(b)
    o = mo.minres(Ad.astype(f64), bd, None if x0 is None else x0.astype(dt).astype(f64), a0, a1, tol=tol, maxiter=500)
    assert o.converged == 1
    infos = []
    for chain in (True, False):
        x, r, info = run(lambda c: kk.B200CSR.from_scipy(c, Ad), n, b, dt, tol, 500, chain, a0, a1, x0)
        assert info.converged == 1 and info.normres < tol
        slack = 0 if dt == f64 else 1                    # Float32: a last-bit difference can move the exit by one
        assert abs(info.numiter - o.numiter) <= slack and abs(info.numops - o.numops) <= slack
        assert np.linalg.norm(bd - (a0 * x + a1 * (Ad.astype(f64) @ x))) < tol * (1.0 + (1e-6 if dt == f64 else 0.5))
        assert np.linalg.norm(x - o.x) <= (1e-9 if dt == f64 else 1e-3) * np.linalg.norm(o.x)
        infos.append(info)
    assert abs(infos[0].numiter - infos[1].numiter) <= slack


def test_host_entry():
    A, b = random_indefinite(5000, seed=2)
    x, info = kk.linsolve(A, b, alg=kk.MINRES(maxiter=300), rtol=1e-9)
    assert info.converged == 1 and np.linalg.norm(b - A @ x) < 1e-9 * np.linalg.norm(b) * (1 + 1e-6)


def test_full_size_shifted_laplacian():
    """4000 x 2500 grid, σ inside the spectrum, 300 iterations: |φ̄| decreases monotonically and — no restart having
    happened — is the norm of the explicit residual the driver returns"""
    import ctypes as C
    nx, ny = 4000, 2500
    n = nx * ny
    sigma = laplace_shift(nx, ny)
    ctx = kk.B200Context(n, 20)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    b = ctx.splitmix(20260923)
    beta1 = b.norm()
    v = {k: ctx.zeros() for k in ("x", "p_prev", "p_cur", "q", "d1", "d2")}
    v["p_cur"].scale_(1.0, b)
    st, phibars = mo.fresh_state(beta1), []
    for _ in range(10):
        rec, done = np.zeros((30, 8)), C.c_int32()
        sin, sout = (C.c_double * 8)(*st), (C.c_double * 8)()
        ctx.check(ctx.lib.b2k_minres_chain(ctx.h, op.h, *[v[k].handle for k in ("x", "p_prev", "p_cur", "q", "d1", "d2")],
                                           -sigma, 1.0, sin, 0.0, 30, rec.ctypes.data_as(C.POINTER(C.c_double)), sout,
                                           C.byref(done)))
        assert done.value == 30          # (an even count: the roles are back where they were)
        st = list(sout)
        phibars += list(rec[:, 4])
    assert np.all(np.diff([beta1] + phibars) <= 0) and phibars[-1] < beta1
    r = b.copy().add_(kk.apply(op, v["x"], -sigma, 1.0), -1.0)
    assert r.norm() == pytest.approx(phibars[-1], rel=1e-6)
    del r, v
    x, info = kk.linsolve(op, b, None, kk.MINRES(maxiter=300, tol=0.0, verbosity=0), -sigma, 1.0)
    assert (info.converged, info.numiter, info.numops) == (0, 300, 302)
    assert info.normres == pytest.approx(phibars[-1], rel=1e-6)
    ctx.close()
