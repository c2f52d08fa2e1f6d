"""GPU tests of lssolve on a device CSR matrix: the chained iterations (b2k_lsmr_chain) against the literal
VectorInterface loop over the (A, Aᵀ) tuple and against the oracle — Float64 and Float32, with and without λ, every
orthogonalizer that chains; batches of N iterations against N batches of one, bit for bit; an exhausted Krylov space;
the refusals of the entry point and of the front end."""
import ctypes as C
import importlib

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

lsq = importlib.import_module("krylovkit_jl_b200.lssolve")
f64, f32 = np.float64, np.float32


def grad2d(nx, ny):
    """forward-difference gradient of an nx x ny grid: (nx(ny-1) + ny(nx-1)) x nx ny"""
    dx = sp.diags([-np.ones(nx - 1), np.ones(nx - 1)], [0, 1], shape=(nx - 1, nx))
    dy = sp.diags([-np.ones(ny - 1), np.ones(ny - 1)], [0, 1], shape=(ny - 1, ny))
    return sp.vstack([sp.kron(sp.eye(ny), dx), sp.kron(dy, sp.eye(nx))]).tocsr()


def rect(rng, m=3000, n=800, seed=4):
    return (sp.random(m, n, density=0.01, random_state=seed) + sp.eye(m, n)).tocsr()


def solve(A, b, alg, lam, dtype, tuple_path=False, **kw):
    """lssolve on the device: the B200CSR entry (chained), or the (A, Aᵀ) tuple (literal loop)"""
    m, n = A.shape
    ctx = kk.B200Context(m, 16, dtype=dtype)
    try:
        sv = ctx.add_space(n, max(alg.krylovdim, 1) + 12, sharded=False)
        Ad = kk.B200CSR.from_scipy(ctx, A.astype(dtype)).with_spaces(sv, 0)
        bd = ctx.from_host(b.astype(dtype))
        if tuple_path:
            At = kk.B200CSR.from_scipy(ctx, A.T.tocsr().astype(dtype)).with_spaces(0, sv)
            x, info = kk.lssolve((Ad, At), bd, alg, lam, **kw)
        else:
            x, info = kk.lssolve(Ad, bd, alg, lam, **kw)
        return x.to_host(), info.residual.to_host(), info
    finally:
        ctx.close()


ORTHS = [("mgs", 1), ("mgs", 5), ("mgs2", 5), ("cgs2", 5)]


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("lam", [0.0, 0.3])
@pytest.mark.parametrize("orth,K", ORTHS)
def test_chain_matches_literal_and_oracle(dtype, lam, orth, K):
    rng = np.random.default_rng(3)
    A = rect(rng)
    b = rng.random(A.shape[0])
    o = getattr(kk, orth)
    # fixed iteration count: the counts match exactly, the iterates to rounding
    alg = kk.LSMR(orth=o, maxiter=40, tol=0.0, krylovdim=K, verbosity=0)
    x, res, info = solve(A, b, alg, lam, dtype)
    xt, rest, infot = solve(A, b, alg, lam, dtype, tuple_path=True)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=40, tol=0.0, krylovdim=K, orth=ko.Orth(o.tag), lam=lam)
    assert (info.numiter, info.numops, info.converged) == (infot.numiter, infot.numops, infot.converged)
    assert info.numops == oinfo["numops"]
    rt = 1e-9 if dtype == f64 else 2e-3
    sc = np.linalg.norm(ox)
    assert np.linalg.norm(x - xt) <= rt * sc
    assert np.linalg.norm(x - ox) <= rt * sc
    # after 40 iterations |ζ̄| is near the rounding floor of the type: relative to ‖Aᵀb‖ in Float32
    if dtype == f64:
        np.testing.assert_allclose(info.normres, infot.normres, rtol=1e-4)
        np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-4)
    else:
        assert abs(info.normres - infot.normres) <= 1e-5 * np.linalg.norm(A.T @ b)
    # the recurrence residual is the explicit one
    r = b - A @ x.astype(f64)
    assert np.linalg.norm(res - r) <= (1e-10 if dtype == f64 else 1e-3) * np.linalg.norm(b)


@pytest.mark.parametrize("dtype", [f64, f32])
def test_chain_converges_grid_gradient(dtype):
    A = grad2d(60, 50)
    rng = np.random.default_rng(5)
    b = A @ rng.random(A.shape[1]) + 0.1 * rng.random(A.shape[0])
    tol = 1e-9 if dtype == f64 else 1e-4
    alg = kk.LSMR(maxiter=2000, tol=tol, krylovdim=8, verbosity=0)
    x, res, info = solve(A, b, alg, 0.0, dtype)
    xt, rest, infot = solve(A, b, alg, 0.0, dtype, tuple_path=True)
    assert info.converged == 1 and infot.converged == 1
    assert abs(info.numiter - infot.numiter) <= max(2, infot.numiter // 20)
    x = x.astype(f64)
    g = A.T @ (b - A @ x)
    assert np.linalg.norm(g) <= 20 * tol
    np.testing.assert_allclose(x, xt, rtol=0, atol=(1e-5 if dtype == f64 else 1e-1) * np.abs(xt).max())
    ox, oinfo = ko.lssolve_lsmr(A, b, maxiter=2000, tol=tol, krylovdim=8)
    assert np.linalg.norm(x - ox) <= (1e-5 if dtype == f64 else 1e-1) * np.linalg.norm(ox)
    # |zetabar| estimates ||A'(b - A x) - lambda^2 x||
    if dtype == f64:
        assert np.linalg.norm(g) <= 10 * info.normres + 1e-12 * np.linalg.norm(A.T @ b)


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("lam", [0.0, 0.2])
@pytest.mark.parametrize("orth,K", [("mgs", 1), ("mgs", 5), ("cgs2", 5)])
def test_batches_are_bit_identical(dtype, lam, orth, K, monkeypatch):
    """13 iterations in one call, in calls of one, and in calls of 4 — past the ring wrap — give the same bits"""
    rng = np.random.default_rng(7)
    A = rect(rng, 2000, 600, seed=8)
    b = rng.random(2000)
    alg = kk.LSMR(orth=getattr(kk, orth), maxiter=13, tol=0.0, krylovdim=K, verbosity=0)
    out = []
    for L_ in (13, 1, 4):
        monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", L_)
        x, res, info = solve(A, b, alg, lam, dtype)
        out.append((x, res, info.normres, info.numops))
    for x, res, nr, no in out[1:]:
        assert np.array_equal(x, out[0][0]) and np.array_equal(res, out[0][1])
        assert nr == out[0][2] and no == out[0][3]


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("lam", [0.0, 0.2])
def test_batch_converging_midway_equals_exact_batch(dtype, lam, monkeypatch):
    rng = np.random.default_rng(9)
    A = rect(rng, 2000, 600, seed=10)
    b = rng.random(2000)
    alg = kk.LSMR(maxiter=500, tol=1e-8 if dtype == f64 else 1e-3, krylovdim=4, verbosity=0)
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", 64)
    x, res, info = solve(A, b, alg, lam, dtype)
    assert info.converged == 1 and info.numiter < 64
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", info.numiter)
    x2, res2, info2 = solve(A, b, alg, lam, dtype)
    assert np.array_equal(x, x2) and np.array_equal(res, res2) and info2.numiter == info.numiter


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("K", [1, 5])
def test_exhausted_krylov_space_matches_literal(dtype, K):
    """A with three distinct singular values and b in its range: the bidiagonalisation ends after three steps
    (beta <= tol, the A' product skipped) and the chained and literal paths report the same counts"""
    rng = np.random.default_rng(11)
    m, n = 400, 120
    U, _ = np.linalg.qr(rng.standard_normal((m, n)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    s = np.repeat([3.0, 2.0, 1.0], n // 3)
    A = sp.csr_matrix(U @ np.diag(s) @ V.T)
    b = A @ rng.standard_normal(n)
    tol = 1e-6 if dtype == f64 else 1e-2
    alg = kk.LSMR(orth=kk.mgs, maxiter=10, tol=tol, krylovdim=K, verbosity=0)
    x, res, info = solve(A, b, alg, 0.0, dtype)
    xt, rest, infot = solve(A, b, alg, 0.0, dtype, tuple_path=True)
    assert (info.numiter, info.numops, info.converged) == (infot.numiter, infot.numops, infot.converged)
    np.testing.assert_allclose(x, xt, rtol=0, atol=(1e-8 if dtype == f64 else 1e-3) * np.abs(xt).max())


@pytest.mark.parametrize("kind", ["beta", "alpha"])
@pytest.mark.parametrize("orth,K", [("mgs", 1), ("mgs", 4), ("cgs2", 4)])
def test_breakdown_then_literal_loop_matches_tuple_path(kind, orth, K):
    """the chain stops at a beta (code 2) or alpha (code 3) breakdown with |zetabar| > tol (test_gpu_lsmr_kernel checks
    the codes) and the literal loop finishes: the counts of the tuple path, x to rounding (an alpha breakdown leaves v
    unnormalised, so later iterates amplify rounding, in the reference too)"""
    from test_gpu_lsmr_kernel import breakdown_problem
    A, b = breakdown_problem(kind)
    alg = kk.LSMR(orth=getattr(kk, orth), maxiter=30, tol=1e-8, krylovdim=K, verbosity=0)
    x, res, info = solve(A, b, alg, 0.0, f64)
    xt, rest, infot = solve(A, b, alg, 0.0, f64, tuple_path=True)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=30, tol=1e-8, krylovdim=K, orth=ko.Orth(getattr(kk, orth).tag))
    assert info.converged == infot.converged == oinfo["converged"] == 1
    assert abs(info.numiter - infot.numiter) <= 1 and abs(info.numops - infot.numops) <= 2
    tolx = 1e-8 if kind == "beta" else 5e-2
    assert np.linalg.norm(x - xt) <= tolx * np.linalg.norm(xt)
    assert np.linalg.norm(x - ox) <= tolx * np.linalg.norm(ox)


@pytest.mark.parametrize("case", ["long_row", "compact"])
def test_parity_long_rows_and_compact_copy(case):
    """a row longer than the 1536-nonzero SpMV tile (A and A' both), and a matrix the compact CSR copy takes"""
    rng = np.random.default_rng(17)
    if case == "long_row":
        A = rect(rng, 3000, 2500, seed=18).tolil()
        A[5, :] = rng.standard_normal(2500)           # a 2500-nonzero row of A
        A[:, 7] = rng.standard_normal((3000, 1))      # a 3000-nonzero row of A'
        A = A.tocsr()
    else:
        A = grad2d(40, 30)                            # +-1 values, short column offsets
    A.sort_indices()
    b = rng.random(A.shape[0])
    alg = kk.LSMR(orth=kk.mgs, maxiter=30, tol=0.0, krylovdim=5, verbosity=0)
    x, res, info = solve(A, b, alg, 0.25, f64)
    xt, rest, infot = solve(A, b, alg, 0.25, f64, tuple_path=True)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=30, tol=0.0, krylovdim=5, lam=0.25)
    assert (info.numiter, info.numops) == (infot.numiter, infot.numops) == (oinfo["numiter"], oinfo["numops"])
    assert np.linalg.norm(x - xt) <= 1e-9 * np.linalg.norm(ox)
    assert np.linalg.norm(x - ox) <= 1e-9 * np.linalg.norm(ox)
    np.testing.assert_allclose(res, b - A @ x, atol=1e-10 * np.linalg.norm(b))


def test_front_end_refusals():
    ctx = kk.B200Context(64, 8)
    try:
        b = ctx.from_host(np.ones(64))
        with pytest.raises(L.B200Error, match="matrix-free"):
            kk.lssolve(kk.B200CSR.stencil_free(ctx, 8, 8), b, kk.LSMR(verbosity=0))
        sv = ctx.add_space(16, 8, sharded=False)
        A = kk.B200CSR.from_scipy(ctx, sp.random(64, 16, density=0.2, random_state=1).tocsr())
        with pytest.raises(ValueError, match="carry its spaces"):
            kk.lssolve(A, b, kk.LSMR(verbosity=0))
        D = kk.B200Dense.from_host(ctx, np.ones((64, 16)), sv)
        fake = object.__new__(kk.B200CSR)            # a dense operator handle dressed as a B200CSR
        fake.ctx, fake.h, fake.n_rows, fake.n_cols = ctx, D.h, 64, 16
        fake.space_in, fake.space_out, fake._explicit_spaces = sv, 0, True
        with pytest.raises(L.B200Error, match="not a stored CSR matrix"):
            kk.lssolve(fake, b, kk.LSMR(verbosity=0))
    finally:
        ctx.close()


def _chain_call(ctx, A, At, vecs, ring, K, alg, nsteps=2, iter0=0):
    state = (C.c_double * 10)(1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0, 0.0, 1.0, 0.0)
    out = (C.c_double * 10)()
    rec = (C.c_double * (16 * 600))()
    done = C.c_int32(-1)
    rh = (L.c_vec * len(ring))(*[v.handle for v in ring])
    return ctx.lib.b2k_lsmr_chain(ctx.h, A.h, At.h, *[v.handle for v in vecs[:8]], rh, K, vecs[8].handle, alg,
                                  iter0, state, 0.0, nsteps, rec, out, C.byref(done)), done.value


def test_entry_refusals_write_nothing():
    rng = np.random.default_rng(13)
    m, n = 300, 100
    ctx = kk.B200Context(m, 16)
    try:
        sv = ctx.add_space(n, 16, sharded=False)
        M = rect(rng, m, n, seed=14)
        A = kk.B200CSR.from_scipy(ctx, M).with_spaces(sv, 0)
        At = A.transpose()
        Wrong = kk.B200CSR.from_scipy(ctx, M)          # not A's transpose
        nvec = [ctx.from_host(rng.random(n), sv) for _ in range(3)]         # x, h, hbar
        mvec = [ctx.from_host(rng.random(m)) for _ in range(5)]             # r, Ah, Ahbar, u, av
        ring = [ctx.from_host(rng.random(n), sv) for _ in range(3)]
        spare = ctx.from_host(rng.random(n), sv)
        sv2 = ctx.add_space(n, 2, sharded=False)
        other = ctx.from_host(rng.random(n), sv2)       # right length, another space
        St = kk.B200CSR.stencil_free(ctx, 30, 10)      # 300 points: the length of space 0
        vecs = nvec + mvec + [spare]
        before = [v.to_host().copy() for v in vecs + ring]
        cases = [
            (dict(K=3, alg=L.CGSIR), L.ENOTSUP),
            (dict(K=3, alg=L.MGS, nsteps=0), L.EINVAL),
            (dict(K=3, alg=L.MGS, nsteps=512), L.EINVAL),
            (dict(K=3, alg=L.MGS, A=At, At=A), L.EDIM),
            (dict(K=3, alg=L.MGS, At=Wrong), L.EDIM),
            (dict(K=3, alg=L.MGS, vecs=nvec + mvec[:4] + [mvec[0]] + [spare]), L.EINVAL),
            (dict(K=3, alg=L.MGS, vecs=mvec[:3] + mvec + [spare]), L.EDIM),
            (dict(K=3, alg=L.MGS, vecs=nvec[:2] + [other] + mvec + [spare]), L.EDIM),
            (dict(K=3, alg=L.MGS, A=St, At=St), L.ENOTSUP),
            (dict(K=129, alg=L.MGS), L.ENOTSUP),
        ]
        for kw, code in cases:
            st, _ = _chain_call(ctx, kw.get("A", A), kw.get("At", At), kw.get("vecs", vecs), ring, kw["K"],
                                kw["alg"], kw.get("nsteps", 2))
            assert st == code, (kw, st)
        for v, w in zip(vecs + ring, before):
            assert np.array_equal(v.to_host(), w)
    finally:
        ctx.close()
