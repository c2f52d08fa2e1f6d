"""linsolve(MINRES) without a GPU: the float64 restatement (tests/minres_oracle.py) against truth and against
scipy.sparse.linalg.minres, and the driver — literal VectorInterface sequence and b2k_minres_chain batches — on the numpy
stand-in of the C-ABI (tests/hostsim_minres.py) against that restatement: equal numiter, numops and converged, the
stopping branches, the slab bookkeeping, the entry forms."""
import importlib
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import hostsim
import hostsim_minres
import minres_oracle as mo

ls = importlib.import_module("krylovkit_jl_b200.linsolve")      # (the package exports the function under this name)


@pytest.fixture()
def sim():
    with hostsim_minres.installed() as lib:
        yield lib
    assert not isinstance(L._lib, hostsim.HostSimLib)


@pytest.fixture(params=["literal", "chain"])
def mode(request, monkeypatch):
    monkeypatch.setattr(ls, "USE_MINRES_CHAIN", request.param == "chain")
    return request.param


def dense_indefinite(seed, n=100, cond=1e4, spd=False):
    """symmetric with prescribed eigenvalues of both signs (or all positive), |λ| in [1/cond, 1]"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.exp(rng.uniform(np.log(1.0 / cond), 0.0, n))
    if not spd:
        lam[::2] *= -1.0
    A = (Q * lam) @ Q.T
    return sp.csr_matrix((A + A.T) / 2), rng.standard_normal(n)      # CSR: the oracle and the stand-in sum rows alike


def shifted_laplacian(nx=30, ny=20):
    """(A, σ) with σ halfway between two neighbouring distinct eigenvalues in the lower part of the spectrum"""
    lam = np.unique(np.round(ko.laplace_eigenvalues(nx, ny), 12))
    k = len(lam) // 5
    return ko.stencil_matrix(nx, ny), 0.5 * (lam[k] + lam[k + 1])


def sparse_indefinite(seed, n=300):
    rng = np.random.default_rng(seed)
    R = sp.random(n, n, density=0.02, random_state=seed)
    d = rng.uniform(0.5, 2.0, n) * np.where(np.arange(n) % 3 == 0, -1.0, 1.0)
    return (sp.diags(d) + 0.05 * (R + R.T)).tocsr(), rng.standard_normal(n)


CASES = {
    "dense-indef": lambda: (*dense_indefinite(1), 0.0, 1.0, None),
    "dense-1e6": lambda: (*dense_indefinite(2, n=60, cond=1e6), 0.0, 1.0, None),
    "dense-spd": lambda: (*dense_indefinite(3, spd=True), 0.0, 1.0, None),
    "laplace-shift": lambda: (shifted_laplacian()[0], ko.splitmix_vector(7, 600), -shifted_laplacian()[1], 1.0, None),
    "x0": lambda: (*dense_indefinite(4), 0.0, 1.0, np.random.default_rng(5).standard_normal(100)),
    "a0a1": lambda: (*dense_indefinite(6), 0.3, -1.7, None),
}


# ---- the restatement against truth and scipy --------------------------------------------------------------------

@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_against_truth_and_scipy(case):
    A, b, a0, a1, x0 = CASES[case]()
    tol = 1e-9 * np.linalg.norm(b)
    o = mo.minres(A, b, x0, a0, a1, tol=tol, maxiter=20000, keep_iterates=True)
    assert o.converged == 1 and (o.restarts == 0 or case == "dense-1e6")
    M = a0 * np.eye(len(b)) + a1 * (A.toarray() if sp.issparse(A) else A)
    assert np.linalg.norm(b - M @ o.x) < tol and o.normres < tol
    assert o.restarts > 0 or np.all(np.diff(o.phibars) <= 0)       # (a restart starts again from the true residual)
    assert o.numops == o.numiter + 2 + o.restarts
    # early iterates: once the Lanczos vectors lose orthogonality two correct implementations drift apart
    for k in (1, 2, 5, 10):
        xs, _ = spl.minres(M, b, x0=x0, rtol=0.0, maxiter=k)
        assert np.linalg.norm(xs - o.iterates[k - 1]) <= 1e-10 * np.linalg.norm(xs), k


# ---- the driver on the stand-in ---------------------------------------------------------------------------------

def solve(sim, A, b, x0=None, a0=0.0, a1=1.0, dtype=np.float64, **kw):
    n = len(b)
    ctx = kk.B200Context(n, 12, dtype=dtype)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    used = sim.b2k_debug_used_columns(ctx.h, 0)
    xv = ctx.from_host(x0) if x0 is not None else None
    x, info = kk.linsolve(op, ctx.from_host(b), xv, kk.MINRES(**kw), a0, a1)
    out = x.to_host(), info.residual.to_host(), info
    del x, xv
    info.residual = None
    assert sim.b2k_debug_used_columns(ctx.h, 0) == used        # every work vector went back to the slab
    ctx.close()
    return out


@pytest.mark.parametrize("case", sorted(CASES))
def test_driver_matches_oracle(sim, mode, case):
    A, b, a0, a1, x0 = CASES[case]()
    tol = 1e-9 * np.linalg.norm(b)
    o = mo.minres(A, b, x0, a0, a1, tol=tol, maxiter=20000)
    x, r, info = solve(sim, A, b, x0, a0, a1, tol=tol, maxiter=20000, verbosity=0)
    assert (info.numiter, info.numops, info.converged) == (o.numiter, o.numops, o.converged)
    assert np.linalg.norm(x - o.x) <= 1e-12 * np.linalg.norm(o.x) * max(1.0, 1e-4 * o.numiter ** 2)
    M = a0 * sp.identity(len(b)) + a1 * sp.csr_matrix(A)
    np.testing.assert_allclose(r, b - M @ x, atol=1e-13 * np.linalg.norm(b))
    assert info.normres == pytest.approx(np.linalg.norm(r), rel=1e-12) and info.normres < tol
    assert sim.minres_calls == (0 if mode == "literal" else -(-o.numiter // ls.MINRES_CHAIN_LEN))


def test_chain_equals_literal_and_batch_boundaries_change_nothing(sim, monkeypatch):
    A, b = sparse_indefinite(11)
    tol = 1e-10 * np.linalg.norm(b)
    monkeypatch.setattr(ls, "USE_MINRES_CHAIN", False)
    xl, _, il = solve(sim, A, b, tol=tol, maxiter=500)
    monkeypatch.setattr(ls, "USE_MINRES_CHAIN", True)
    xs = []
    for m in (1, 3, 32):
        monkeypatch.setattr(ls, "MINRES_CHAIN_LEN", m)
        x, _, info = solve(sim, A, b, tol=tol, maxiter=500)
        assert (info.numiter, info.numops, info.converged) == (il.numiter, il.numops, 1)
        xs.append(x)
    assert np.array_equal(xs[0], xs[1]) and np.array_equal(xs[0], xs[2])
    assert np.max(np.abs(xs[0] - xl)) <= 16 * np.finfo(float).eps * np.max(np.abs(xl))


def test_float32(sim, mode):
    A, b = sparse_indefinite(12)
    tol = 1e-4 * np.linalg.norm(b)
    x, _, info = solve(sim, A.astype(np.float32), b.astype(np.float32), dtype=np.float32, tol=tol, maxiter=500)
    assert info.converged == 1 and x.dtype == np.float32
    assert np.linalg.norm(b - A @ x) < 1.01 * tol


def test_maxiter_warns(sim, mode):
    A, b = dense_indefinite(1)
    o = mo.minres(A, b, tol=1e-12, maxiter=7)
    with pytest.warns(UserWarning, match="without converging after 7 iterations"):
        x, _, info = solve(sim, A, b, tol=1e-12, maxiter=7)
    assert (info.converged, info.numiter, info.numops) == (0, 7, 9) == (o.converged, o.numiter, o.numops)
    assert info.normres == pytest.approx(np.linalg.norm(b - A @ x), rel=1e-10)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        solve(sim, A, b, tol=1e-12, maxiter=7, verbosity=0)


def test_zero_residual_start(sim, mode):
    A, b = dense_indefinite(1)
    x0 = np.linalg.solve(A.toarray(), b)
    x, _, info = solve(sim, A, b, x0=x0, tol=1e-8)
    assert (info.converged, info.numiter, info.numops) == (1, 0, 1) and np.array_equal(x, x0)


def test_lucky_breakdown(sim, mode):
    A = np.diag([2.0, -3.0, 5.0, 7.0])
    b = np.array([0.0, 4.0, 0.0, 0.0])               # an eigenvector: β₂ = 0 after one iteration
    x, _, info = solve(sim, A, b, tol=1e-12)
    assert (info.converged, info.numiter, info.numops) == (1, 1, 3)
    np.testing.assert_allclose(x, [0.0, -4.0 / 3.0, 0.0, 0.0], rtol=1e-15)
    x, _, info = solve(sim, A, b, tol=0.0, maxiter=3)        # |φ̄| = 0 is not < 0: β₂ == 0 and a zero residual end it
    assert (info.converged, info.numiter, info.normres) == (1, 1, 0.0) and np.all(np.isfinite(x))


def test_singular_operator(sim, mode):
    A = np.diag([1.0, 0.0, 2.0])
    b = np.array([0.0, 1.0, 0.0])                    # in the null space: not in the range
    o = mo.minres(A, b, tol=1e-12)
    assert o.singular and o.converged == 0
    with pytest.warns(UserWarning, match="singular"):
        x, _, info = solve(sim, A, b, tol=1e-12)
    assert (info.converged, info.numiter, info.numops) == (0, o.numiter, o.numops) == (0, 1, 3)
    assert np.array_equal(x, np.zeros(3)) and info.normres == 1.0


def test_false_convergence_restarts(sim, monkeypatch):
    monkeypatch.setattr(ls, "USE_MINRES_CHAIN", True)
    A, b = sparse_indefinite(13)
    tol = 1e-10 * np.linalg.norm(b)
    _, _, honest = solve(sim, A, b, tol=tol, maxiter=500)
    sim.minres_lie = (1, 1e-6)                       # one convergence test sees a |φ̄| a million times too small
    x, _, info = solve(sim, A, b, tol=tol, maxiter=500)
    assert sim.minres_lie[0] == 0
    assert info.converged == 1 and np.linalg.norm(b - A @ x) < tol
    assert info.numops == info.numiter + 3 and info.numiter != honest.numiter     # one extra explicit residual


def test_host_entry_and_tolerances(sim, mode):
    A, b = sparse_indefinite(14)
    x, info = kk.linsolve(A, b, alg=kk.MINRES(maxiter=500), rtol=1e-8)
    assert isinstance(x, np.ndarray) and info.converged == 1
    assert np.linalg.norm(b - A @ x) < 1e-8 * np.linalg.norm(b)
    assert isinstance(info.residual, np.ndarray)
    x2, info2 = kk.linsolve(A, b, alg=kk.MINRES(maxiter=500, tol=1e-8 * np.linalg.norm(b)))
    assert info2.numiter == info.numiter
    with pytest.raises(TypeError):
        kk.linsolve(A, b, alg=kk.MINRES(), krylovdim=3)


def test_callable_and_dense_operators_take_the_literal_path(sim):
    A, b = dense_indefinite(8, n=40)
    ctx = kk.B200Context(40, 12)
    csr = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    bv = ctx.from_host(b)
    x, info = kk.linsolve(lambda v: kk.apply(csr, v), bv, None, kk.MINRES(tol=1e-9, maxiter=400))
    assert info.converged == 1 and sim.minres_calls == 0
    assert np.linalg.norm(b - A @ x.to_host()) < 1e-9
    ctx.close()


def test_algorithm_struct_and_selector():
    alg = kk.MINRES()
    assert (alg.maxiter, alg.tol, alg.verbosity) == (kk.KrylovDefaults.maxiter, kk.KrylovDefaults.tol,
                                                     kk.KrylovDefaults.verbosity)
    with pytest.raises(Exception):
        alg.tol = 1.0
    A, b = sparse_indefinite(15)
    sel = kk.linselector(A, b, issymmetric=True, isposdef=False)
    assert isinstance(sel, kk.GMRES)                  # the reference's choice for symmetric indefinite input
    assert isinstance(kk.linselector(A, b, issymmetric=True, isposdef=True), kk.CG)


# ---- the stand-in's refusals are the library's ------------------------------------------------------------------

def test_chain_refusals(sim):
    import ctypes as C
    n = 30
    A, _ = sparse_indefinite(16, n)
    ctx = kk.B200Context(n, 12)
    op = kk.B200CSR.from_scipy(ctx, A)
    dense = kk.B200Dense.from_host(ctx, np.eye(n), ctx.add_space(n, 2, sharded=False))
    vs = [ctx.full(float(i + 1)) for i in range(6)]
    other = ctx.add_space(n + 1, 2)
    long = ctx.zeros(other)
    st, out, rec, done = (C.c_double * 8)(1, 1, 0, -1, 0, 0, 0, 1), (C.c_double * 8)(), (C.c_double * 8)(), C.c_int32(7)

    def call(o, hs, nsteps=1):
        return sim.b2k_minres_chain(ctx.h, o, *hs, 0.0, 1.0, st, 0.0, nsteps, rec, out, C.byref(done))

    hs = [v.handle for v in vs]
    assert call(op.h, hs, 0) == L.EINVAL
    assert call(dense.h, hs) == L.ENOTSUP
    assert call(op.h, hs[:5] + [long.handle]) == L.EDIM
    assert call(op.h, hs[:5] + [hs[1]]) == L.EINVAL
    assert done.value == 7 and all(np.array_equal(v.to_host(), np.full(n, i + 1.0)) for i, v in enumerate(vs))
    assert call(op.h, hs) == L.OK and done.value == 1
    ctx.close()
