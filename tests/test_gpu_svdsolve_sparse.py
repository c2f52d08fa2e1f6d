"""End-to-end GPU tests of svdsolve on sparse matrices of about 2e5 rows: the scipy sparse host entry and the B200CSR
device entry (A' built on the device, the expansions chained by b2k_gkl_expand_many), Float64.

  * a tall and a wide random matrix (index pairs drawn directly: scipy.sparse.random is too slow at this size) and the
    Dirichlet forward-difference gradient G of an nx x ny grid, whose singular values are
    sqrt(4 sin^2(pi i / 2(nx+1)) + 4 sin^2(pi j / 2(ny+1)));
  * sigma against the oracle's step-by-step svdsolve at 1e-10 relative with equal numiter / numops, against
    scipy.sparse.linalg.svds, and against the closed form for the gradient;
  * ||A'u - sigma v|| and ||A v - sigma u - residual|| at the level of the dense test (test_gpu_solvers.py);
  * the same problem through the literal (A, At) tuple path: equal numops and numiter, sigma equal to rounding.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from oracle import krylov_oracle as ko


def random_sparse(m, n, per_row, seed):
    """per_row entries in every row, the columns (tall) or rows (wide) scaled by 1/sqrt(1 + j) so that the largest
    singular values are separated and GKL converges in a few restarts"""
    rng = np.random.default_rng(seed)
    nnz = per_row * m
    A = sp.csr_matrix((rng.standard_normal(nnz), (np.repeat(np.arange(m), per_row), rng.integers(0, n, nnz))),
                      shape=(m, n))
    A.sum_duplicates()
    if m >= n:
        return (A @ sp.diags(1 / np.sqrt(1.0 + np.arange(n)))).tocsr()
    return (sp.diags(1 / np.sqrt(1.0 + np.arange(m))) @ A).tocsr()


def gradient(nx, ny):
    def d1(k):          # (k + 1) x k forward difference with Dirichlet ends
        return sp.diags([np.ones(k), -np.ones(k)], [0, -1], shape=(k + 1, k))
    return sp.vstack([sp.kron(sp.identity(ny), d1(nx)), sp.kron(d1(ny), sp.identity(nx))]).tocsr()


def gradient_sigmas(nx, ny):
    sx = 4 * np.sin(np.pi * np.arange(1, nx + 1) / (2 * (nx + 1))) ** 2
    sy = 4 * np.sin(np.pi * np.arange(1, ny + 1) / (2 * (ny + 1))) ** 2
    return np.sort(np.sqrt((sx[:, None] + sy[None, :]).ravel()))[::-1]


# builder, howmany, tol, krylovdim.  The gradient's largest singular values are clustered (relative gaps ~1e-5), so it
# asks for one value to 1e-6 (a Ritz value error of ~ normres^2 / gap, far below the 1e-7 the closed form is held to).
CASES = {
    "tall": (lambda: random_sparse(200000, 5000, 8, seed=1), 4, 1e-10, 30),
    "wide": (lambda: random_sparse(20000, 200000, 60, seed=2), 4, 1e-10, 30),
    "gradient": (lambda: gradient(300, 330), 1, 1e-6, 40),
}


def check_triplets(A, S, U, V, res, tol):
    for s, u, v, r in zip(S, U, V, res):
        assert np.linalg.norm(A.T @ u - s * v) < tol
        assert np.linalg.norm(A @ v - s * u - r) < tol


@pytest.mark.parametrize("orth", ["cgs2", "mgs2b"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_host_sparse_entry(case, orth):
    build, how, tol, kd = CASES[case]
    A = build()
    m, n = A.shape
    u0 = ko.splitmix_vector(2026, m)
    alg = kk.GKL(orth=kk.cgs2 if orth == "cgs2" else kk.mgs2b, krylovdim=kd, maxiter=300, tol=tol, verbosity=0)
    S, U, V, info = kk.svdsolve(A, u0, how, "LR", alg)
    assert info.converged >= how
    oS, _, _, oinfo = ko.svdsolve_gkl(A, u0, how, "LR", krylovdim=kd, maxiter=300, tol=tol,
                                      orth=ko.Orth(ko.CGS2 if orth == "cgs2" else ko.MGS2))
    np.testing.assert_allclose(S[:how], oS[:how], rtol=1e-10)
    if orth == "cgs2":          # the oracle has no MGS2B: its MGS2 takes the same steps, not necessarily as many
        assert (info.numiter, info.numops) == (oinfo["numiter"], oinfo["numops"])
    if case == "gradient":
        np.testing.assert_allclose(S[:how], gradient_sigmas(300, 330)[:how], rtol=1e-7)
    else:
        ref = spl.svds(A, k=how, which="LM", return_singular_vectors=False, tol=1e-12, random_state=0)
        np.testing.assert_allclose(S[:how], np.sort(ref)[::-1], rtol=1e-9)
    check_triplets(A, S[:how], U, V, info.residual, 1e-8 * max(1.0, S[0]))


@pytest.mark.parametrize("case", ["tall", "gradient"])
def test_device_entry_matches_tuple_path(case):
    build, how, tol, kd = CASES[case]
    A = build()
    m, n = A.shape
    u0 = ko.splitmix_vector(7, m)
    ctx = kk.B200Context(m, 3 * kd + 14)
    try:
        sv = ctx.add_space(n, 2 * kd + 14, sharded=False)
        op = kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        opt = kk.B200CSR.from_scipy(ctx, A.T.tocsr()).with_spaces(0, sv)
        alg = kk.GKL(orth=kk.cgs2, krylovdim=kd, maxiter=300, tol=tol, verbosity=0)
        launches = ctx.launches
        S1, U1, V1, i1 = kk.svdsolve(op, ctx.from_host(u0), how, "LR", alg)
        l_chain = ctx.launches - launches
        launches = ctx.launches
        S2, _, _, i2 = kk.svdsolve((op, opt), ctx.from_host(u0), how, "LR", alg)
        l_tuple = ctx.launches - launches
        assert (i1.numops, i1.numiter) == (i2.numops, i2.numiter)
        np.testing.assert_allclose(S1[:how], S2[:how], rtol=1e-10)
        assert l_chain < l_tuple
        check_triplets(A, S1[:how], [u.to_host() for u in U1], [v.to_host() for v in V1],
                       [r.to_host() for r in i1.residual], 1e-8 * max(1.0, S1[0]))
    finally:
        ctx.close()
