"""GPU tests of geneigsolve (Golub-Ye) end to end.

(a) Closed form: K the 5-point Dirichlet Laplacian on a 100 x 80 grid, M = I + K/8 a second assembled stencil with
    K's pattern (the fused path).  The generalized eigenvalues are μ = λ / (1 + λ/8) with λ from SURVEY §8c; :LR and
    :SR match them to 1e-10 relative in Float64.
(b) A 2e5-row pencil: A a diagonal with separated outliers plus a weak symmetric random coupling, B SPD and
    diagonally dominant with A's pattern (the fused path), and the same B with one explicitly stored zero (another
    pattern: the composed path).  Float64: the same numops, numiter and converged as the numpy restatement
    (tests/golubye_oracle.py), values within 1e-10 relative; Float32 (the device in Float32, the restatement in
    Float64, tol = 1e-4): values within 1e-4 relative, relations to 1e-3.  The relations A U = B U D + R and U'BU = I
    hold, and the values agree with scipy.sparse.linalg.eigsh(A, M=B).  The two paths give values within 1e-12 of
    each other; they are not bit-identical because the fused dots are summed in another order.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import golubye_oracle as go

SEED = 20261016
N = 200_000
HOWMANY = 3
f64, f32 = np.float64, np.float32


def pencil():
    rng = np.random.default_rng(SEED)
    d = rng.random(N)
    d[:3] = [-3.0, -2.4, -1.9]
    d[3:6] = [3.0, 3.6, 4.3]
    rows, cols = rng.integers(0, N, 3 * N), rng.integers(0, N, 3 * N)
    R = sp.csr_matrix((rng.random(3 * N), (rows, cols)), shape=(N, N))
    R = (R + R.T) * 0.01
    A = (sp.diags(d) + R).tocsr()
    Bp = abs(R) * 0.5
    B = (sp.diags(np.asarray(Bp.sum(axis=1)).ravel() + 1.0) + Bp).tocsr()
    A.sort_indices()
    B.sort_indices()
    assert np.array_equal(A.indptr, B.indptr) and np.array_equal(A.indices, B.indices)
    return A, B, rng.random(N)


def with_explicit_zero(B):
    row0 = set(B.indices[B.indptr[0]:B.indptr[1]].tolist())
    c = next(c for c in range(B.shape[1]) if c not in row0)
    coo = B.tocoo()
    Z = sp.csr_matrix((np.append(coo.data, 0.0), (np.append(coo.row, 0), np.append(coo.col, c))), shape=B.shape)
    Z.sort_indices()
    assert Z.nnz == B.nnz + 1
    return Z


def upload(ctx, M):
    return kk.B200CSR.from_csr_arrays(ctx, M.shape[0], M.shape[1], M.indptr, M.indices, M.data)


@pytest.mark.parametrize("which", ["LR", "SR"])
def test_laplacian_pencil_closed_form(which):
    nx, ny, h = 100, 80, 2
    n = nx * ny
    lam = np.sort(ko.laplace_eigenvalues(nx, ny))
    mu = lam / (1 + lam / 8)
    ref = mu[::-1][:h] if which == "LR" else mu[:h]
    ctx = kk.B200Context(n, 140)
    try:
        K = kk.B200CSR.stencil(ctx, nx, ny)
        M = kk.B200CSR.stencil(ctx, nx, ny, coeffs=(1.5, -0.125, -0.125, -0.125, -0.125, 0.0, 0.0))
        x0 = ctx.from_host(np.random.default_rng(1).random(n))
        vals, vecs, info = kk.geneigsolve((K, M), x0, h, which, krylovdim=30, maxiter=100, tol=1e-10,
                                          ishermitian=True, isposdef=True, verbosity=0)
        assert L.load().b2k_debug_pencil_path() == 1
        assert info.converged >= h
        np.testing.assert_allclose(vals[:h], ref, rtol=1e-10)
    finally:
        ctx.close()


def run(dt, B, A, x, tol):
    ctx = kk.B200Context(N, 4 * 31 + 3, dtype=dt)
    try:
        dA, dB = upload(ctx, A.astype(dt)), upload(ctx, B.astype(dt))
        P = kk.B200Pencil(dA, dB)
        vals, vecs, info = kk.geneigsolve(P, ctx.from_host(x.astype(dt)), HOWMANY, "SR", krylovdim=30, maxiter=100,
                                          tol=tol, ishermitian=True, isposdef=True, verbosity=0)
        path = L.load().b2k_debug_pencil_path()
        U = np.column_stack([v.to_host().astype(f64) for v in vecs])
        R = np.column_stack([r.to_host().astype(f64) for r in info.residual])
        P.free()
        return vals, U, R, info, path
    finally:
        ctx.close()


@pytest.fixture(scope="module")
def problem():
    A, B, x = pencil()
    o = go.golubye(A, B, x, HOWMANY, "SR", krylovdim=30, maxiter=100, tol=1e-10)
    Minv = spla.LinearOperator((N, N), matvec=lambda v: spla.cg(B, v, rtol=1e-14, maxiter=1000)[0], dtype=f64)
    ref = np.sort(spla.eigsh(A, k=HOWMANY, M=B, Minv=Minv, which="SA", tol=1e-12, return_eigenvectors=False))
    return A, B, x, o, ref


def test_pencil_2e5_float64_both_paths(problem):
    A, B, x, o, ref = problem
    out = {}
    for label, Bm in (("fused", B), ("composed", with_explicit_zero(B))):
        vals, U, R, info, path = run(f64, Bm, A, x, 1e-10)
        assert path == (1 if label == "fused" else 0)
        assert (info.numops, info.numiter, info.converged) == (o.numops, o.numiter, o.converged), label
        np.testing.assert_allclose(vals, o.values, rtol=1e-10)
        np.testing.assert_allclose(vals[:HOWMANY], ref, rtol=1e-9)
        BU = B @ U
        np.testing.assert_allclose(U.T @ BU, np.eye(U.shape[1]), atol=1e-9)
        np.testing.assert_allclose(A @ U, BU * vals + R, atol=1e-9 * np.abs(vals).max())
        out[label] = vals
    np.testing.assert_allclose(out["fused"], out["composed"], rtol=1e-12)


def test_pencil_2e5_float32(problem):
    A, B, x, o, ref = problem
    vals, U, R, info, path = run(f32, B, A, x, 1e-4)
    assert path == 1 and info.converged >= HOWMANY
    np.testing.assert_allclose(vals[:HOWMANY], ref, rtol=1e-4)
    BU = B @ U
    np.testing.assert_allclose(U.T @ BU, np.eye(U.shape[1]), atol=1e-3)
    np.testing.assert_allclose(A @ U, BU * vals + R, atol=1e-3 * np.abs(vals).max())
