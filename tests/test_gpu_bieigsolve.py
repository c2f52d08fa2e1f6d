"""GPU tests of bieigsolve (BiArnoldi) end to end, on a sparse non-symmetric matrix of 2e5 rows whose largest
eigenvalues are separated from the rest and include one complex pair: against the numpy restatement of the reference
(tests/biarnoldi_oracle.py: the same counts, the same values) and against scipy.sparse.linalg.eigs on A and on A'.
The relations A V = V D + R, A' W = W conj(D) + R_W and W' V = I hold for what comes back, and the path that builds
A' on the device (B200CSR) gives the bits of the path that is handed a host-built A' as an (A, At) tuple.

Tolerances.  Float64: values within 1e-10 relative of the restatement, relations to 1e-9 relative.  Float32 (the
device works in Float32, the restatement in Float64, tol = 1e-4): values within 1e-4 relative, relations to 1e-3.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
import biarnoldi_oracle as bo

SEED = 20261016
N = 200_000
HOWMANY = 4
f64, f32 = np.float64, np.float32


def matrix():
    """diagonal bulk in [0, 1] plus outliers 3, 2.5 and the block [[2, 0.5], [-0.5, 2]] (2 ± 0.5i), coupled by a weak
    non-symmetric random sparse part"""
    rng = np.random.default_rng(SEED)
    d = rng.random(N)
    d[:4] = (3.0, 2.5, 2.0, 2.0)
    A = sp.diags(d).tolil()
    A[2, 3], A[3, 2] = 0.5, -0.5
    R = sp.random(N, N, density=3.0 / N, random_state=rng, format="csr") * 0.02
    R.data -= 0.01
    A = (A.tocsr() + R).tocsr()
    A.sort_indices()
    return A


_A = []


def mat():
    if not _A:
        _A.append(matrix())
    return _A[0]


def run(A, dt, form, tol):
    rng = np.random.default_rng(SEED + 1)
    v0, w0 = rng.random(N).astype(dt), rng.random(N).astype(dt)
    ctx = kk.B200Context(N, 2 * 30 + 24 + 8 * (HOWMANY + 2), dtype=dt)
    op = kk.B200CSR.from_scipy(ctx, A.astype(dt))
    if form == "tuple":
        op = (op, kk.B200CSR.from_scipy(ctx, A.T.tocsr().astype(dt)))
    vals, (V, W), (iV, iW) = kk.bieigsolve(op, ctx.from_host(v0), ctx.from_host(w0), HOWMANY, "LM", tol=tol,
                                           krylovdim=30, maxiter=100)
    out = (vals, [v.to_host() for v in V], [w.to_host() for w in W], [r.to_host() for r in iV.residual],
           [r.to_host() for r in iW.residual], iV, iW)
    ctx.close()
    return out, v0, w0


def relations(A, vals, V, W, rV, rW, rel):
    nA = spla.norm(A, 1)
    for lam, v, w, r, s in zip(vals, V, W, rV, rW):
        assert np.linalg.norm(A @ v - lam * v - r) <= rel * nA * np.linalg.norm(v)
        assert np.linalg.norm(A.T @ w - np.conj(lam) * w - s) <= rel * nA * np.linalg.norm(w)
    G = np.column_stack(W).conj().T @ np.column_stack(V)
    assert np.abs(G - np.eye(len(vals))).max() <= rel * max(1.0, np.abs(G).max())


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
def test_bieigsolve_against_oracle_and_eigs(dt):
    A = mat()
    tol = 1e-10 if dt == f64 else 1e-4
    (vals, V, W, rV, rW, iV, iW), v0, w0 = run(A, dt, "csr", tol)
    ovals, _, (oiV, oiW), _ = bo.bieigsolve_biarnoldi(A, A.T, v0.astype(f64), w0.astype(f64), HOWMANY, "LM",
                                                     krylovdim=30, maxiter=100, tol=tol)
    assert iV.converged >= HOWMANY and iW.converged >= HOWMANY
    if dt == f64:
        for info, o in ((iV, oiV), (iW, oiW)):
            assert (info.converged, info.numiter, info.numops) == (o["converged"], o["numiter"], o["numops"])
        assert np.abs(vals - ovals).max() <= 1e-10 * np.abs(ovals).max()
    else:
        assert np.abs(vals[:HOWMANY] - ovals[:HOWMANY]).max() <= 1e-4 * np.abs(ovals).max()
    assert np.any(np.abs(vals.imag) > 0.4)                 # the complex pair is among them
    truth = spla.eigs(A, k=HOWMANY, which="LM", tol=1e-12)[0]
    truth_left = spla.eigs(A.T.tocsr(), k=HOWMANY, which="LM", tol=1e-12)[0]
    rel = 1e-10 if dt == f64 else 1e-4
    for lam in vals[:HOWMANY]:
        assert np.min(np.abs(truth - lam)) <= rel * 3.0
        assert np.min(np.abs(truth_left - np.conj(lam))) <= rel * 3.0
    relations(A, vals, V, W, rV, rW, 1e-9 if dt == f64 else 1e-3)


def test_device_transpose_equals_host_transpose_bitwise():
    A = mat()
    (a, Va, Wa, rVa, rWa, iVa, iWa), _, _ = run(A, f64, "csr", 1e-10)
    (b, Vb, Wb, rVb, rWb, iVb, iWb), _, _ = run(A, f64, "tuple", 1e-10)
    assert np.array_equal(a, b)
    for x, y in zip(Va + Wa + rVa + rWa, Vb + Wb + rVb + rWb):
        assert np.array_equal(x, y)
    assert (iVa.numiter, iVa.numops, iVa.converged) == (iVb.numiter, iVb.numops, iVb.converged)


def test_host_matrix_entry():
    """scipy sparse host matrix: uploaded once, transposed on the device, complex numpy vectors back"""
    A = mat()
    rng = np.random.default_rng(SEED + 1)
    v0, w0 = rng.random(N), rng.random(N)
    vals, (V, W), (iV, iW) = kk.bieigsolve(A, v0, w0, HOWMANY, "LM", tol=1e-10)
    (ref, *_), _, _ = run(A, f64, "csr", 1e-10)
    assert np.allclose(vals, ref, rtol=1e-12, atol=0)
    assert all(isinstance(v, np.ndarray) and v.dtype == np.complex128 for v in V + W)
    relations(A, vals, V, W, iV.residual, iW.residual, 1e-9)
