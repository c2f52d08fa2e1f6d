"""geneigsolve (Golub-Ye) without a GPU: the numpy restatement of the reference (tests/golubye_oracle.py, with the
reference's per-step inner products) against dense truth, and the driver on the numpy stand-in of the C-ABI
(tests/hostsim.py, extended by tests/hostsim_bieig.py and tests/hostsim_geneig.py) against that restatement: equal
numops, numiter and converged, values within 1e-12, every entry form and orthogonalizer, the selector's errors, the
warnings, the aliasing of `vold` and one cross Gram call per process step.
"""
import warnings

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L

import golubye_oracle as go
import hostsim
import hostsim_geneig

ORTHS = {"cgs": (kk.cgs, go.CGS), "mgs": (kk.mgs, go.MGS), "cgs2": (kk.cgs2, go.CGS2), "mgs2": (kk.mgs2, go.MGS2),
         "cgsr": (kk.cgsr, go.CGSIR), "mgsr": (kk.mgsr, go.MGSIR), "mgs2b": (kk.mgs2b, go.MGS2B)}


@pytest.fixture()
def sim():
    with hostsim_geneig.installed() as lib:
        yield lib
    assert not isinstance(L._lib, hostsim.HostSimLib)


def dense_case(seed, n):
    """test/geneigsolve.jl's matrices: A = (R + R')/2, B = sqrt(S S') with R, S uniform in [-1/2, 1/2)."""
    rng = np.random.default_rng(seed)
    A = rng.random((n, n)) - 0.5
    A = (A + A.T) / 2
    S = rng.random((n, n)) - 0.5
    B = np.real(sl.sqrtm(S @ S.T))
    return A, (B + B.T) / 2, rng.random(n)


def sparse_case(seed, n=300):
    """separated outliers on a diagonal plus a weak symmetric coupling; B SPD, diagonally dominant, A's pattern"""
    rng = np.random.default_rng(seed)
    d = np.linspace(0.0, 1.0, n)
    d[:4] = [-3.0, -2.5, -2.0, -1.6]
    d[-4:] = [3.0, 3.5, 4.0, 4.6]
    R = sp.random(n, n, density=0.02, random_state=seed)
    R = (R + R.T) * 0.02
    A = (sp.diags(d) + R).tocsr()
    Bp = abs(R) * 0.5
    B = (sp.diags(np.asarray(Bp.sum(axis=1)).ravel() + 1.0) + Bp).tocsr()
    return A, B, rng.random(n)


def check_against(o, vals, info):
    assert (info.numops, info.numiter, info.converged) == (o.numops, o.numiter, o.converged)
    assert len(vals) == len(o.values)
    np.testing.assert_allclose(vals, o.values, rtol=1e-12, atol=1e-12)


# ---- the restatement against dense truth (test/geneigsolve.jl) --------------------------------------------------

@pytest.mark.parametrize("orth", ["cgs2", "mgs2", "cgsr", "mgsr"])
def test_oracle_full(orth):
    n = 10
    A, B, x = dense_case(1, n)
    n1 = n // 2
    o1 = go.golubye(A, B, x, n1, "SR", krylovdim=n, maxiter=1, tol=1e-12, orth=ORTHS[orth][1])
    o2 = go.golubye(A, B, x, n - n1, "LR", krylovdim=n, maxiter=1, tol=1e-12, orth=ORTHS[orth][1])
    D = sl.eigh(A, B, eigvals_only=True)
    np.testing.assert_allclose(np.concatenate([o1.values[:n1], o2.values[:n - n1][::-1]]), D, rtol=1e-10, atol=1e-10)
    for o in (o1, o2):
        U = np.column_stack(o.vectors)
        np.testing.assert_allclose(U.T @ B @ U, np.eye(U.shape[1]), atol=1e-10)
        np.testing.assert_allclose(A @ U, B @ U @ np.diag(o.values), atol=1e-9)


@pytest.mark.parametrize("orth", ["cgs2", "mgs2", "cgsr", "mgsr"])
def test_oracle_iterative(orth):
    N, n = 100, 10
    A, B, x = dense_case(2, N)
    tol = np.linalg.cond(B) * 1e-12
    D = sl.eigh(A, B, eigvals_only=True)
    for which, ref in (("SR", D), ("LR", D[::-1])):
        o = go.golubye(A, B, x, n, which, krylovdim=3 * n, maxiter=100, tol=tol, orth=ORTHS[orth][1])
        assert o.converged > 0
        c = o.converged
        np.testing.assert_allclose(o.values[:c], ref[:c], rtol=1e-6)
        U, R = np.column_stack(o.vectors), np.column_stack(o.residuals)
        np.testing.assert_allclose(U.T @ B @ U, np.eye(U.shape[1]), atol=1e-8)
        np.testing.assert_allclose(A @ U, B @ U @ np.diag(o.values) + R, atol=1e-8)


# ---- the driver on the stand-in against the restatement ---------------------------------------------------------

@pytest.mark.parametrize("orth", list(ORTHS))
@pytest.mark.parametrize("which", ["SR", "LR"])
def test_driver_matches_oracle(sim, orth, which):
    A, B, x = sparse_case(3)
    o = go.golubye(A, B, x, 3, which, krylovdim=12, maxiter=100, tol=1e-10, orth=ORTHS[orth][1])
    vals, vecs, info = kk.geneigsolve((A, B), x, 3, which, krylovdim=12, maxiter=100, tol=1e-10,
                                      orth=ORTHS[orth][0], verbosity=0)
    check_against(o, vals, info)
    assert sim.pencil_calls[0] == 0 and sim.pencil_calls[1] == info.numops      # same pattern: every product fused
    U = np.column_stack(vecs)
    np.testing.assert_allclose(U.T @ (B @ U), np.eye(U.shape[1]), atol=1e-10)


@pytest.mark.parametrize("orth", list(ORTHS))
def test_driver_dense_full(sim, orth):
    A, B, x = dense_case(1, 10)
    o = go.golubye(A, B, x, 5, "SR", krylovdim=10, maxiter=1, tol=1e-12, orth=ORTHS[orth][1])
    vals, _, info = kk.geneigsolve((A, B), x, 5, "SR", krylovdim=10, maxiter=1, tol=1e-12, orth=ORTHS[orth][0],
                                   verbosity=0)
    check_against(o, vals, info)


def _device(ctx, A, B):
    return kk.B200CSR.from_scipy(ctx, A), kk.B200CSR.from_scipy(ctx, B)


@pytest.mark.parametrize("form", ["pencil", "csr_tuple", "callable_tuple", "callable", "composed_pencil"])
def test_entry_forms(sim, form):
    A, B, x = sparse_case(4)
    o = go.golubye(A, B, x, 2, "LR", krylovdim=10, maxiter=100, tol=1e-10, orth=go.MGS2)
    ctx = kk.B200Context(A.shape[0], 64)
    dA, dB = _device(ctx, A, B)
    if form == "composed_pencil":
        Bz = B.tocoo()                       # B with one explicitly stored zero: the same matrix, another pattern
        Bz = sp.csr_matrix((np.append(Bz.data, 0.0), (np.append(Bz.row, 0), np.append(Bz.col, A.shape[0] - 1))),
                           shape=B.shape)
        Bz.sum_duplicates()
        dB = kk.B200CSR.from_csr_arrays(ctx, B.shape[0], B.shape[1], Bz.indptr, Bz.indices, Bz.data)
    f = {"pencil": lambda: kk.B200Pencil(dA, dB), "composed_pencil": lambda: kk.B200Pencil(dA, dB),
         "csr_tuple": lambda: (dA, dB), "callable_tuple": lambda: (lambda v: dA(v), lambda v: dB(v)),
         "callable": lambda: (lambda v: (dA(v), dB(v)))}[form]()
    vals, vecs, info = kk.geneigsolve(f, ctx.from_host(x), 2, "LR", krylovdim=10, maxiter=100, tol=1e-10, orth=kk.mgs2,
                                      ishermitian=True, isposdef=True, verbosity=0)
    check_against(o, vals, info)
    assert all(isinstance(v, kk.B200Vec) for v in vecs)
    fused = sim.pencil_calls[1]
    if form in ("pencil", "csr_tuple"):
        assert fused == info.numops and sim.pencil_calls[0] == 0 and sim.b2k_debug_pencil_path() == 1
    elif form == "composed_pencil":
        assert fused == 0 and sim.pencil_calls[0] == info.numops and sim.b2k_debug_pencil_path() == 0
    else:
        assert fused == 0 and sim.pencil_calls[0] == 0
    if form == "csr_tuple":
        assert not sim.pencils                      # the pencil made internally is freed
    ctx.close()


def test_host_forms_default_start_and_float32(sim):
    A, B, _ = sparse_case(5)
    vals, vecs, info = kk.geneigsolve((A, B), None, 2, "SR", krylovdim=10, tol=1e-10, verbosity=0)
    assert info.converged >= 2 and isinstance(vecs[0], np.ndarray)
    D = sl.eigh(A.toarray(), B.toarray(), eigvals_only=True)
    np.testing.assert_allclose(vals[:2], D[:2], rtol=1e-9)
    vals, _, info = kk.geneigsolve((A.toarray(), B.toarray()), np.random.default_rng(1).random(A.shape[0]), 2, "SR",
                                   krylovdim=10, tol=1e-10, verbosity=0)
    np.testing.assert_allclose(vals[:2], D[:2], rtol=1e-9)
    vals, vecs, info = kk.geneigsolve((A, B), np.random.default_rng(1).random(A.shape[0]).astype(np.float32), 2, "SR",
                                      krylovdim=10, tol=1e-4, verbosity=0)
    assert vecs[0].dtype == np.float32
    np.testing.assert_allclose(vals[:2], D[:2], rtol=1e-4)


def test_selector_errors(sim):
    A, B, x = sparse_case(6)
    msg = "Only symmetric or hermitian generalized"
    with pytest.raises(ValueError, match=msg):
        kk.geneigsolve((A + sp.triu(A, 1), B), x, 1, "SR")                   # A not symmetric
    Bd = B.toarray()
    Bd[0, 0] = -5.0
    with pytest.raises(ValueError, match=msg):
        kk.geneigsolve((A.toarray(), Bd), x, 1, "SR")                         # dense Cholesky fails
    Bw = B.copy()
    Bw.setdiag(0.01)
    with pytest.raises(ValueError, match="isposdef=True"):
        kk.geneigsolve((A, Bw), x, 1, "SR")                                   # Gershgorin test fails
    ctx = kk.B200Context(A.shape[0], 40)
    dA, dB = _device(ctx, A, B)
    with pytest.raises(ValueError, match=msg):
        kk.geneigsolve((dA, dB), ctx.from_host(x), 1, "SR")                   # device operators: declared only
    with pytest.raises(ValueError, match=msg):
        kk.geneigsolve((dA, dB), ctx.from_host(x), 1, "SR", ishermitian=True)
    assert isinstance(kk.geneigselector((dA, dB), ishermitian=True, isposdef=True, krylovdim=7), kk.GolubYe)
    for which in ("LI", "SI"):
        with pytest.raises(ValueError, match="real eigenvalues expected with Lanczos algorithm"):
            kk.geneigsolve((A, B), x, 1, which)
    with pytest.raises(ValueError, match="too small to compute"):
        kk.geneigsolve((A, B), x, 11, "SR", krylovdim=10)
    with pytest.raises(ValueError, match="initial vector should not have norm zero"):
        kk.geneigsolve((A, B), np.zeros(A.shape[0]), 1, "SR")
    with pytest.raises(TypeError):
        kk.GolubYe(eager=True)                                                  # the reference struct has no eager
    ctx.close()


def test_invariant_subspace_warning_and_howmany(sim):
    n = 40
    A = sp.diags(np.r_[np.arange(1.0, 4.0), np.zeros(n - 3)]).tocsr()
    B = sp.identity(n, format="csr")
    x = np.zeros(n)
    x[:3] = 1.0                                     # a start vector in a 3-dimensional invariant subspace
    o = go.golubye(A, B, x, 5, "LR", krylovdim=10, maxiter=3, tol=1e-10)
    with hostsim_geneig.installed():
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            vals, _, info = kk.geneigsolve((A, B), x, 5, "LR", krylovdim=10, maxiter=3, tol=1e-10)
    inv = [m for m in w if "Invariant subspace" in str(m.message)]
    assert len(inv) == o.warnings.count("invariant") >= 1
    assert "setting `howmany = 3`" in str(inv[0].message)
    check_against(o, vals, info)
    assert info.converged == 3


def test_no_convergence_warning(sim):
    A, B, x = dense_case(2, 60)
    o = go.golubye(A, B, x, 4, "SR", krylovdim=6, maxiter=3, tol=1e-14)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        vals, _, info = kk.geneigsolve((A, B), x, 4, "SR", krylovdim=6, maxiter=3, tol=1e-14)
    stop = [m for m in w if "stopped without convergence" in str(m.message)]
    assert len(stop) == o.warnings.count("noconv") == 1
    assert (info.numops, info.numiter, info.converged) == (o.numops, o.numiter, o.converged)
    assert info.numiter == 3 and len(vals) == 4          # the last cycle keeps unconverged vectors up to howmany
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        kk.geneigsolve((A, B), x, 4, "SR", krylovdim=6, maxiter=3, tol=1e-14, verbosity=0)
    assert not [m for m in w if "stopped without convergence" in str(m.message)]


def test_vold_aliasing_matters(sim):
    """`vold` is orthonormalized in place every cycle (golubye.jl:30, 64): a restatement that copies it instead takes
    a different path; the driver follows the aliasing one."""
    A, B, x = dense_case(7, 30)
    kw = dict(krylovdim=4, maxiter=6, tol=1e-12)
    o = go.golubye(A, B, x, 2, "SR", **kw)
    oc = go.golubye(A, B, x, 2, "SR", alias=False, **kw)
    assert o.numops != oc.numops or not np.allclose(o.values, oc.values, rtol=1e-12, atol=0)
    vals, _, info = kk.geneigsolve((A, B), x, 2, "SR", verbosity=0, **kw)
    check_against(o, vals, info)


def test_numops_count(sim):
    """1 at the start, 1 per expansion, 1 for vold and 1 per converged vector per later process step, 1 per Ritz
    vector formed (counted independently from the stand-in's calls)."""
    A, B, x = sparse_case(8)
    vals, _, info = kk.geneigsolve((A, B), x, 3, "SR", krylovdim=12, tol=1e-10, verbosity=0)
    assert sim.pencil_calls[1] == info.numops


def test_one_cross_inner_per_process_step(sim, monkeypatch):
    A, B, x = sparse_case(9)
    import importlib
    gm = importlib.import_module("krylovkit_jl_b200.geneigsolve")
    calls = []
    orig = gm.cross_inner

    def spy(X, Y, *a, **k):
        calls.append((len(X), sim.pencil_calls[1]))
        return orig(X, Y, *a, **k)

    monkeypatch.setattr(gm, "cross_inner", spy)
    o = go.golubye(A, B, x, 3, "SR", krylovdim=12, maxiter=100, tol=1e-10)
    vals, _, info = kk.geneigsolve((A, B), x, 3, "SR", krylovdim=12, maxiter=100, tol=1e-10, verbosity=0)
    check_against(o, vals, info)
    assert len(calls) == sim.cross_calls == info.numiter          # every cycle ends in exactly one process step
    # between two process steps only expansions (and the next step's vold / converged products) take products
    assert all(k <= 12 + 1 + 3 for k, _ in calls)


def test_hb_width_limit(sim):
    class Fake(list):
        pass
    with pytest.raises(ValueError, match="at most 256"):
        from krylovkit_jl_b200.geneigsolve import buildHB_
        buildHB_(np.zeros((300, 300)), Fake([None] * 257), [None] * 257)


def test_no_slab_columns_leak_across_cycles(sim):
    A, B, x = sparse_case(10)
    kd = 8
    ctx = kk.B200Context(A.shape[0], 4 * (kd + 1) + 3)
    dA, dB = _device(ctx, A, B)
    P = kk.B200Pencil(dA, dB)
    x0 = ctx.from_host(x)
    base = sim.b2k_debug_used_columns(ctx.h, 0)
    vals, vecs, info = kk.geneigsolve(P, x0, 3, "SR", krylovdim=kd, maxiter=100, tol=1e-10, ishermitian=True,
                                      isposdef=True, verbosity=0)
    assert info.numiter > 2
    held = len(vecs) + len(info.residual)
    assert sim.b2k_debug_used_columns(ctx.h, 0) == base + held
    del vecs, info
    assert sim.b2k_debug_used_columns(ctx.h, 0) == base
    ctx.close()


def test_pencil_refusals_write_nothing(sim):
    A, B, x = sparse_case(11, n=50)
    ctx = kk.B200Context(50, 16)
    ctx.add_space(49, 4)
    dA, dB = _device(ctx, A, B)
    P = kk.B200Pencil(dA, dB)
    vs = [ctx.from_host(np.full(50, i + 1.0)) for i in range(4)]
    short = ctx.from_host(np.ones(49), space=1)
    before = [v.to_host().copy() for v in vs]
    lib, h = ctx.lib, ctx.h
    x, w, bx, vp = (v.handle for v in vs)
    cases = [(L.EINVAL, lambda: lib.b2k_pencil_apply(h, P.h, x, x, bx, 1.0, -1, 0.0, None)),
             (L.EINVAL, lambda: lib.b2k_pencil_apply(h, P.h, x, w, bx, 1.0, w, 0.5, None)),
             (L.EDIM, lambda: lib.b2k_pencil_apply(h, P.h, x, w, short.handle, 1.0, -1, 0.0, None)),
             (L.EINVAL, lambda: lib.b2k_pencil_rayleigh(h, P.h, x, w, w, None, None)),
             (L.EINVAL, lambda: lib.b2k_pencil_create(h, None, dA.h, dA.h))]
    for code, call in cases:
        assert call() == code
    for v, b in zip(vs, before):
        np.testing.assert_array_equal(v.to_host(), b)
    ctx2 = kk.B200Context(50, 8)
    y = [ctx2.from_host(np.ones(50)) for _ in range(3)]
    assert lib.b2k_pencil_apply(ctx2.h, P.h, y[0].handle, y[1].handle, y[2].handle, 1.0, -1, 0.0, None) == L.EINVAL
    with pytest.raises(L.DimensionMismatch):
        kk.B200Pencil(dA, kk.B200CSR.from_scipy(ctx, sp.identity(49, format="csr")))
    ctx2.close()
    ctx.close()
