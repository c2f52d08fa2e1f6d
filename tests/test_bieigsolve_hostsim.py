"""bieigsolve (BiArnoldi) without a GPU: the numpy restatement of the reference (tests/biarnoldi_oracle.py, with the
reference's per-step inner products) against dense truth, and the driver on the numpy stand-in of the C-ABI
(tests/hostsim.py, extended by tests/hostsim_bieig.py) against that restatement.  Also the stand-in's simulation of the two entry points the driver
adds (b2k_basis_cross_inner, b2k_op_create_transpose) and the driver's bookkeeping of the known block of M.

Tolerances are float64 ones: values within 1e-10 relative of the restatement; the relations A V = V D + R and
A' W = W conj(D) + R_W and W' V = I to 1e-9 after normalising by the sizes involved.
"""
import warnings

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import biarnoldi_oracle as bo
import hostsim
import hostsim_bieig


@pytest.fixture()
def sim():
    with hostsim_bieig.installed() as lib:
        yield lib
    assert not isinstance(L._lib, hostsim.HostSimLib)


def nonsym(seed, n=80, pairs=True):
    """a non-symmetric matrix with a spread real spectrum (pairs=False: similar to a diagonal one) or with complex
    pairs among its extreme eigenvalues"""
    rng = np.random.default_rng(seed)
    if pairs:
        return rng.standard_normal((n, n)) / np.sqrt(n) + np.diag(np.linspace(0.0, 3.0, n))
    P = np.eye(n) + 0.3 * rng.standard_normal((n, n)) / np.sqrt(n)
    return P @ np.diag(np.linspace(-2.0, 4.0, n) + 0.01 * rng.standard_normal(n)) @ np.linalg.inv(P)


def starts(seed, n):
    rng = np.random.default_rng(seed + 1000)
    return rng.random(n), rng.random(n)


def ordered_truth(A, which):
    ev = sl.eigvals(A)
    if isinstance(which, kk.EigSorter):
        return ev[which.permutation(ev)]
    key = {"LM": -np.abs(ev), "LR": -ev.real, "SR": ev.real}[which]
    return ev[np.argsort(key, kind="stable")]


def check_relations(A, vals, V, W, rV, rW, scale=1.0):
    """A v = λ v + r, A' w = conj(λ) w + r_W, W^H V = I"""
    Vm, Wm = np.column_stack(V), np.column_stack(W)
    nA = np.linalg.norm(A, 2) if isinstance(A, np.ndarray) else sp.linalg.norm(A)
    for i, lam in enumerate(vals):
        assert np.linalg.norm(A @ Vm[:, i] - lam * Vm[:, i] - rV[i]) <= 1e-9 * scale * nA * np.linalg.norm(Vm[:, i])
        assert np.linalg.norm(A.T @ Wm[:, i] - np.conj(lam) * Wm[:, i] - rW[i]) <= \
            1e-9 * scale * nA * np.linalg.norm(Wm[:, i])
    G = Wm.conj().T @ Vm
    assert np.abs(G - np.eye(len(vals))).max() <= 1e-9 * scale * max(1.0, np.abs(G).max())


SORTERS = ["LM", "LR", "SR", kk.EigSorter(lambda v: np.abs(v + 1.0), rev=True)]


@pytest.mark.parametrize("pairs", [False, True], ids=["real", "pairs"])
@pytest.mark.parametrize("which", SORTERS, ids=["LM", "LR", "SR", "sorter"])
@pytest.mark.parametrize("eager", [False, True])
def test_oracle_against_dense_truth(pairs, which, eager):
    A = nonsym(7, pairs=pairs)
    v0, w0 = starts(7, A.shape[0])
    howmany = 4
    vals, (V, W), (iV, iW), msgs = bo.bieigsolve_biarnoldi(A, A.T, v0, w0, howmany, which, krylovdim=12,
                                                          maxiter=400, tol=1e-12, eager=eager)
    assert iV["converged"] >= howmany and iV["numiter"] > 1 and not msgs
    truth = ordered_truth(A, which)
    for lam in vals:
        assert np.min(np.abs(truth[:len(vals) + 2] - lam)) <= 1e-9 * np.abs(truth).max()
    check_relations(A, vals, V, W, iV["residual"], iW["residual"])
    if pairs:
        assert np.any(np.abs(np.asarray(vals).imag) > 1e-3)


def test_oracle_keep_adjustment_runs():
    """a complex pair straddling `keep`: the 2x2-block adjustment of keep (both Schur forms) is exercised"""
    hits = 0
    for seed in range(40):
        A = nonsym(seed, n=60, pairs=True)
        v0, w0 = starts(seed, 60)
        kd, conv = 10, 0
        keep = (3 * kd + 2 * conv) // 5
        (S, T), *_ = bo.bischursolve(A, A.T, v0, w0, 3, "LR", kd, 1, 0.0, ko.Orth(ko.MGS2), False, lambda m: None)
        if S[keep, keep - 1] != 0 or T[keep, keep - 1] != 0:
            hits += 1
            vals, _, (iV, _), _ = bo.bieigsolve_biarnoldi(A, A.T, v0, w0, 3, "LR", krylovdim=kd, maxiter=300)
            assert iV["converged"] >= 3
    assert hits > 0


def run_driver(A, v0, w0, howmany, which, **kw):
    n = A.shape[0]
    ctx = kk.B200Context(n, 2 * kw.get("krylovdim", 30) + 24 + 8 * (howmany + 1))     # + the returned vectors
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        vals, (V, W), (iV, iW) = kk.bieigsolve(op, ctx.from_host(v0), ctx.from_host(w0), howmany, which, **kw)
    return ctx, vals, V, W, iV, iW, [str(r.message) for r in rec]


@pytest.mark.parametrize("seed", range(12))
def test_driver_matches_oracle(sim, seed):
    A = nonsym(seed, n=70, pairs=seed % 2 == 0)
    v0, w0 = starts(seed, 70)
    which = SORTERS[seed % 4]
    eager = seed % 3 == 0
    kw = dict(krylovdim=10 + seed % 5, maxiter=300, tol=1e-10, eager=eager)
    ctx, vals, V, W, iV, iW, msgs = run_driver(A, v0, w0, 3, which, **kw)
    ovals, (oV, oW), (oiV, oiW), omsgs = bo.bieigsolve_biarnoldi(A, A.T, v0, w0, 3, which, **kw)
    for info, oinfo in ((iV, oiV), (iW, oiW)):
        assert (info.converged, info.numiter, info.numops) == (oinfo["converged"], oinfo["numiter"], oinfo["numops"])
    assert len(vals) == len(ovals)
    assert np.abs(vals - ovals).max() <= 1e-10 * np.abs(ovals).max()
    Vh, Wh = [v.to_host() for v in V], [w.to_host() for w in W]
    rV, rW = [r.to_host() for r in iV.residual], [r.to_host() for r in iW.residual]
    check_relations(A, vals, Vh, Wh, rV, rW)
    assert np.allclose(iV.normres, [np.linalg.norm(r) for r in rV], rtol=1e-12, atol=1e-300)
    assert bool(msgs) == bool(omsgs)
    ctx.close()


def test_driver_warnings_as_the_reference(sim):
    """krylovdim = howmany + 2 and maxiter = 1: not converged, the same warning as the restatement"""
    A = nonsym(3, n=60)
    v0, w0 = starts(3, 60)
    ctx, vals, V, W, iV, iW, msgs = run_driver(A, v0, w0, 4, "LM", krylovdim=6, maxiter=1)
    *_, omsgs = bo.bieigsolve_biarnoldi(A, A.T, v0, w0, 4, "LM", krylovdim=6, maxiter=1)
    assert iV.converged < 4 and any("stopped without convergence" in m for m in msgs)
    assert any("stopped without convergence" in m for m in omsgs)
    assert iV.numiter == 1 and iV.numops == 1 + 2 * 5
    ctx.close()
    # an invariant subspace smaller than howmany: the reference's warning
    D = np.diag(np.arange(1.0, 31.0)) + 1e-14 * (np.eye(30, k=1) + np.eye(30, k=-1))
    e1 = np.zeros(30)
    e1[0] = 1.0
    ctx, vals, V, W, iV, iW, msgs = run_driver(D, e1, e1, 3, "LM", krylovdim=10, maxiter=2)
    *_, omsgs = bo.bieigsolve_biarnoldi(D, D.T, e1, e1, 3, "LM", krylovdim=10, maxiter=2)
    assert any("Invariant subspace of dimension 1" in m for m in msgs) and "Invariant subspace" in omsgs
    assert len(vals) == 1 and abs(vals[0] - 1.0) < 1e-12 and iV.numops == 1
    ctx.close()


def test_krylovdim_too_small(sim):
    A = nonsym(1, n=30)
    with pytest.raises(ValueError, match="too small"):
        run_driver(A, *starts(1, 30), 5, "LM", krylovdim=4)


def test_no_inner_products_during_expansions(sim):
    """k_known bookkeeping: M and the projections come from one cross Gram call per process step, which skips the
    block known from the previous step or restart; nothing else takes inner products"""
    A = nonsym(11, n=70)
    v0, w0 = starts(11, 70)
    calls, other = [], []
    real_cross = sim.b2k_basis_cross_inner

    def cross(h, X, p, Y, q, p0, q0, G, ldg):
        calls.append((p, q, p0, q0))
        return real_cross(h, X, p, Y, q, p0, q0, G, ldg)

    sim.b2k_basis_cross_inner = cross
    for name in ("b2k_vec_inner", "b2k_basis_project", "b2k_block_inner"):
        real = getattr(sim, name)
        setattr(sim, name, lambda *a, _r=real, _n=name: (other.append(_n), _r(*a))[1])
    kd = 10
    ctx, vals, V, W, iV, iW, msgs = run_driver(A, v0, w0, 3, "LR", krylovdim=kd, maxiter=50)
    assert other == ["b2k_vec_inner"] * 4               # the initialisation's orthogonalize!! of each side only
    assert len(calls) == iV.numiter                    # one process step per cycle (not eager)
    assert calls[0] == (kd + 1, kd + 1, 0, 0)
    assert all(c[:2] == (kd + 1, kd + 1) and 0 < c[2] == c[3] < kd for c in calls[1:])
    ctx.close()
    # eager: a process step at every size >= howmany, each computing only the new rows and columns
    calls.clear()
    other.clear()
    ctx, vals, V, W, iV, iW, msgs = run_driver(A, v0, w0, 3, "LR", krylovdim=kd, maxiter=3, eager=True)
    assert other == ["b2k_vec_inner"] * 4
    first = [c for c in calls[:kd - 2]]
    assert [c[0] for c in first] == list(range(4, kd + 2))
    assert [c[2] for c in first] == [0] + list(range(3, kd))
    ctx.close()


def test_entry_forms(sim):
    A = nonsym(5, n=50)
    v0, w0 = starts(5, 50)
    kw = dict(krylovdim=12, maxiter=300)
    ovals, *_ = bo.bieigsolve_biarnoldi(A, A.T, v0, w0, 2, "LR", **kw)
    ctx = kk.B200Context(50, 60)
    V0, W0 = ctx.from_host(v0), ctx.from_host(w0)
    csr = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    csrT = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A.T))
    dense = kk.B200Dense.from_host(ctx, A, 0)

    def f(x, adjoint):
        return kk.apply(csrT if adjoint else csr, x)

    forms = {"csr": csr, "dense": dense, "tuple": (csr, csrT), "tuple-callables": (lambda x: csr(x), lambda x: csrT(x)),
             "callable": f}
    for name, op in forms.items():
        vals, (V, W), (iV, iW) = kk.bieigsolve(op, V0, W0, 2, "LR", **kw)
        assert np.abs(vals - ovals).max() <= 1e-10 * np.abs(ovals).max(), name
        assert isinstance(V[0], kk.ComplexVec) and isinstance(W[0], kk.ComplexVec)
    for host in (sp.csr_matrix(A), A):
        vals, (V, W), (iV, iW) = kk.bieigsolve(host, v0, w0, 2, "LR", **kw)
        assert np.abs(vals - ovals).max() <= 1e-10 * np.abs(ovals).max()
        assert isinstance(V[0], np.ndarray) and V[0].dtype == np.complex128
        check_relations(A, vals, V, W, iV.residual, iW.residual)
    vals, (V, W), _ = kk.bieigsolve(sp.csr_matrix(A), howmany=2, which="LR", **kw)      # random starts
    assert np.abs(vals - ovals).max() <= 1e-8 * np.abs(ovals).max()
    alg = kk.BiArnoldi(krylovdim=12, maxiter=300)
    assert alg.tol == kk.KrylovDefaults.tol and alg.orth == kk.KrylovDefaults.orth and not alg.eager
    vals, _, _ = kk.bieigsolve(csr, V0, W0, 2, "LR", alg)
    assert np.abs(vals - ovals).max() <= 1e-10 * np.abs(ovals).max()
    with pytest.raises(ValueError, match="which = LI"):
        kk.bieigsolve(csr, V0, W0, 2, "LI")
    with pytest.raises(ValueError, match="conj"):
        kk.bieigsolve(csr, V0, W0, 2, kk.EigSorter(lambda v: v.imag))
    with pytest.raises(TypeError):
        kk.bieigsolve(csr, V0, W0, 2, "LR", alg, krylovdim=5)
    ctx.close()


def test_row_sharded_context_is_refused(sim):
    ctx = kk.B200Context(40, 20)
    ctx.nranks = 2                       # what a row-sharded context reports
    x = ctx.from_host(np.ones(40))
    op = kk.B200CSR.from_scipy(ctx, sp.eye(40, format="csr"))
    with pytest.raises(L.B200Error, match="row-sharded"):
        kk.bieigsolve(op, x, x, 1, "LM")
    ctx.close()


# ---- the stand-in's new entry points -------------------------------------------------------------------------

def test_stand_in_cross_inner_and_refusals(sim):
    import ctypes as C
    from krylovkit_jl_b200.vectors import handles
    rng = np.random.default_rng(2)
    ctx = kk.B200Context(30, 12)
    s1 = ctx.add_space(31, 2)
    X = [ctx.from_host(rng.standard_normal(30)) for _ in range(3)]
    Y = [ctx.from_host(rng.standard_normal(30)) for _ in range(4)]
    other = ctx.from_host(rng.standard_normal(31), space=s1)
    G = np.full((5, 4), 9.0, order="F")
    Gp = G.ctypes.data_as(C.POINTER(C.c_double))
    lib = ctx.lib
    assert lib.b2k_basis_cross_inner(ctx.h, handles(X), 3, handles(Y), 4, 1, 2, Gp, 5) == L.OK
    ref = np.column_stack([x.to_host() for x in X]).T @ np.column_stack([y.to_host() for y in Y])
    assert np.all(G[:1, :2] == 9.0) and np.all(G[3:, :] == 9.0)
    mask = np.ones((3, 4), bool)
    mask[:1, :2] = False
    assert np.allclose(G[:3][mask], ref[mask])
    G[:] = 9.0
    for code, args in [(L.EINVAL, (3, 4, 4, 0, 5)), (L.EINVAL, (3, 4, 0, 5, 5)), (L.EINVAL, (3, 4, 0, 0, 2)),
                       (L.EINVAL, (0, 4, 0, 0, 5)), (L.EINVAL, (257, 4, 0, 0, 300))]:
        p, q, p0, q0, ldg = args
        assert lib.b2k_basis_cross_inner(ctx.h, handles(X), p, handles(Y), q, p0, q0, Gp, ldg) == code
    assert lib.b2k_basis_cross_inner(ctx.h, handles(X), 3, handles(Y[:3] + [other]), 4, 0, 0, Gp, 5) == L.EDIM
    assert np.all(G == 9.0)
    ctx.close()


def test_stand_in_transpose(sim):
    rng = np.random.default_rng(4)
    ctx = kk.B200Context(40, 4)
    ctx.add_space(25, 4)
    A = sp.random(40, 25, density=0.2, random_state=rng, format="csr")
    t = kk.B200CSR.from_scipy(ctx, A).transpose()
    assert (abs(t.to_scipy() - A.T)).nnz == 0 and (t.n_rows, t.n_cols) == (25, 40)
    B = sp.random(40, 33, density=0.2, random_state=rng, format="csr")
    with pytest.raises(L.DimensionMismatch):
        kk.B200CSR.from_scipy(ctx, B).transpose()
    D = kk.B200Dense.from_host(ctx, np.ones((40, 40)), 0)
    import ctypes as C
    h = L.c_op()
    assert ctx.lib.b2k_op_create_transpose(ctx.h, C.byref(h), D.h) == L.ENOTSUP
    ctx.close()


# ---- the spectrum the measurement script checks against ---------------------------------------------------------

def test_convection_diffusion_spectrum():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "bieig_measure.py")
    spec = importlib.util.spec_from_file_location("bieig_measure", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    nx, ny = 13, 9
    A = ko.stencil_matrix(nx, ny, 1, m.COEFFS)
    ev = np.sort_complex(sl.eigvals(A.toarray()))
    an = np.sort_complex(m.convdiff_eigenvalues(nx, ny, m.COEFFS).astype(complex))
    assert np.allclose(ev.real, an.real, rtol=0, atol=1e-10) and np.abs(ev.imag).max() < 1e-8
    lead = m.convdiff_eigenvalues(nx, ny, m.COEFFS, top=3)
    assert np.allclose(lead, np.sort(an.real)[::-1][:3])
