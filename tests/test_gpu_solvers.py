"""GPU parity of the factorizations and drivers (called through the C-ABI via the host
mirror) against the CPU oracle on identical (A, x0): per-step Lanczos/Arnoldi/GKL
coefficients, Ritz values within 1e-10 relative (FP64), residual identities within the
reference's own tolerances (test/testsetup.jl:14-15)."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.factorizations import arnoldi as ar
from krylovkit_jl_b200.factorizations import lanczos as lz
from oracle import krylov_oracle as ko

SEED = 20260923
PAIRS = [(kk.cgs, ko.Orth(ko.CGS)), (kk.mgs, ko.Orth(ko.MGS)), (kk.cgs2, ko.Orth(ko.CGS2)),
         (kk.mgs2, ko.Orth(ko.MGS2)), (kk.ClassicalGramSchmidtIR(eta=0.75), ko.Orth(ko.CGSIR, 0.75)),
         (kk.ModifiedGramSchmidtIR(eta=0.75), ko.Orth(ko.MGSIR, 0.75)),
         # the flagged blocked mode of MGS2 (B2K_MGS2B) is checked against the REFERENCE's MGS2
         (kk.mgs2b, ko.Orth(ko.MGS2))]
IDS = ["cgs", "mgs", "cgs2", "mgs2", "cgsr", "mgsr", "mgs2b"]


def conv_diff(nx, ny):
    return ko.stencil_matrix(nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0, 0))


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
@pytest.mark.parametrize("fused", [True, False])
def test_lanczos_steps_match_oracle(pair, fused):
    """expand! step by step: alpha_k, beta_k equal the oracle's to <= 1e-12 relative for the
    reorthogonalised variants; V'V = I, A V = V T + r e' (test/factorize.jl:140-148)."""
    orth, oorth = pair
    nx, ny = 61, 43
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(SEED, n)
    ctx = kk.B200Context(n, 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    it = lz.LanczosIterator(op, ctx.from_host(x0), orth)
    f = lz.initialize(it)
    g = ko.lanczos_initialize(A, x0, oorth)
    steps = 24
    for _ in range(steps):
        f = lz.expand_(it, f, fused=fused)
        g = ko.lanczos_expand(A, g, oorth)
    tol = 1e-12 if orth.tag not in (L.CGS, L.MGS) else 1e-6
    np.testing.assert_allclose(f.alphas, g.alphas, rtol=tol, atol=tol)
    np.testing.assert_allclose(f.betas, g.betas, rtol=tol, atol=tol)
    V = np.column_stack([v.to_host() for v in f.V])
    k = f.k
    T = np.diag(f.alphas) + np.diag(f.betas[:k - 1], 1) + np.diag(f.betas[:k - 1], -1)
    r = f.r.to_host()
    if orth.tag not in (L.CGS, L.MGS):
        assert np.abs(V.T @ V - np.eye(k)).max() < 1e-12
    E = A @ V - V @ T
    E[:, -1] -= r
    assert np.abs(E).max() < 1e-11
    assert abs(np.linalg.norm(r) - f.normres()) < 1e-12
    lz.shrink_(f, 10)
    assert f.k == 10 and len(f.V) == 10
    ctx.close()


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_arnoldi_steps_match_oracle(pair):
    orth, oorth = pair
    nx, ny = 50, 37
    n = nx * ny
    A = conv_diff(nx, ny)
    x0 = ko.splitmix_vector(SEED, n)
    ctx = kk.B200Context(n, 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    it = ar.ArnoldiIterator(op, ctx.from_host(x0), orth)
    f = ar.initialize(it)
    g = ko.arnoldi_initialize(A, x0, oorth)
    for _ in range(20):
        f = ar.expand_(it, f)
        g = ko.arnoldi_expand(A, g, oorth)
    tol = 1e-12 if orth.tag not in (L.CGS, L.MGS) else 1e-8
    np.testing.assert_allclose(f.H, g.H, rtol=tol, atol=tol)
    V = np.column_stack([v.to_host() for v in f.V])
    H = f.rayleighquotient()
    E = A @ V - V @ H
    E[:, -1] -= f.r.to_host()
    assert np.abs(E).max() < 1e-11
    ctx.close()


@pytest.mark.parametrize("which", ["SR", "LR"])
@pytest.mark.parametrize("pair", [PAIRS[2], PAIRS[3], PAIRS[4], PAIRS[6]], ids=["cgs2", "mgs2", "cgsr", "mgs2b"])
def test_eigsolve_config1_matches_oracle_and_closed_form(pair, which):
    """BASELINE config 1 (1e4 x 1e4 5-point Laplacian, krylovdim 30, howmany 4): Ritz values
    within 1e-10 relative of the oracle and of the closed form, residuals within tol."""
    orth, oorth = pair
    nx, ny = 125, 80
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    lam = ko.laplace_eigenvalues(nx, ny)
    x0 = ko.splitmix_vector(SEED, n)
    alg = kk.Lanczos(orth=orth, krylovdim=30, maxiter=300, tol=1e-10, verbosity=0)
    ctx = kk.B200Context(n, 48)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0), 4, which, alg)
    ovals, ovecs, oinfo = ko.eigsolve_lanczos(A, x0, 4, which, krylovdim=30, maxiter=300, tol=1e-10,
                                              orth=oorth)
    assert info.converged >= 4
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    np.testing.assert_allclose(vals[:4], ovals[:4], rtol=1e-10)
    ref = lam[:4] if which == "SR" else lam[::-1][:4]
    np.testing.assert_allclose(vals[:4], ref, rtol=1e-10)
    for i in range(4):
        v = vecs[i].to_host()
        assert np.linalg.norm(A @ v - vals[i] * v) < 1e-8
        assert abs(np.linalg.norm(v) - 1) < 1e-10
    ctx.close()


def test_eigsolve_unconverged_fixed_cycles_matches_oracle():
    """The benchmark regime: a fixed number of restart cycles far from convergence.  Ritz
    values and residual norms agree with the oracle at that point."""
    nx, ny = 300, 200
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(SEED, n)
    ctx = kk.B200Context(n, 80)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=60, maxiter=3, tol=1e-14, verbosity=0)
    vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0), 4, "SR", alg)
    ovals, _, oinfo = ko.eigsolve_lanczos(A, x0, 4, "SR", krylovdim=60, maxiter=3, tol=1e-14,
                                          orth=ko.Orth(ko.CGS2))
    assert info.numops == oinfo["numops"] == 60 + 2 * 24
    np.testing.assert_allclose(vals, ovals, rtol=1e-10)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-6, atol=1e-12)
    ctx.close()


def test_eigsolve_host_buffers_end_to_end():
    nx, ny = 64, 48
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(3, nx * ny)
    vals, vecs, info = kk.eigsolve(A, x0, 2, "LR", kk.Lanczos(orth=kk.cgs2, krylovdim=30, tol=1e-10,
                                                              verbosity=0))
    lam = ko.laplace_eigenvalues(nx, ny)
    assert info.converged >= 2
    np.testing.assert_allclose(vals[:2], lam[::-1][:2], rtol=1e-10)
    assert isinstance(vecs[0], np.ndarray)
    assert np.linalg.norm(A @ vecs[0] - vals[0] * vecs[0]) < 1e-8


def test_issue143_and_toric_on_gpu():
    """the reference's known-answer fixtures through the GPU path."""
    import os
    A = np.load(os.path.join(os.path.dirname(__file__), "golden", "issue143_matrix.npy"))
    n = A.shape[0]
    rng = np.random.default_rng(143)
    vals, vecs, info = kk.eigsolve(sp.csr_matrix(A), rng.standard_normal(n), n, "SR",
                                   kk.Lanczos(orth=kk.mgs2, krylovdim=n, maxiter=1, tol=1e-12, verbosity=0))
    ref = np.linalg.eigvalsh(A)
    np.testing.assert_allclose(vals, ref, rtol=1e-10, atol=1e-10 * np.abs(ref).max())
    H = ko.toric_code_hamiltonian(3, 3)
    x0 = ko.splitmix_vector(7, H.shape[0])
    vals, vecs, info = kk.eigsolve(-H, x0, 1, "SR", kk.Lanczos(orth=kk.cgs2, krylovdim=30, maxiter=30,
                                                               tol=1e-8, verbosity=0))
    assert info.converged >= 1 and abs(vals[0] + 16.0) < 1e-8


@pytest.mark.parametrize("pair", [PAIRS[2], PAIRS[3], PAIRS[6]], ids=["cgs2", "mgs2", "mgs2b"])
@pytest.mark.parametrize("literal", [False, True])
def test_gmres_matches_oracle(pair, literal):
    """config 3 at test size: nonsymmetric convection-diffusion, b = A*1, restarted GMRES."""
    from krylovkit_jl_b200 import linsolve as ls
    orth, oorth = pair
    nx, ny = 80, 50
    n = nx * ny
    A = conv_diff(nx, ny)
    b = A @ np.ones(n)
    ls.LITERAL_GIVENS_RESTART = literal
    ctx = kk.B200Context(n, 60)
    op = kk.B200CSR.from_scipy(ctx, A)
    alg = kk.GMRES(orth=orth, krylovdim=40, maxiter=5, tol=1e-12, verbosity=0)
    x, info = kk.linsolve(op, ctx.from_host(b), None, alg)
    ox, oinfo = ko.linsolve_gmres(A, b, None, krylovdim=40, maxiter=5, tol=1e-12, orth=oorth)
    ls.LITERAL_GIVENS_RESTART = False
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    xh = x.to_host()
    # b = A x + residual  (test/linsolve.jl:230)
    np.testing.assert_allclose(A @ xh + info.residual.to_host(), b, atol=1e-10)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-6, atol=1e-13)
    np.testing.assert_allclose(xh, ox, rtol=1e-8, atol=1e-10)
    # converged solve
    alg2 = kk.GMRES(orth=orth, krylovdim=40, maxiter=100, tol=1e-10, verbosity=0)
    x2, info2 = kk.linsolve(op, ctx.from_host(b), None, alg2, 0.5, 1.5)
    assert info2.converged == 1
    x2h = x2.to_host()
    assert np.linalg.norm(0.5 * x2h + 1.5 * (A @ x2h) - b) < 1e-9
    ctx.close()


@pytest.mark.parametrize("literal", [False, True])
def test_gmres_singular_in_krylov_subspace_branch(literal):
    """gmres.jl:79-86: when hypot(R[k,k], α₁·normres) < tol the weight is rotated into y[k+1] with
    Givens(k+1, k, ...) and the cheap restart (:110-117) still runs.  Same numops / x / residual as the oracle."""
    import scipy.sparse as sp
    from krylovkit_jl_b200 import linsolve as ls
    n = 40
    A = sp.lil_matrix((n, n))
    A[1, 0] = 1.0
    A[2, 1] = 1e-6                      # A e2 = 1e-6 e3: R[2,2] = 0 and normres = 1e-6 < tol at step 2
    for i in range(3, n):
        A[i, i] = 1.0 + 0.01 * i
    A = A.tocsr()
    b = np.zeros(n)
    b[0] = 1.0
    ls.LITERAL_GIVENS_RESTART = literal
    try:
        ctx = kk.B200Context(n, 24)
        op = kk.B200CSR.from_scipy(ctx, A)
        alg = kk.GMRES(orth=kk.mgs2, krylovdim=6, maxiter=3, tol=1e-3, verbosity=0)
        x, info = kk.linsolve(op, ctx.from_host(b), None, alg)
        ox, oinfo = ko.linsolve_gmres(A, b, None, krylovdim=6, maxiter=3, tol=1e-3, orth=ko.Orth(ko.MGS2))
    finally:
        ls.LITERAL_GIVENS_RESTART = False
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    assert info.converged == oinfo["converged"]
    np.testing.assert_allclose(x.to_host(), ox, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(info.residual.to_host(), oinfo["residual"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-9, atol=1e-14)
    ctx.close()


@pytest.mark.parametrize("pair", [PAIRS[2], PAIRS[3], PAIRS[4]], ids=["cgs2", "mgs2", "cgsr"])
def test_svdsolve_matches_oracle_f64(pair):
    orth, oorth = pair
    m, n = 3001, 120
    rng = np.random.default_rng(11)
    A = rng.standard_normal((m, n))
    u0 = rng.standard_normal(m)
    alg = kk.GKL(orth=orth, krylovdim=25, maxiter=100, tol=1e-10, verbosity=0)
    S, Lv, Rv, info = kk.svdsolve(A, u0, 5, "LR", alg)
    oS, _, _, oinfo = ko.svdsolve_gkl(A, u0, 5, "LR", krylovdim=25, maxiter=100, tol=1e-10, orth=oorth)
    ref = np.linalg.svd(A, compute_uv=False)
    assert info.converged >= 5
    np.testing.assert_allclose(S[:5], ref[:5], rtol=1e-10)
    np.testing.assert_allclose(S[:5], oS[:5], rtol=1e-10)
    U, V = np.column_stack(Lv), np.column_stack(Rv)
    c = U.shape[1]
    assert np.abs(U.T @ U - np.eye(c)).max() < 1e-9
    np.testing.assert_allclose(A.T @ U, V * S[:c], atol=1e-8)
    Rm = np.column_stack(info.residual)
    np.testing.assert_allclose(A @ V, U * S[:c] + Rm, atol=1e-8)


def test_svdsolve_config4_small_f32():
    """config 4 at test size: dense tall Float32, 6 triplets, GKL(krylovdim=30, tol=1e-5)."""
    m, n = 20000, 512
    A = ko.dense_splitmix(SEED, m, n)
    u0 = ko.splitmix_vector(SEED + 1, m, dtype=np.float32)
    alg = kk.GKL(orth=kk.cgs2, krylovdim=30, maxiter=100, tol=1e-5, verbosity=0)
    ctx = kk.B200Context(m, 56, dtype=np.float32)
    sv = ctx.add_space(n, 48, sharded=False)
    op = kk.B200Dense.splitmix(ctx, m, n, SEED, sv)
    S, Lv, Rv, info = kk.svdsolve(op, ctx.from_host(u0), 6, "LR", alg)
    ref = np.linalg.svd(A.astype(np.float64), compute_uv=False)
    assert info.converged >= 6
    np.testing.assert_allclose(S[:6], ref[:6], rtol=3e-5)
    u, v = Lv[0].to_host().astype(np.float64), Rv[0].to_host().astype(np.float64)
    assert np.linalg.norm(A.astype(np.float64) @ v - S[0] * u) < 1e-3 * S[0]
    ctx.close()


def test_block_primitives_gpu():
    n, p, k = 5003, 5, 12
    rng = np.random.default_rng(12)
    ctx = kk.B200Context(n, 40)
    import ctypes as C
    from krylovkit_jl_b200.vectors import handles
    Xh = rng.standard_normal((n, p))
    Yh = rng.standard_normal((n, p))
    X = [ctx.from_host(Xh[:, j]) for j in range(p)]
    Y = [ctx.from_host(Yh[:, j]) for j in range(p)]
    M = np.zeros((p, p), order="F")
    ctx.check(ctx.lib.b2k_block_inner(ctx.h, handles(X), p, handles(Y), p,
                                      M.ctypes.data_as(C.POINTER(C.c_double))))
    np.testing.assert_allclose(M, Xh.T @ Yh, rtol=1e-12, atol=1e-10)
    Q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    V = [ctx.from_host(Q[:, j]) for j in range(k)]
    ctx.check(ctx.lib.b2k_block_reorthogonalize(ctx.h, handles(X), p, handles(V), k))
    Xr = np.column_stack([x.to_host() for x in X])
    assert np.abs(Q.T @ Xr).max() < 1e-11
    # block_qr with a dependent column
    Zh = rng.standard_normal((n, p))
    Zh[:, 3] = 2 * Zh[:, 0] - Zh[:, 1]
    Z = [ctx.from_host(Zh[:, j]) for j in range(p)]
    R = np.zeros((p, p), order="F")
    good = (C.c_int32 * p)()
    drift = C.c_int32()
    ctx.check(ctx.lib.b2k_block_qr(ctx.h, handles(Z), p, 1e-8, R.ctypes.data_as(C.POINTER(C.c_double)),
                                   good, C.byref(drift)))
    oR, ogood, odrift = ko.block_qr([Zh[:, j].copy() for j in range(p)], 1e-8)
    assert [i for i in range(p) if good[i]] == ogood == [0, 1, 2, 4]
    Qz = np.column_stack([Z[i].to_host() for i in ogood])
    np.testing.assert_allclose(Qz @ R[ogood, :], Zh, atol=1e-8)
    np.testing.assert_allclose(R[ogood, :], oR, rtol=1e-8, atol=1e-8)
    ctx.close()


@pytest.mark.parametrize("fused", [True, False])
def test_cg_matches_oracle(fused):
    """SURVEY §8f-2: conjugate gradients (src/linsolve/cg.jl) — fused one-sync step and the literal
    VectorInterface mirror against the oracle: same iteration count, same solution."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    nx, ny = 70, 45
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    b = A @ np.ones(n)
    ls.USE_FUSED_CG = fused
    ctx = kk.B200Context(n, 16)
    op = kk.B200CSR.from_scipy(ctx, A)
    for (a0, a1) in ((0.0, 1.0), (0.3, 1.5)):
        alg = kk.CG(maxiter=1000, tol=1e-10, verbosity=0)
        x, info = kk.linsolve(op, ctx.from_host(b), None, alg, a0, a1)
        ox, oinfo = ko.linsolve_cg(A, b, None, maxiter=1000, tol=1e-10, a0=a0, a1=a1)
        assert info.converged == 1 and oinfo["converged"] == 1
        assert abs(info.numiter - oinfo["numiter"]) <= 1 and info.numops == info.numiter + 1
        xh = x.to_host()
        np.testing.assert_allclose(xh, ox, rtol=1e-8, atol=1e-9)
        assert np.linalg.norm(a0 * xh + a1 * (A @ xh) - b) < 1e-8
        np.testing.assert_allclose(info.residual.to_host(), b - (a0 * xh + a1 * (A @ xh)), atol=1e-9)
    # non-converged, fixed iterations: residual identity b - A x = r
    alg = kk.CG(maxiter=7, tol=1e-14, verbosity=0)
    x, info = kk.linsolve(op, ctx.from_host(b), None, alg)
    ox, oinfo = ko.linsolve_cg(A, b, None, maxiter=7, tol=1e-14)
    assert info.converged == 0 and info.numiter == 7
    np.testing.assert_allclose(x.to_host(), ox, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-9)
    # the first iteration never looks at maxiter (cg.jl:35-60): maxiter = 1 still does two
    x, info = kk.linsolve(op, ctx.from_host(b), None, kk.CG(maxiter=1, tol=1e-300, verbosity=0))
    ox, oinfo = ko.linsolve_cg(A, b, None, maxiter=1, tol=1e-300)
    assert info.numiter == oinfo["numiter"] == 2 and info.numops == oinfo["numops"] == 3
    np.testing.assert_allclose(x.to_host(), ox, rtol=1e-10, atol=1e-12)
    ls.USE_FUSED_CG = True
    ctx.close()


@pytest.mark.parametrize("fused", [True, False])
def test_bicgstab_matches_oracle_and_reference_properties(fused):
    """SURVEY §8f-2: BiCGStab (src/linsolve/bicgstab.jl) on a nonsymmetric sparse operator, through the
    fused two-call step (b2k_bicgstab_half/_full) and through the literal VectorInterface sequence — the
    properties test/linsolve.jl:287-403 checks (converged, b = (a0 + a1 A) x, warm restart costs one
    operator application, non-converged run satisfies b = A x + r) plus step-for-step agreement
    with the oracle."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    saved = ls.USE_FUSED_BICGSTAB
    ls.USE_FUSED_BICGSTAB = fused
    rng = np.random.default_rng(11)
    n = 4000
    # convection-diffusion-like: 1-D Laplacian + skew part, diagonally dominant
    A = (sp.diags([-1.3, 2.6, -0.7], [-1, 0, 1], shape=(n, n)) +
         sp.random(n, n, density=2e-3, random_state=3) * 0.05).tocsr()
    b = rng.random(n)
    tol = 1e-12 * np.linalg.norm(b)
    ctx = kk.B200Context(n, 20)
    op = kk.B200CSR.from_scipy(ctx, A)
    for (a0, a1) in ((0.0, 1.0), (1.4, 0.6)):
        alg = kk.BiCGStab(maxiter=4 * n, tol=tol, verbosity=0)
        x, info = kk.linsolve(op, ctx.from_host(b), None, alg, a0, a1)
        ox, oinfo = ko.linsolve_bicgstab(A, b, None, maxiter=4 * n, tol=tol, a0=a0, a1=a1)
        assert info.converged == 1 and oinfo["converged"] == 1
        assert abs(info.numiter - oinfo["numiter"]) <= 1
        xh = x.to_host()
        np.testing.assert_allclose(xh, ox, rtol=1e-8, atol=1e-10)
        assert np.linalg.norm(a0 * xh + a1 * (A @ xh) - b) < 10 * tol
        np.testing.assert_allclose(info.residual.to_host(), b - (a0 * xh + a1 * (A @ xh)), atol=1e-11)
        # restart from the solution: one application, immediately converged (linsolve.jl:328-332)
        x2, info2 = kk.linsolve(op, ctx.from_host(b), x, alg, a0, a1)
        assert info2.numops == 1 and info2.converged == 1
    # fixed, too small iteration budget: identical iterates and the residual identity (:360-366)
    alg = kk.BiCGStab(maxiter=3, tol=1e-300, verbosity=0)
    x, info = kk.linsolve(op, ctx.from_host(b), None, alg)
    ox, oinfo = ko.linsolve_bicgstab(A, b, None, maxiter=3, tol=1e-300)
    assert info.converged == 0 and info.numiter == 3 == oinfo["numiter"] and info.numops == oinfo["numops"]
    np.testing.assert_allclose(x.to_host(), ox, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(A @ x.to_host() + info.residual.to_host(), b, atol=1e-12)
    # maxiter is first consulted in the second iteration (bicgstab.jl:170 sits inside the loop)
    x, info = kk.linsolve(op, ctx.from_host(b), None, kk.BiCGStab(maxiter=1, tol=1e-300, verbosity=0))
    assert info.numiter == 2
    # f32
    ctx32 = kk.B200Context(n, 20, dtype=np.float32)
    op32 = kk.B200CSR.from_scipy(ctx32, A.astype(np.float32))
    b32 = b.astype(np.float32)
    x, info = kk.linsolve(op32, ctx32.from_host(b32), None,
                          kk.BiCGStab(maxiter=4 * n, tol=1e-5 * float(np.linalg.norm(b32)), verbosity=0))
    assert info.converged == 1
    assert np.linalg.norm(A @ x.to_host().astype(np.float64) - b) < 1e-4 * np.linalg.norm(b)
    ctx32.close()
    ctx.close()
    ls.USE_FUSED_BICGSTAB = saved


@pytest.mark.parametrize("orth", ["mgs", "cgs2", "mgsr"])
def test_lsmr_matches_oracle_and_reference_properties(orth):
    """SURVEY §8f-2: LSMR (src/lssolve/lsmr.jl) — test/lssolve.jl's assertions through the device
    path (dense operator with two vector spaces, and a rectangular sparse (A, Aᵀ) pair), and
    iterate-for-iterate agreement with the oracle including the sliding reorthogonalisation ring."""
    o = getattr(kk, orth)
    oo = ko.Orth(o.tag, o.eta) if o.is_ir else ko.Orth(o.tag)
    rng = np.random.default_rng(21)
    n, N = 10, 100
    A = rng.random((2 * n, n))
    U, S, Vt = np.linalg.svd(A, full_matrices=False)
    invS = 1 / S
    S[-1] = 0
    invS[-1] = 0
    A = U @ np.diag(S) @ Vt
    b = rng.random(2 * n)
    tol = 10 * n * np.finfo(float).eps
    # host entry, no reorthogonalisation, three iterations
    x, info = kk.lssolve(A, b, kk.LSMR(orth=o, maxiter=3, krylovdim=1, verbosity=0))
    ox, oinfo = ko.lssolve_lsmr(A, b, maxiter=3, krylovdim=1, orth=oo)
    r = b - A @ x
    np.testing.assert_allclose(info.residual, r, atol=1e-13)
    np.testing.assert_allclose(info.normres, np.linalg.norm(A.T @ r), rtol=1e-8)
    assert info.converged == 0 and info.numops == oinfo["numops"] == 7
    np.testing.assert_allclose(x, ox, rtol=1e-11, atol=1e-14)
    # full reorthogonalisation: minimum-norm solution within n iterations
    alg = kk.LSMR(orth=o, maxiter=n, tol=tol, krylovdim=n, verbosity=0)
    x, info = kk.lssolve(A, b, alg)
    assert info.converged > 0
    assert abs(Vt[-1] @ x) < tol
    np.testing.assert_allclose(x, Vt.T @ np.diag(invS) @ U.T @ b, rtol=1e-8)
    lam = 0.37
    x, info = kk.lssolve(A, b, alg, lam)
    assert info.converged > 0
    np.testing.assert_allclose(A.T @ (b - A @ x), lam ** 2 * x, atol=2 * tol)
    # large problem, ring of 5 (exercises slot replacement), against the oracle
    A = rng.random((2 * N, N)) - 0.5
    b = rng.random(2 * N) - 0.5
    tol = 10 * N * np.finfo(float).eps
    x, info = kk.lssolve(A, b, kk.LSMR(orth=o, maxiter=N, tol=tol, krylovdim=5, verbosity=0))
    ox, oinfo = ko.lssolve_lsmr(A, b, maxiter=N, tol=tol, krylovdim=5, orth=oo)
    assert info.converged > 0 and abs(info.numiter - oinfo["numiter"]) <= 2
    assert np.linalg.norm(A.T @ (b - A @ x)) < 5 * tol
    np.testing.assert_allclose(x, ox, rtol=1e-8, atol=1e-11)
    x12, info12 = kk.lssolve(A, b, kk.LSMR(orth=o, maxiter=12, tol=0.0, krylovdim=5, verbosity=0))
    ox12, oinfo12 = ko.lssolve_lsmr(A, b, maxiter=12, tol=0.0, krylovdim=5, orth=oo)
    np.testing.assert_allclose(x12, ox12, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(info12.normres, oinfo12["normres"], rtol=1e-8)
    # issue #133 (test/issues.jl:21-29): literal fixture
    x, info = kk.lssolve(np.eye(2), np.array([1.0, 0.0]), kk.LSMR(orth=o, verbosity=0))
    assert np.array_equal(x, [1.0, 0.0])
    assert info.converged == 1 and info.numiter == 1 and info.numops == 2 and info.normres == 0.0
    # sparse rectangular operator as an (A, Aᵀ) pair
    As = sp.random(3000, 800, density=0.01, random_state=4).tocsr() + sp.eye(3000, 800).tocsr()
    bs = rng.random(3000)
    tol = 1e-10
    x, info = kk.lssolve(As, bs, kk.LSMR(orth=o, maxiter=400, tol=tol, krylovdim=8, verbosity=0))
    assert info.converged > 0
    assert np.linalg.norm(As.T @ (bs - As @ x)) < 50 * tol
    np.testing.assert_allclose(info.residual, bs - As @ x, atol=1e-10)


def _mat_with_eigrepetition(rng, N, mult):
    """test/testsetup.jl:46-58: symmetric matrix with repeated extremal eigenvalues."""
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    D = np.sort(rng.standard_normal(N))
    i = 0
    while mult >= 2 and i + mult <= N // 2:
        D[i:i + mult] = D[i]
        D[N - i - mult:N - i] = D[N - i - 1]
        i += mult
        mult -= 1
    A = Q @ np.diag(D) @ Q.T
    return (A + A.T) / 2


def _dense_sym_op(ctx, A):
    return kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))


def test_blocklanczos_reference_properties():
    """SURVEY §8f-3 / test/eigsolve.jl:552-770 through the device path: full spectrum from both ends
    with repeated eigenvalues, orthonormal Ritz vectors, A v = λ v, agreement with the oracle, the
    single-vector block reproducing Lanczos (same numiter, numops + 1), and the restart improving
    accuracy."""
    rng = np.random.default_rng(17)
    n, N = 10, 100
    tol = 1e-12
    # --- full
    A = _mat_with_eigrepetition(rng, n, 2)
    X0 = [rng.random(n) for _ in range(2)]
    ev = np.linalg.eigvalsh(A)
    ctx = kk.B200Context(n, 128)
    op = _dense_sym_op(ctx, A)
    n1 = n // 2
    n2 = n - n1
    blk = lambda: kk.Block([ctx.from_host(x) for x in X0])
    D1, V1, info1 = kk.eigsolve(op, blk(), n1, "SR", kk.BlockLanczos(krylovdim=n, maxiter=1, tol=tol, verbosity=0))
    D2, V2, info2 = kk.eigsolve(op, blk(), n2, "LR", kk.BlockLanczos(krylovdim=2 * n, maxiter=4, tol=tol, verbosity=0))
    np.testing.assert_allclose(np.concatenate([D1[:n1], D2[:n2][::-1]]), ev, rtol=1e-9, atol=1e-11)
    for D, V in ((D1, V1), (D2, V2)):
        Uh = np.column_stack([v.to_host() for v in V])
        np.testing.assert_allclose(Uh.T @ Uh, np.eye(Uh.shape[1]), atol=1e-9)
        np.testing.assert_allclose(A @ Uh, Uh * D, atol=1e-9)
    oD1, _, oinfo1 = ko.eigsolve_blocklanczos(A, X0, n1, "SR", krylovdim=n, maxiter=1, tol=tol)
    np.testing.assert_allclose(D1, oD1, rtol=1e-9, atol=1e-11)
    assert info1.numops == oinfo1["numops"] and info1.converged == oinfo1["converged"]
    with pytest.raises(ValueError):
        kk.eigsolve(op, blk(), n + 1, "SR", kk.BlockLanczos(krylovdim=n, verbosity=0))
    ctx.close()
    # --- iterative, eager, block of 4 with multiplicity 4
    A = _mat_with_eigrepetition(rng, N, 4)
    X0 = [rng.random(N) for _ in range(4)]
    ev = np.linalg.eigvalsh(A)
    ctx = kk.B200Context(N, 800)
    op = _dense_sym_op(ctx, A)
    blk = lambda: kk.Block([ctx.from_host(x) for x in X0])
    alg = kk.BlockLanczos(krylovdim=N, maxiter=10, tol=tol, eager=True, verbosity=0)
    D1, V1, info1 = kk.eigsolve(op, blk(), n, "SR", alg)
    D2, V2, info2 = kk.eigsolve(op, blk(), n, "LR", alg)
    l1, l2 = info1.converged, info2.converged
    assert l1 >= n and l2 >= n
    np.testing.assert_allclose(D1[:l1], ev[:l1], rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(D2[:l2], ev[::-1][:l2], rtol=1e-9, atol=1e-10)
    U1 = np.column_stack([v.to_host() for v in V1])
    np.testing.assert_allclose(U1.T @ U1, np.eye(U1.shape[1]), atol=1e-9)
    R1 = np.column_stack([r.to_host() for r in info1.residual])
    np.testing.assert_allclose(A @ U1, U1 * D1 + R1, atol=1e-9)
    # --- shrink makes it better (:741-770)
    A = _mat_with_eigrepetition(rng, N, 5)
    X0 = [rng.random(N) for _ in range(5)]
    v0 = np.linalg.eigvalsh(A)[:n]
    op = _dense_sym_op(ctx, A)
    va, _, _ = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), n, "SR",
                           kk.BlockLanczos(krylovdim=3 * n // 2, maxiter=1, tol=1e-12, verbosity=0))
    vb, _, infob = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), n, "SR",
                               kk.BlockLanczos(krylovdim=3 * n // 2, maxiter=2, tol=1e-12, verbosity=0))
    assert np.linalg.norm(vb[:n // 2] - v0[:n // 2]) < np.linalg.norm(va[:n // 2] - v0[:n // 2])
    ovb, _, oinfob = ko.eigsolve_blocklanczos(A, X0, n, "SR", krylovdim=3 * n // 2, maxiter=2, tol=1e-12)
    np.testing.assert_allclose(vb, ovb, rtol=1e-8, atol=1e-9)
    assert infob.numops == oinfob["numops"] and infob.numiter == oinfob["numiter"] == 2
    ctx.close()
    # --- block size 1 reproduces Lanczos (:685-712)
    A = rng.random((2 * N, 2 * N)) - 0.5
    A = (A + A.T) / 2
    x0 = rng.random(2 * N)
    ctx = kk.B200Context(2 * N, 200)
    op = _dense_sym_op(ctx, A)
    e1, _, j1 = kk.eigsolve(op, ctx.from_host(x0), n, "SR",
                            kk.Lanczos(krylovdim=2 * n, maxiter=10, tol=tol, verbosity=0))
    e2, _, j2 = kk.eigsolve(op, kk.Block([ctx.from_host(x0)]), n, "SR",
                            kk.BlockLanczos(krylovdim=2 * n, maxiter=10, tol=tol, verbosity=0))
    assert j1.converged == j2.converged and j1.numiter == j2.numiter and j1.numops + 1 == j2.numops
    np.testing.assert_allclose(j1.normres, j2.normres[:len(j1.normres)], atol=1e-9)
    np.testing.assert_allclose(e1[:j1.converged], e2[:j2.converged], rtol=1e-9, atol=1e-11)
    ctx.close()


def test_blocklanczos_toric_code_degenerate_ground_space():
    """test/eigsolve.jl:471-549: −H of the 3×3 toric code (2^18 states) has a four-fold degenerate
    lowest eigenvalue −16, which a block of 5 resolves in one sweep (krylovdim 100, no restart); a
    second run with krylovdim 60 and restarts exercises the wide (K > 96 columns not needed) and the
    thick-restart path at scale."""
    H = ko.toric_code_hamiltonian(3, 3)
    M = H.shape[0]
    rng = np.random.default_rng(1)
    X0 = [rng.random(M) for _ in range(5)]
    # every converged Ritz pair is returned (here ~80 of the 100), each with its residual vector
    ctx = kk.B200Context(M, 480)
    op = kk.B200CSR.from_scipy(ctx, (-H).tocsr())
    alg = kk.BlockLanczos(tol=1e-6, maxiter=1, verbosity=0)
    D, U, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 10, "SR", alg)
    assert np.sum(np.abs(D[:10] + 16.0) < 2.0 - 1e-6) == 4
    assert np.sum(np.abs(D[:10] + 16.0) < 1e-6) == 4
    assert len(U) == max(10, info.converged) and len(info.residual) == len(U)
    del U, info
    # map input: any callable on device vectors
    D, U, info = kk.eigsolve(lambda x: op(x), kk.Block([ctx.from_host(x) for x in X0]), 10, "SR", alg)
    assert np.sum(np.abs(D[:10] + 16.0) < 1e-6) == 4
    del U, info
    alg = kk.BlockLanczos(tol=1e-8, krylovdim=40, maxiter=30, verbosity=0)
    D, U, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
    assert info.converged >= 4 and info.numiter > 1
    np.testing.assert_allclose(D[:4], -16.0, atol=1e-7)
    G = np.column_stack([u.to_host() for u in U[:4]])
    np.testing.assert_allclose(G.T @ G, np.eye(4), atol=1e-7)
    ctx.close()


@pytest.mark.parametrize("orth", ["cgs2", "mgs2", "cgsr", "mgsr"])
def test_arnoldi_eigsolve_and_schursolve(orth):
    """SURVEY §8f-4 / test/eigsolve.jl:138-300 through the device path: non-symmetric real operator,
    complex Ritz pairs returned as (re, im) device vectors; SR half + LR half = eigvals(A), A V = V D,
    orthonormal Schur vectors with A Q = Q T; restarted runs agree with the oracle's values."""
    o = getattr(kk, orth)
    oo = ko.Orth(o.tag, o.eta) if o.is_ir else ko.Orth(o.tag)
    rng = np.random.default_rng(31)
    n, N, tol = 10, 100, 1e-12
    A = rng.random((n, n)) - 0.5
    v = rng.random(n)
    n1 = n // 2
    n2 = n - n1
    ctx = kk.B200Context(n, 120)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    D1, V1, i1 = kk.eigsolve(op, ctx.from_host(v), n1, "SR", kk.Arnoldi(orth=o, krylovdim=n, maxiter=1, tol=tol, verbosity=0))
    D2, V2, i2 = kk.eigsolve(op, ctx.from_host(v), n2, "LR", kk.Arnoldi(orth=o, krylovdim=2 * n, maxiter=1, tol=tol, verbosity=0))
    def srt(D):
        D = np.asarray(D)
        D = D[np.argsort(-D.imag, kind="stable")]
        return D[np.argsort(D.real, kind="stable")]
    D2s = srt(D2)
    np.testing.assert_allclose(np.concatenate([D1[:n1], D2s[len(D2s) - n2:]]), srt(np.linalg.eigvals(A)),
                               rtol=1e-9, atol=1e-11)
    for D, V in ((D1, V1), (D2, V2)):
        Uh = np.column_stack([x.to_host() for x in V])
        np.testing.assert_allclose(A @ Uh, Uh * D, atol=1e-9)
    oD1, _, oi1 = ko.eigsolve_arnoldi(A, v, n1, "SR", krylovdim=n, maxiter=1, tol=tol, orth=oo)
    np.testing.assert_allclose(D1, oD1, rtol=1e-9, atol=1e-11)
    assert i1.numops == oi1["numops"] and i1.converged == oi1["converged"]
    T, Q, vals, info = kk.schursolve(op, ctx.from_host(v), n1, "SR", kk.Arnoldi(orth=o, krylovdim=n, maxiter=1, tol=tol, verbosity=0))
    Qh = np.column_stack([q.to_host() for q in Q])
    np.testing.assert_allclose(Qh.T @ Qh, np.eye(Qh.shape[1]), atol=1e-10)
    np.testing.assert_allclose(A @ Qh, Qh @ T, atol=1e-9)
    np.testing.assert_allclose(vals, D1[:len(vals)], rtol=1e-9, atol=1e-11)
    ctx.close()
    # restarts
    A = rng.random((N, N)) - 0.5
    v = rng.random(N)
    ctx = kk.B200Context(N, 200)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    Dfull = np.linalg.eigvals(A)
    Dfull = Dfull[np.argsort(-Dfull.imag, kind="stable")]
    for which, key in (("SR", lambda d: d.real), ("LR", lambda d: -d.real), ("LM", lambda d: -np.abs(d))):
        alg = kk.Arnoldi(orth=o, krylovdim=3 * n, maxiter=20, tol=tol, eager=True, verbosity=0)
        Dw, Vw, iw = kk.eigsolve(op, ctx.from_host(v), n, which, alg)
        l = iw.converged
        assert l > 0 and iw.numiter > 1
        want = Dfull[np.argsort(key(Dfull), kind="stable")][:l]
        if which == "LM":
            np.testing.assert_allclose(np.abs(Dw[:l]), np.abs(want), rtol=1e-8)
        else:
            np.testing.assert_allclose(Dw[:l], want, rtol=1e-8, atol=1e-10)
        Uw = np.column_stack([x.to_host() for x in Vw])
        Rw = np.column_stack([x.to_host() for x in iw.residual])
        np.testing.assert_allclose(A @ Uw, Uw * Dw + Rw, atol=1e-9)
        np.testing.assert_allclose(iw.normres, np.linalg.norm(Rw, axis=0), rtol=1e-6, atol=1e-13)
        del Vw, iw
    ctx.close()


def test_realeigsolve():
    """test/eigsolve.jl:330-440 through the device path: real spectrum in, real eigenpairs out; a complex
    pair among the requested values is flattened with a warning."""
    from scipy.linalg import expm
    rng = np.random.default_rng(5)
    n, N = 10, 100
    V = expm(rng.standard_normal((N, N)) / 10)
    D = rng.standard_normal(N)
    A = V @ np.diag(D) @ np.linalg.inv(V)
    v = rng.random(N)
    ctx = kk.B200Context(N, 120)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    alg = kk.Arnoldi(krylovdim=3 * n, maxiter=20, tol=1e-12, eager=True, verbosity=0)
    for which, want in (("SR", np.sort(D)), ("LR", np.sort(D)[::-1]), ("LM", D[np.argsort(-np.abs(D))])):
        D1, V1, i1 = kk.realeigsolve(op, ctx.from_host(v), n, which, alg)
        oD1, _, oi1 = ko.realeigsolve_arnoldi(A, v, n, which, krylovdim=3 * n, maxiter=20, tol=1e-12, eager=True)
        l = i1.converged
        assert l > 0 and D1.dtype == np.float64
        np.testing.assert_allclose(D1[:l], want[:l], rtol=1e-8, atol=1e-10)
        m = min(l, oi1["converged"])
        np.testing.assert_allclose(D1[:m], oD1[:m], rtol=1e-8, atol=1e-10)
        U1 = np.column_stack([x.to_host() for x in V1])
        R1 = np.column_stack([x.to_host() for x in i1.residual])
        np.testing.assert_allclose(A @ U1, U1 * D1 + R1, atol=1e-9)
        del V1, i1
    ctx.close()
    ctx = kk.B200Context(2, 16)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(np.array([[1.0, -1.0], [1.0, 1.0]])))
    with pytest.warns(UserWarning, match="2 x 2 Schur block"):
        D1, _, _ = kk.realeigsolve(op, ctx.from_host(np.array([1.0, 0.3])), 1, "LM", kk.Arnoldi(tol=1e-8, verbosity=1))
    np.testing.assert_allclose(D1, 1.0)
    ctx.close()


def _phi(A, v, p):
    """ϕ_p(A) v through the augmented-matrix exponential — test/expintegrator.jl:1-13."""
    from scipy.linalg import expm
    m = A.shape[0]
    if p == 0:
        return expm(A) @ v
    Ap = np.zeros((m + p, m + p))
    Ap[:m, :m] = A
    Ap[:m, m] = v
    for k in range(1, p):
        Ap[m + k - 1, m + k] = 1
    return expm(Ap)[:m, -1]


@pytest.mark.parametrize("method", ["lanczos", "arnoldi"])
def test_exponentiate_and_expintegrator(method):
    """SURVEY §8f-4 / test/expintegrator.jl:15-190 (real time steps): exponentiate reproduces exp(A)
    column by column; expintegrator reproduces Σ_j t^j ϕ_j(tA) u_j for p = 1..5 in the full-space and in
    the restarted (krylovdim ≪ N, eager) regime; loose tolerance gives proportionally loose answers;
    the device result follows the oracle step for step."""
    from scipy.linalg import expm
    rng = np.random.default_rng(41)
    n, N = 10, 100
    Alg = kk.Lanczos if method == "lanczos" else kk.Arnoldi
    for orth in ("cgs2", "mgs2", "cgsr", "mgsr"):
        o = getattr(kk, orth)
        A = rng.random((n, n)) - 0.5
        if method == "lanczos":
            A = (A + A.T) / 2
        ctx = kk.B200Context(n, 80)
        op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
        alg = Alg(orth=o, krylovdim=n, maxiter=2, tol=1e-12, verbosity=0)
        W = np.zeros((n, n))
        for k in range(n):
            w, info = kk.exponentiate(op, 1.0, ctx.from_host(np.eye(n)[:, k]), alg)
            W[:, k] = w.to_host()
        np.testing.assert_allclose(W, expm(A), rtol=1e-9, atol=1e-11)
        for t in (rng.random(), -rng.random()):
            for p in range(1, 6):
                u = tuple(rng.random(n) for _ in range(p + 1))
                w, info = kk.expintegrator(op, t, tuple(ctx.from_host(x) for x in u), alg)
                w2 = expm(t * A) @ u[0]
                for j in range(1, p + 1):
                    w2 = w2 + t ** j * _phi(t * A, u[j], j)
                assert info.converged > 0
                np.testing.assert_allclose(w.to_host(), w2, rtol=1e-9, atol=1e-11)
        with pytest.raises(TypeError):
            kk.exponentiate(op, 1j, ctx.from_host(np.eye(n)[:, 0]), alg)
        ctx.close()
    A = 0.5 * (rng.random((N, N)) - 0.5)
    if method == "lanczos":
        A = (A + A.T) / 2
    ctx = kk.B200Context(N, 80)
    op = kk.B200CSR.from_scipy(ctx, sp.csr_matrix(A))
    restarts = 0
    for t in (0.9 + rng.random(), -0.9 - rng.random()):
        for p in range(1, 6):
            u = tuple(rng.random(N) for _ in range(p + 1))
            alg = Alg(krylovdim=n, maxiter=100, tol=1e-12, eager=True, verbosity=0)
            w, info = kk.expintegrator(op, t, tuple(ctx.from_host(x) for x in u), alg)
            ow, oinfo = ko.expintegrator(A, t, u, method, ko.Orth(ko.MGS2), krylovdim=n, maxiter=100, tol=1e-12, eager=True)
            w2 = expm(t * A) @ u[0]
            for j in range(1, p + 1):
                w2 = w2 + t ** j * _phi(t * A, u[j], j)
            assert info.converged > 0
            np.testing.assert_allclose(w.to_host(), w2, rtol=1e-8, atol=1e-10)
            np.testing.assert_allclose(w.to_host(), ow, rtol=1e-8, atol=1e-10)
            assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
            restarts += info.numiter - 1
            alg = Alg(krylovdim=n, maxiter=100, tol=1e-3, eager=True, verbosity=0)
            w, info = kk.expintegrator(op, t, tuple(ctx.from_host(x) for x in u), alg)
            np.testing.assert_allclose(w.to_host(), w2, atol=1e-2 * abs(t))
    assert restarts > 0
    ctx.close()


def test_invariant_subspace_early_exit():
    """eigsolve/lanczos.jl:38-44, 45: beta <= tol stops the expansion loop early (also inside
    b2k_lanczos_expand_many) and reports the exact eigenvalues of the invariant subspace."""
    n = 3000
    d = np.repeat([1.0, 2.5, 7.0], n // 3)
    A = sp.diags(d).tocsr()
    x0 = ko.splitmix_vector(5, n) + 0.5
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=20, maxiter=5, tol=1e-9, verbosity=0)
    ctx = kk.B200Context(n, 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0), 3, "SR", alg)
    ovals, _, oinfo = ko.eigsolve_lanczos(A, x0, 3, "SR", krylovdim=20, maxiter=5, tol=1e-9, orth=ko.Orth(ko.CGS2))
    assert info.numops == oinfo["numops"] == 3          # the Krylov space is exhausted after 3 vectors
    assert info.converged == 3
    np.testing.assert_allclose(vals, [1.0, 2.5, 7.0], rtol=1e-12)
    np.testing.assert_allclose(vals, ovals, rtol=1e-12)
    ctx.close()


def test_zero_start_vector_raises():
    """lanczos.jl:184: ArgumentError("initial vector should not have norm zero")."""
    ctx = kk.B200Context(100, 16)
    op = kk.B200CSR.stencil(ctx, 10, 10)
    with pytest.raises(ValueError):
        kk.eigsolve(op, ctx.zeros(), 1, "SR", kk.Lanczos(krylovdim=5, verbosity=0))
    ctx.close()


def _expand_many_run(chain, nx=97, ny=61, steps=30, tol=0.0, diag=None, orth=None):
    """initialize + one b2k_lanczos_expand_many batch; returns (alphas, betas, V (host), r (host), free columns).
    chain: False = one synchronous step at a time, True = the device-chained steps."""
    lib = L.load()
    lib.b2k_debug_set_chain(1 if chain else 0)
    try:
        n = nx * ny
        ctx = kk.B200Context(n, steps + 8)
        if diag is None:
            op = kk.B200CSR.stencil(ctx, nx, ny)
            x0 = ctx.from_host(ko.splitmix_vector(SEED, n))
        else:
            op = kk.B200CSR.from_scipy(ctx, sp.diags(diag).tocsr())
            x0 = ctx.from_host(ko.splitmix_vector(5, n) + 0.5)
        it = lz.LanczosIterator(op, x0, orth or kk.cgs2)
        used = lambda: lib.b2k_debug_used_columns(ctx.h, 0)
        f = lz.initialize(it)
        u0 = used()
        done = lz.expand_many_(it, f, steps, tol)
        # x0, the basis, the residual — and nothing else (the batch recycles columns internally)
        assert u0 == 3 and used() == 1 + len(f.V) + 1, (u0, used(), done, len(f.V), list(f.betas))
        out = (done, np.array(f.alphas), np.array(f.betas), np.column_stack([v.to_host() for v in f.V]),
               f.r.to_host())
        live = {"x0": hex(x0.handle), "V": [hex(v.handle) for v in f.V], "r": hex(f.r.handle)}
        del f, it, x0
        import gc
        gc.collect()
        assert used() == 0, (used(), live, [o for o in gc.get_objects() if type(o).__name__ == "B200Vec"])
        ctx.close()
        return out
    finally:
        lib.b2k_debug_set_chain(1)


def test_chained_lanczos_batch_is_bit_identical_to_stepping():
    """b2k_lanczos_expand_many with the device-chained steps (normalisation fused into the SpMV gather, scalars
    kept in device records, in-kernel finalisation, no host round trip) gives the same bits as one synchronous
    b2k_lanczos_expand per step: same kernels' arithmetic, same operand bits (lanczos.jl:250-272, 313-324)."""
    for orth in (kk.cgs2, kk.mgs2b):
        d1, a1, b1, V1, r1 = _expand_many_run(True, orth=orth)
        d0, a0, b0, V0, r0 = _expand_many_run(False, orth=orth)
        assert d1 == d0 == 30
        if orth is kk.cgs2:
            assert np.array_equal(a1, a0) and np.array_equal(b1, b0)
            assert np.array_equal(V1, V0) and np.array_equal(r1, r0)
        else:
            # the synchronous mgs2b step computes alpha with a separate dot kernel (other summation order than
            # the SpMV epilogue of the chained step): equal to rounding, not to the bit
            np.testing.assert_allclose(a1, a0, rtol=1e-13)
            np.testing.assert_allclose(b1, b0, rtol=1e-12)
            np.testing.assert_allclose(V1, V0, atol=1e-11)
        assert np.abs(V1.T @ V1 - np.eye(V1.shape[1])).max() < 1e-12


def test_chained_lanczos_batch_stops_at_breakdown_on_the_device():
    """beta <= tol in the middle of a batch (eigsolve/lanczos.jl:45): the kernels enqueued behind that step do
    nothing, the factorization is the one of the synchronous loop and the residual is intact."""
    n = 3000
    d = np.repeat([1.0, 2.5, 7.0, 11.0], n // 4)
    d0, a0, b0, V0, r0 = _expand_many_run(False, nx=n, ny=1, steps=12, tol=1e-9, diag=d)
    d1, a1, b1, V1, r1 = _expand_many_run(True, nx=n, ny=1, steps=12, tol=1e-9, diag=d)
    assert d1 == d0 == 3                    # 4 distinct eigenvalues: the Krylov space is exhausted at K = 4
    assert np.array_equal(a1, a0) and np.array_equal(b1, b0)
    assert np.array_equal(V1, V0) and np.array_equal(r1, r0)
    assert b1[-1] <= 1e-9


def test_blocklanczos_fast_block_mode_matches_reference_mode():
    """The flagged block mode (SpMM + block-classical Gram-Schmidt twice + CholeskyQR2) against the
    reference's arithmetic (modified Gram-Schmidt loops) and the oracle: same Ritz values after a fixed number of
    restart cycles, converged eigenpairs with the closed form, and the four-fold degenerate toric-code ground
    space (test/eigsolve.jl:471-549)."""
    nx, ny = 120, 91
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    X0 = [ko.splitmix_vector(100 + i, n) for i in range(4)]
    ctx = kk.B200Context(n, 120)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    res = {}
    for fast in (False, True):
        alg = kk.BlockLanczos(krylovdim=48, maxiter=4, tol=0.0, verbosity=0, fast_block=fast)
        vals, vecs, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
        res[fast] = (np.array(vals[:4]), info.numops)
        del vecs, info
    ovals, _, oinfo = ko.eigsolve_blocklanczos(A, X0, 4, "SR", krylovdim=48, maxiter=4, tol=0.0)
    assert res[False][1] == res[True][1] == oinfo["numops"]
    np.testing.assert_allclose(res[False][0], ovals[:4], rtol=1e-8)
    np.testing.assert_allclose(res[True][0], ovals[:4], rtol=1e-8)
    alg = kk.BlockLanczos(krylovdim=60, maxiter=200, tol=1e-10, verbosity=0, fast_block=True)
    vals, vecs, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
    assert info.converged >= 4
    np.testing.assert_allclose(vals[:4], ko.laplace_eigenvalues(nx, ny)[:4], rtol=1e-9)
    U = np.column_stack([v.to_host() for v in vecs[:4]])
    np.testing.assert_allclose(U.T @ U, np.eye(4), atol=1e-9)
    assert np.abs(A @ U - U * vals[:4]).max() < 1e-8
    ctx.close()
    H = ko.toric_code_hamiltonian(3, 3)
    rng = np.random.default_rng(1)
    X0 = [rng.random(H.shape[0]) for _ in range(5)]
    ctx = kk.B200Context(H.shape[0], 120)
    op = kk.B200CSR.from_scipy(ctx, (-H).tocsr())
    alg = kk.BlockLanczos(tol=1e-8, krylovdim=40, maxiter=30, verbosity=0, fast_block=True)
    D, U, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
    assert info.converged >= 4
    np.testing.assert_allclose(D[:4], -16.0, atol=1e-7)
    ctx.close()


def test_cg_chained_iterations_equal_stepwise():
    """b2k_cg_chain (rho, beta, <p,q>, ||r|| on the device; one host sync per 32 iterations; convergence test on the
    device) gives the same iterates as one b2k_cg_step per iteration: same numiter / numops, same x bit for bit."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    nx, ny = 181, 97
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    b = A @ np.ones(n) + 0.01 * ko.splitmix_vector(3, n)
    ctx = kk.B200Context(n, 16)
    op = kk.B200CSR.from_scipy(ctx, A)
    out = {}
    try:
        for chain in (True, False):
            ls.USE_CG_CHAIN = chain
            res = []
            for alg in (kk.CG(maxiter=2000, tol=1e-9, verbosity=0), kk.CG(maxiter=45, tol=1e-300, verbosity=0)):
                x, info = kk.linsolve(op, ctx.from_host(b), None, alg, 0.1, 1.2)
                res.append((x.to_host(), info.numiter, info.numops, info.converged, info.normres))
            out[chain] = res
    finally:
        ls.USE_CG_CHAIN = True
    for (x1, it1, ops1, c1, nr1), (x0, it0, ops0, c0, nr0) in zip(out[True], out[False]):
        assert (it1, ops1, c1) == (it0, ops0, c0)
        assert np.array_equal(x1, x0) and nr1 == nr0
    assert out[True][0][3] == 1 and out[True][1][3] == 0 and out[True][1][1] == 45
    ctx.close()


def test_bicgstab_chained_iterations_equal_stepwise():
    """b2k_bicgstab_chain (rho, rho_old, alpha, omega on the device; both convergence tests of an iteration made by
    the kernels; one host sync per 32 iterations) gives the same iterates as b2k_bicgstab_half/_full called in turn:
    same numiter / numops / converged, same x bit for bit — for a converging run (which ends through one of the two
    device-side tests), a fixed iteration budget, and a tolerance the half step meets first."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    rng = np.random.default_rng(5)
    n = 6000
    A = (sp.diags([-1.3, 2.6, -0.7], [-1, 0, 1], shape=(n, n)) +
         sp.random(n, n, density=1e-3, random_state=4) * 0.05).tocsr()
    b = rng.random(n)
    nb = float(np.linalg.norm(b))
    ctx = kk.B200Context(n, 20)
    op = kk.B200CSR.from_scipy(ctx, A)
    algs = [kk.BiCGStab(maxiter=4 * n, tol=1e-12 * nb, verbosity=0), kk.BiCGStab(maxiter=37, tol=1e-300, verbosity=0),
            kk.BiCGStab(maxiter=4 * n, tol=3e-4 * nb, verbosity=0), kk.BiCGStab(maxiter=4 * n, tol=1e-9 * nb, verbosity=0)]
    out = {}
    try:
        for chain in (True, False):
            ls.USE_BICGSTAB_CHAIN = chain
            res = []
            for alg in algs:
                x, info = kk.linsolve(op, ctx.from_host(b), None, alg, 0.2, 0.9)
                res.append((x.to_host(), info.numiter, info.numops, info.converged, info.normres))
            out[chain] = res
    finally:
        ls.USE_BICGSTAB_CHAIN = True
    for (x1, it1, ops1, c1, nr1), (x0, it0, ops0, c0, nr0) in zip(out[True], out[False]):
        assert (it1, ops1, c1) == (it0, ops0, c0), ((it1, ops1, c1), (it0, ops0, c0))
        assert np.array_equal(x1, x0) and nr1 == nr0
    assert [r[3] for r in out[True]] == [1, 0, 1, 1] and out[True][1][1] == 37
    # both exits are taken: run 0 ends through the full-step test (numops = 2 numiter + 2), run 3 through the half step
    assert out[True][0][2] == 2 * out[True][0][1] + 2 and out[True][3][2] == 2 * out[True][3][1] + 1
    ctx.close()


def test_chained_step_event_trace():
    """b2k_debug_trace: the kernels of a device-chained batch record one event per stage and step (SpMV begin / halo
    present / CTA 0 done / <v,Av> published; sweep begin / alpha present / two phases, one boundary / finaliser in
    and out), in time order within a step; with the trace off nothing is recorded."""
    import ctypes as C
    lib = L.load()
    nx, ny, steps = 301, 97, 12
    ctx = kk.B200Context(nx * ny, steps + 8)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    it = lz.LanczosIterator(op, ctx.from_host(ko.splitmix_vector(SEED, nx * ny)), kk.cgs2)
    f = lz.initialize(it)
    ctx.check(lib.b2k_debug_trace(ctx.h, 1))
    done = lz.expand_many_(it, f, steps, 0.0)
    assert done == steps
    buf = (C.c_uint64 * (2 * 4096))()
    n = C.c_int64()
    ctx.check(lib.b2k_debug_trace_read(ctx.h, buf, 4096, C.byref(n)))
    ev = np.frombuffer(buf, dtype=np.uint64)[: 2 * n.value].reshape(-1, 2).astype(np.int64)
    ev = ev[np.argsort(ev[:, 0], kind="stable")]
    codes = ev[:, 1].tolist()
    per_step = [1, 2, 3, 4, 10, 11, 12, 15, 13, 18, 19]       # two phases: prologue + projection | update + norm
    assert n.value == steps * len(per_step), (n.value, codes[:30])
    assert sorted(codes) == sorted(per_step * steps)
    starts = [i for i, c in enumerate(codes) if c == 1]
    assert len(starts) == steps
    t = ev[:, 0]
    assert t[-1] > t[0]
    ctx.check(lib.b2k_debug_trace(ctx.h, 0))
    lz.expand_many_(it, f, 2, 0.0)
    ctx.check(lib.b2k_debug_trace_read(ctx.h, buf, 4096, C.byref(n)))
    assert n.value == 0
    ctx.close()
