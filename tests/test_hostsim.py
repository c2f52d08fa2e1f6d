"""Host-side driver logic without a GPU: the bodies of the GPU parity tests, run against
tests/hostsim.py (a numpy stand-in for the C-ABI, test infrastructure only).  What this covers is
everything ABOVE the C-ABI — restart bookkeeping, Schur reordering, block bookkeeping, step-size
control, handle lifetimes and slab column budgets; the kernels themselves are covered by `-m gpu`."""
import numpy as np
import pytest

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import hostsim
import test_gpu_solvers as G


@pytest.fixture()
def sim():
    with hostsim.installed() as lib:
        yield lib
    assert not isinstance(L._lib, hostsim.HostSimLib)


def test_simulator_is_not_the_product(sim):
    """The stand-in lives under tests/ only and the package cannot reach it."""
    import os
    pkg = os.path.dirname(os.path.abspath(kk._lib.__file__))
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert "hostsim" not in src and "from oracle" not in src and "import oracle" not in src


def test_vector_interface_and_errors(sim):
    ctx = kk.B200Context(50, 6)
    x = ctx.from_host(np.arange(50.0))
    y = x.copy().scale_(2.0)
    assert y.inner(x) == pytest.approx(2 * np.sum(np.arange(50.0) ** 2))
    y = y.add_(x, -2.0)
    assert y.norm() == 0.0
    vs = [ctx.empty() for _ in range(4)]
    with pytest.raises(L.B200Error):                      # slab exhausted -> loud failure, no silent growth
        ctx.empty()
    del vs
    ctx.empty()
    ctx.close()


def test_bicgstab(sim):
    G.test_bicgstab_matches_oracle_and_reference_properties(False)


@pytest.mark.parametrize("orth", ["mgs", "cgs2", "mgsr"])
def test_lsmr(sim, orth):
    G.test_lsmr_matches_oracle_and_reference_properties(orth)


def test_blocklanczos(sim):
    G.test_blocklanczos_reference_properties()


@pytest.mark.parametrize("orth", ["cgs2", "mgs2", "cgsr", "mgsr"])
def test_arnoldi_eigsolve_and_schursolve(sim, orth):
    G.test_arnoldi_eigsolve_and_schursolve(orth)


@pytest.mark.parametrize("method", ["lanczos", "arnoldi"])
def test_exponentiate_and_expintegrator(sim, method):
    G.test_exponentiate_and_expintegrator(method)


def test_cg_literal_path(sim):
    G.test_cg_matches_oracle(False)


def test_lanczos_eigsolve_with_restarts(sim):
    """eigsolve(::Lanczos) host loop incl. the native restart helper, vs the oracle."""
    nx, ny = 40, 25
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(7, nx * ny)
    ctx = kk.B200Context(nx * ny, 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=20, maxiter=60, tol=1e-10, verbosity=0)
    D, V, info = kk.eigsolve(op, ctx.from_host(x0), 3, "SR", alg)
    oD, _, oinfo = ko.eigsolve_lanczos(A, x0, 3, "SR", krylovdim=20, maxiter=60, tol=1e-10, orth=ko.Orth(ko.CGS2))
    assert info.converged >= 3 and info.numiter > 1
    np.testing.assert_allclose(D[:3], oD[:3], rtol=1e-10)
    np.testing.assert_allclose(D[:3], ko.laplace_eigenvalues(nx, ny)[:3], rtol=1e-9)
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    for lam, v in zip(D[:3], V[:3]):
        vh = v.to_host()
        assert np.linalg.norm(A @ vh - lam * vh) < 1e-8
    ctx.close()


@pytest.mark.parametrize("pair", G.PAIRS, ids=G.IDS)
def test_lanczos_and_arnoldi_steps(sim, pair):
    G.test_lanczos_steps_match_oracle(pair, False)
    G.test_arnoldi_steps_match_oracle(pair)


@pytest.mark.parametrize("pair", [G.PAIRS[2], G.PAIRS[3], G.PAIRS[6]], ids=["cgs2", "mgs2", "mgs2b"])
@pytest.mark.parametrize("literal", [False, True])
def test_gmres(sim, pair, literal):
    G.test_gmres_matches_oracle(pair, literal)


@pytest.mark.parametrize("literal", [False, True])
def test_gmres_singular_branch(sim, literal):
    G.test_gmres_singular_in_krylov_subspace_branch(literal)


@pytest.mark.parametrize("pair", [G.PAIRS[2], G.PAIRS[3], G.PAIRS[4]], ids=["cgs2", "mgs2", "cgsr"])
def test_svdsolve(sim, pair):
    G.test_svdsolve_matches_oracle_f64(pair)


def test_misc_drivers(sim):
    G.test_eigsolve_unconverged_fixed_cycles_matches_oracle()
    G.test_block_primitives_gpu()
    G.test_invariant_subspace_early_exit()
    G.test_zero_start_vector_raises()


def test_blocklanczos_toric(sim):
    G.test_blocklanczos_toric_code_degenerate_ground_space()


def test_keyword_front_ends_select_like_the_reference(sim):
    """eigselector / linselector (eigsolve.jl:238-321, linsolve.jl:123-180) and the `which` checks
    (eigsolve.jl:210-222)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(3)
    n = 60
    S = ko.stencil_matrix(10, 6)
    Nn = (S + sp.diags([0.3], [1], shape=(n, n))).tocsr()
    assert isinstance(kk.eigselector(S), kk.Lanczos) and isinstance(kk.eigselector(Nn), kk.Arnoldi)
    assert isinstance(kk.eigselector(lambda x: x), kk.Arnoldi)            # a function: not assumed symmetric
    assert isinstance(kk.eigselector(lambda x: x, issymmetric=True), kk.Lanczos)
    assert kk.eigselector(S, block=True).krylovdim == 100
    with pytest.raises(ValueError):
        kk.eigselector(Nn, block=True)
    x0 = rng.random(n)
    vals, vecs, info = kk.eigsolve(S, x0, 2, "SR", krylovdim=30, tol=1e-10)
    np.testing.assert_allclose(vals[:2], ko.laplace_eigenvalues(10, 6)[:2], rtol=1e-9)
    vals, vecs, info = kk.eigsolve(Nn, x0, 2, "LR", krylovdim=n, tol=1e-10)    # -> Arnoldi, host buffers
    want = np.linalg.eigvals(Nn.toarray())
    want = want[np.argsort(-want.real, kind="stable")]
    np.testing.assert_allclose(np.sort(vals[:2].real), np.sort(want[:2].real), rtol=1e-8)
    for lam, v in zip(vals, vecs):
        assert np.linalg.norm(Nn @ v - lam * v) < 1e-7
    with pytest.raises(ValueError):
        kk.eigsolve(S, x0, 1, "LI", krylovdim=20)
    with pytest.raises(ValueError):
        kk.eigsolve(Nn, x0, 1, "SI", krylovdim=20)
    with pytest.raises(ValueError):
        kk.eigsolve(S, x0, 1, "XX", krylovdim=20)
    with pytest.raises(TypeError):
        kk.eigsolve(S, x0, 1, "SR", kk.Lanczos(), krylovdim=20)
    b = rng.random(n)
    alg = kk.linselector(S, b, isposdef=True, krylovdim=10, maxiter=7)
    assert isinstance(alg, kk.CG) and alg.maxiter == 70
    assert alg.tol == pytest.approx(max(1e-12, 1e-12 * np.linalg.norm(b)))
    assert isinstance(kk.linselector(S, b), kk.GMRES) and isinstance(kk.linselector(Nn, b, isposdef=True), kk.GMRES)
    x, info = kk.linsolve(S, b, isposdef=True, rtol=1e-10)
    assert info.converged == 1 and np.linalg.norm(S @ x - b) < 1e-9 * np.linalg.norm(b) * 10
    x, info = kk.linsolve(Nn, b, krylovdim=20, rtol=1e-10)
    assert info.converged == 1 and np.linalg.norm(Nn @ x - b) < 1e-8
    x, info = kk.linsolve(Nn, b, None, kk.BiCGStab(maxiter=500, tol=1e-10, verbosity=0))
    assert info.converged == 1 and np.linalg.norm(Nn @ x - b) < 1e-9


def test_realeigsolve(sim):
    G.test_realeigsolve()


@pytest.mark.parametrize("seed", [0, 40, 114, 149])        # 40 / 114 / 149: all 20 triplets converge at once
def test_matrix_only_front_ends_draw_a_random_start(sim, seed, monkeypatch):
    """eigsolve(A, howmany, which; …) / svdsolve(A, howmany, which; …) — eigsolve.jl:195-201, svdsolve.jl:123-129."""
    rng0 = np.random.default_rng
    monkeypatch.setattr(np.random, "default_rng", lambda *a: rng0(seed))      # deterministic "random" start
    S = ko.stencil_matrix(12, 9)
    vals, vecs, info = kk.eigsolve(S, None, 2, "SR", krylovdim=40, tol=1e-9)
    np.testing.assert_allclose(vals[:2], ko.laplace_eigenvalues(12, 9)[:2], rtol=1e-8)
    D = rng0(2).standard_normal((50, 20))
    sv, U, V, info = kk.svdsolve(D, None, 2, "LR", krylovdim=20, tol=1e-10)
    assert len(U) == len(V) == max(2, info.converged)
    np.testing.assert_allclose(sv[:2], np.linalg.svd(D, compute_uv=False)[:2], rtol=1e-8)
    with pytest.raises(TypeError):
        kk.eigsolve(lambda x: x, None, 1, "SR")


def test_eigsorter_selects_interior_targets(sim):
    """EigSorter(by; rev) — eigsolve.jl:181-192: e.g. the eigenvalues closest to a shift (full-space run)."""
    n = 24
    rng = np.random.default_rng(8)
    d = np.sort(rng.standard_normal(n))
    A = sp_diags(d)
    ctx = kk.B200Context(n, 240)           # every converged pair comes back with its residual vector
    op = kk.B200CSR.from_scipy(ctx, A)
    target = 0.1
    sorter = kk.EigSorter(lambda lam: np.abs(lam - target))
    vals, vecs, info = kk.eigsolve(op, ctx.from_host(rng.random(n)), 3, sorter,
                                   kk.Lanczos(krylovdim=n, maxiter=1, tol=1e-10, verbosity=0))
    want = d[np.argsort(np.abs(d - target))][:3]
    np.testing.assert_allclose(vals[:3], want, rtol=1e-8, atol=1e-10)
    vals, _, _ = kk.eigsolve(op, ctx.from_host(rng.random(n)), 2, kk.EigSorter(lambda lam: np.real(lam), rev=True),
                             kk.Arnoldi(krylovdim=n, maxiter=1, tol=1e-10, verbosity=0))
    np.testing.assert_allclose(np.real(vals[:2]), d[::-1][:2], rtol=1e-8)
    with pytest.raises(ValueError):
        kk.eigsolve(op, ctx.from_host(rng.random(n)), 1, kk.EigSorter(lambda lam: np.imag(lam)),
                    kk.Arnoldi(krylovdim=n, maxiter=1, verbosity=0))
    ctx.close()


def sp_diags(d):
    import scipy.sparse as sp
    return sp.diags(d).tocsr()


@pytest.fixture()
def simf():
    """The simulator with the product's fused entry points left ON."""
    with hostsim.installed(fused=True) as lib:
        yield lib


def test_fused_branches_bookkeeping(simf):
    """Host-side bookkeeping of the fused branches — handle accounting of expand_/expand_many_ (library-
    allocated residual columns adopted by Python), the one-call CG step, the two-call BiCGStab flow with
    its half-step exit — against the oracle, exactly as the GPU tests run them."""
    for pair in (G.PAIRS[2], G.PAIRS[3], G.PAIRS[4], G.PAIRS[0], G.PAIRS[6]):
        G.test_lanczos_steps_match_oracle(pair, True)
    G.test_cg_matches_oracle(True)
    G.test_bicgstab_matches_oracle_and_reference_properties(True)
    G.test_eigsolve_unconverged_fixed_cycles_matches_oracle()
    G.test_invariant_subspace_early_exit()


def test_matrix_free_stencil(simf):
    import test_gpu_primitives as P
    P.test_matrix_free_stencil_equals_assembled_operator((23, 17, 13), (6.0, -1.0, -1.1, -0.9, -1.0, -1.2, -0.8))


def test_cg_chain_bookkeeping(simf):
    G.test_cg_chained_iterations_equal_stepwise()


def test_bicgstab_chain_bookkeeping(simf):
    G.test_bicgstab_chained_iterations_equal_stepwise()


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_cg_and_bicgstab_chains_refuse_aliased_vectors(simf, dt):
    import test_gpu_blas1 as B
    B.test_cg_and_bicgstab_chains_refuse_aliased_vectors(dt)


def test_basistransform_refusals(sim):
    """b2k_basis_transform's refusals (bad sizes, m > 256, two spaces, a repeated handle) leave every column as it
    was, on the simulator as on the device"""
    import test_gpu_transform as T
    T.test_refusals_leave_every_column_untouched(check_kernel=False)


def test_block_fast_mode(sim):
    """the flagged block mode's host logic (BCGS2 coefficients -> M, Gram -> CholeskyQR2, rank fallback)"""
    import test_gpu_primitives as P
    P.test_block_multi_rhs_kernels()
    G.test_blocklanczos_fast_block_mode_matches_reference_mode()


def test_chained_batch_bookkeeping(simf):
    """handle accounting of the device-chained b2k_lanczos_expand_many contract (new column per basis vector,
    the old residual's column recycled, breakdown in the middle of a batch) without a GPU"""
    G.test_chained_lanczos_batch_is_bit_identical_to_stepping()
    G.test_chained_lanczos_batch_stops_at_breakdown_on_the_device()


def test_fused_eigsolve_with_restarts(simf):
    nx, ny = 40, 25
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(7, nx * ny)
    ctx = kk.B200Context(nx * ny, 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    for orth, oorth in ((kk.cgs2, ko.Orth(ko.CGS2)), (kk.mgs2, ko.Orth(ko.MGS2))):
        alg = kk.Lanczos(orth=orth, krylovdim=20, maxiter=60, tol=1e-10, verbosity=0)
        live0 = len(ctx.lib.ctxs[ctx.h.value].spaces[0].cols)
        D, V, info = kk.eigsolve(op, ctx.from_host(x0), 3, "SR", alg)
        oD, _, oinfo = ko.eigsolve_lanczos(A, x0, 3, "SR", krylovdim=20, maxiter=60, tol=1e-10, orth=oorth)
        assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"] and info.numiter > 1
        np.testing.assert_allclose(D[:3], oD[:3], rtol=1e-10)
        n_out = len(V) + len(info.residual)
        del V, info
        # every column the library allocated inside expand_many was adopted and released again
        assert len(ctx.lib.ctxs[ctx.h.value].spaces[0].cols) == live0, "leaked slab columns"
    ctx.close()


# ---- the flagged one-pass GKL mode (tests/test_gpu_zzz_onepass.py bodies on the simulator) ----------------------
import test_gpu_zzz_onepass as OP  # noqa: E402


@pytest.mark.parametrize("m,n,dtype", [(2000, 64, np.float32), (500, 70, np.float64)])
def test_onepass_apply(sim, m, n, dtype):
    OP.test_apply_normal_gram(m, n, dtype)


def test_onepass_variant_switch(sim):
    lib = kk._lib.load()
    assert lib.b2k_debug_set_onepass_variant(1) == 0 and lib.b2k_debug_set_onepass_variant(0) == 0
    assert lib.b2k_debug_set_onepass_variant(2) != 0


def test_onepass_apply_errors(sim):
    OP.test_apply_normal_gram_errors()


@pytest.mark.parametrize("which", [0, 1, 2], ids=["mgs2", "cgs2", "cgsr"])
def test_onepass_svdsolve_f64(sim, which):
    orth, oorth = [(kk.mgs2, ko.Orth(ko.MGS2)), (kk.cgs2, ko.Orth(ko.CGS2)),
                   (kk.ClassicalGramSchmidtIR(eta=0.75), ko.Orth(ko.CGSIR, 0.75))][which]
    OP.test_svdsolve_onepass_f64(orth, oorth)


def test_onepass_svdsolve_f32(sim):
    OP.test_svdsolve_onepass_config4_small_f32()


def test_config4_fullsize_test_body_on_the_simulator(sim, monkeypatch):
    """tests/test_gpu_fullsize.py::test_svdsolve_config4_full_size_vs_float64_truth with the truth of a 6000-row matrix of
    the same generator: the body (column budgets, residual identities on the device vectors, pass count) runs here too."""
    import test_gpu_fullsize as F
    m, n = 6000, 512
    A = ko.dense_splitmix(F.SEED, m, n)
    truth = np.linalg.svd(A.astype(np.float64), compute_uv=False)[:6]
    monkeypatch.setitem(F.GOLD, "c4_truth", {"shape": [m, n], "seed": F.SEED, "sigma_float64_truth": [float(x) for x in truth]})
    for orth_name in ("mgs2", "cgsr"):
        F.test_svdsolve_config4_full_size_vs_float64_truth(orth_name)
