"""svdsolve on sparse matrices (B200CSR, scipy sparse host matrices) on the numpy stand-in of the C-ABI
(tests/hostsim_gkl.py): the driver's batching of expansions through gkl.expand_many_ / b2k_gkl_expand_many against the
oracle's step-by-step svdsolve on the same (A, u0), the entry forms, the refusals and the column bookkeeping."""
from __future__ import annotations

import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import hostsim_gkl

ORTHS = {"cgs2": (kk.cgs2, ko.CGS2), "mgs2b": (kk.mgs2b, ko.MGS2), "mgs2": (kk.mgs2, ko.MGS2)}


def _matrix(m, n, seed, density=6):
    rng = np.random.default_rng(seed)
    nnz = density * max(m, n)
    A = sp.coo_matrix((rng.standard_normal(nnz), (rng.integers(0, m, nnz), rng.integers(0, n, nnz))), shape=(m, n))
    A = A.tocsr()
    A.sum_duplicates()
    return A


def _oracle(A, u0, howmany, which, orth_tag, krylovdim, tol, eager=False, maxiter=100):
    return ko.svdsolve_gkl(A, u0, howmany, which, krylovdim=krylovdim, maxiter=maxiter, tol=tol,
                           orth=ko.Orth(orth_tag), eager=eager)


@pytest.mark.parametrize("orth", sorted(ORTHS))
@pytest.mark.parametrize("which", ["LR", "SR"])
@pytest.mark.parametrize("shape", [(400, 150), (150, 400)])
def test_host_sparse_matches_oracle(orth, which, shape):
    A = _matrix(*shape, seed=3)
    u0 = ko.splitmix_vector(11, shape[0])
    alg_orth, otag = ORTHS[orth]
    kw = dict(krylovdim=24, tol=1e-10)
    with hostsim_gkl.installed() as lib:
        S, U, V, info = kk.svdsolve(A, u0, 3, which, kk.GKL(orth=alg_orth, maxiter=100, verbosity=0, **kw))
        calls = lib.gkl_calls
    So, _, _, oinfo = _oracle(A, u0, 3, which, otag, **kw)
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    assert info.passes == info.numops
    # 1e-10 relative, and relative to sigma_max for the (numerically) zero values SR finds on a tall A
    np.testing.assert_allclose(S[:3], So[:3], rtol=1e-10, atol=1e-10 * So.max())
    assert (calls > 0) == (orth != "mgs2")           # MGS2 steps through the literal recurrence
    for s, u, v, r in zip(S, U, V, info.residual):
        assert isinstance(u, np.ndarray) and isinstance(v, np.ndarray) and isinstance(r, np.ndarray)
        if which == "SR":
            continue        # a tall A's zero values belong to u0's part outside range(A): no triplet relation
        assert np.linalg.norm(A.T @ u - s * v) < 1e-8 * So.max()
        assert np.linalg.norm(A @ v - s * u - r) < 1e-8 * So.max()


@pytest.mark.parametrize("orth", ["cgs2", "mgs2b"])
def test_eager_steps_one_at_a_time(orth):
    A = _matrix(300, 120, seed=5)
    u0 = ko.splitmix_vector(12, 300)
    alg_orth, otag = ORTHS[orth]
    with hostsim_gkl.installed() as lib:
        S, _, _, info = kk.svdsolve(A, u0, 2, "LR", kk.GKL(orth=alg_orth, krylovdim=20, tol=1e-10, eager=True,
                                                           verbosity=0))
        assert lib.gkl_calls == lib.gkl_steps            # one step per call
    So, _, _, oinfo = _oracle(A, u0, 2, "LR", otag, 20, 1e-10, eager=True)
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"]
    np.testing.assert_allclose(S[:2], So[:2], rtol=1e-10)


def test_device_csr_rectangular_and_square():
    with hostsim_gkl.installed() as lib:
        m, n = 350, 140
        A = _matrix(m, n, seed=7)
        u0 = ko.splitmix_vector(13, m)
        ctx = kk.B200Context(m, 80)
        sv = ctx.add_space(n, 60, sharded=False)
        op = kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        used = (lib.b2k_debug_used_columns(ctx.h, 0), lib.b2k_debug_used_columns(ctx.h, sv))
        nops = len(lib.ops)
        S, U, V, info = kk.svdsolve(op, ctx.from_host(u0), 2, "LR", kk.GKL(krylovdim=20, tol=1e-10,
                                                                          orth=kk.cgs2, verbosity=0))
        So, _, _, oinfo = _oracle(A, u0, 2, "LR", ko.CGS2, 20, 1e-10)
        assert info.numops == oinfo["numops"] and info.numiter == oinfo["numiter"]
        np.testing.assert_allclose(S[:2], So[:2], rtol=1e-10)
        assert lib.gkl_calls > 0 and len(lib.ops) == nops          # A' was freed
        assert U[0].space == 0 and V[0].space == sv
        # no leaked slab columns: what is in use beyond the start is exactly what was returned
        nres = len(info.residual)
        assert lib.b2k_debug_used_columns(ctx.h, 0) == used[0] + len(U) + nres
        assert lib.b2k_debug_used_columns(ctx.h, sv) == used[1] + len(V)
        del U, V, info
        # square, no explicit spaces: both sides in the space of u0
        B = _matrix(200, 200, seed=8)
        x0 = ko.splitmix_vector(14, 200)
        ctx2 = kk.B200Context(200, 120)
        opb = kk.B200CSR.from_scipy(ctx2, B)
        S2, U2, V2, _ = kk.svdsolve(opb, ctx2.from_host(x0), 2, "LR", kk.GKL(krylovdim=20, tol=1e-10, orth=kk.cgs2,
                                                                             verbosity=0))
        So2, _, _, _ = _oracle(B, x0, 2, "LR", ko.CGS2, 20, 1e-10)
        np.testing.assert_allclose(S2[:2], So2[:2], rtol=1e-10)
        assert U2[0].space == V2[0].space == 0
        ctx2.close()
        ctx.close()


def test_host_sparse_random_start():
    A = _matrix(260, 90, seed=9)
    with hostsim_gkl.installed() as lib:
        S, U, V, info = kk.svdsolve(A, None, 2, "LR", kk.GKL(krylovdim=20, tol=1e-10, orth=kk.cgs2, verbosity=0))
        assert lib.gkl_calls > 0
    sref = np.linalg.svd(A.toarray(), compute_uv=False)
    np.testing.assert_allclose(S[:2], sref[:2], rtol=1e-8)
    assert U[0].shape == (260,) and V[0].shape == (90,)


def test_rank_deficient_stops_mid_batch_like_stepping():
    """A of rank 3: beta falls below tol inside a chained batch (at K = 3 of 20).  The chained run gives the warnings,
    the counts and the values of the literal tuple path, which steps one expansion at a time."""
    rng = np.random.default_rng(21)
    m, n = 240, 100
    L3 = sp.csr_matrix(rng.standard_normal((m, 3)))
    R3 = sp.csr_matrix(rng.standard_normal((3, n)))
    A = (L3 @ R3).tocsr()
    u0 = ko.splitmix_vector(15, m)
    alg = kk.GKL(krylovdim=20, tol=1e-8, orth=kk.cgs2, verbosity=1)
    runs = []
    with hostsim_gkl.installed() as lib:
        ctx = kk.B200Context(m, 100)
        sv = ctx.add_space(n, 60, sharded=False)
        op = kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        opt = kk.B200CSR.from_scipy(ctx, A.T.tocsr()).with_spaces(0, sv)
        for target in (op, (op, opt)):
            calls = lib.gkl_calls
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                S, _, _, info = kk.svdsolve(target, ctx.from_host(u0), 3, "LR", alg)
            msgs = sorted(str(x.message) for x in w)
            runs.append((S, info.numops, info.numiter, msgs, lib.gkl_calls - calls))
        ctx.close()
    (S1, ops1, it1, w1, c1), (S2, ops2, it2, w2, c2) = runs
    assert c1 == 1 and c2 == 0                     # one batch that stopped early / no chained call
    assert w1 == w2
    assert (ops1, it1) == (ops2, it2) and ops1 <= 2 * 5          # stopped long before krylovdim = 20
    np.testing.assert_allclose(S1, S2, rtol=1e-10)


def test_refusals():
    with hostsim_gkl.installed() as lib:
        ctx = kk.B200Context(64, 40)
        free = kk.B200CSR.stencil_free(ctx, 8, 8)
        with pytest.raises(kk.B200Error, match="matrix-free stencil has no transpose.*B200CSR"):
            kk.svdsolve(free, ctx.from_host(np.ones(64)), 1, "LR", kk.GKL(krylovdim=10))
        sv = ctx.add_space(20, 30, sharded=False)
        rect = kk.B200CSR.from_scipy(ctx, _matrix(64, 20, seed=1))
        with pytest.raises(ValueError, match="with_spaces"):
            kk.svdsolve(rect, ctx.from_host(np.ones(64)), 1, "LR", kk.GKL(krylovdim=10))
        ctx.nranks = 2                                  # what a row-sharded context reports
        with pytest.raises(kk.B200Error, match="row-sharded contexts are not supported.*scipy sparse"):
            kk.svdsolve(rect.with_spaces(sv, 0), ctx.from_host(np.ones(64)), 1, "LR", kk.GKL(krylovdim=10))
        ctx.nranks = 1
        # the C-ABI entry: a refused call writes nothing
        rect_t = rect.transpose()
        u = [ctx.from_host(np.ones(64)) for _ in range(2)]
        v = [ctx.from_host(np.ones(20), sv)]
        import ctypes as C
        for (A_, At_, alg, ucols, vcols, code) in (
                (rect, rect_t, L.MGS2, u, v, L.ENOTSUP),
                (rect, rect, L.CGS2, u, v, L.EDIM),                     # At is not A's shape transposed
                (rect, rect_t, L.CGS2, u, [u[0]], L.EDIM),              # V from the wrong space
                (free, free, L.CGS2, u, v, L.ENOTSUP)):
            uc = (L.c_vec * 8)(*[x.handle for x in ucols])
            vc = (L.c_vec * 8)(*[x.handle for x in vcols])
            before_u, before_v = list(uc), list(vc)
            al, be = (C.c_double * 4)(), (C.c_double * 4)()
            done, rout = C.c_int32(-7), L.c_vec(-7)
            used = lib.b2k_debug_used_columns(ctx.h, 0), lib.b2k_debug_used_columns(ctx.h, sv)
            st = ctx.lib.b2k_gkl_expand_many(ctx.h, A_.h, At_.h, uc, vc, 1, 4, 1.0, 0.0, alg, al, be,
                                             C.byref(done), C.byref(rout))
            assert st == code
            assert list(uc) == before_u and list(vc) == before_v and done.value == -7 and rout.value == -7
            assert (lib.b2k_debug_used_columns(ctx.h, 0), lib.b2k_debug_used_columns(ctx.h, sv)) == used
        assert lib.gkl_calls == 0
        ctx.close()


def test_tuple_path_is_unchanged():
    """A user's (A, At) pair keeps the literal sequence: it is not known to be an exact transpose."""
    A = _matrix(200, 80, seed=4)
    u0 = ko.splitmix_vector(16, 200)
    with hostsim_gkl.installed() as lib:
        ctx = kk.B200Context(200, 100)
        sv = ctx.add_space(80, 60, sharded=False)
        pair = (kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0), kk.B200CSR.from_scipy(ctx, A.T.tocsr())
                .with_spaces(0, sv))
        S, _, _, info = kk.svdsolve(pair, ctx.from_host(u0), 2, "LR", kk.GKL(krylovdim=16, tol=1e-10, orth=kk.cgs2,
                                                                            verbosity=0))
        assert lib.gkl_calls == 0
        with pytest.raises(kk.B200Error, match="pass \\(A, At\\)"):
            kk.operators.apply_adjoint(pair[0], ctx.from_host(u0))
        ctx.close()
    So, _, _, oinfo = _oracle(A, u0, 2, "LR", ko.CGS2, 16, 1e-10)
    assert info.numops == oinfo["numops"]
    np.testing.assert_allclose(S[:2], So[:2], rtol=1e-10)
