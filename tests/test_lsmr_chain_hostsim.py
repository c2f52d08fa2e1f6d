"""lssolve on a B200CSR through the numpy stand-in of b2k_lsmr_chain (tests/hostsim_lsmr.py): the driver's batching,
its hand-over to the literal loop after a beta or alpha breakdown, its fall-back when the library refuses the chain, the orthogonalizers that do not chain, atol / rtol, the refusals
and the column bookkeeping, against the oracle's LSMR on the same (A, b)."""
from __future__ import annotations

import importlib

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import hostsim_lsmr

lsq = importlib.import_module("krylovkit_jl_b200.lssolve")


def _matrix(m, n, seed):
    A = sp.random(m, n, density=0.05, random_state=seed).tocsr() + sp.eye(m, n).tocsr()
    A.sort_indices()
    return A


def _solve(A, b, alg, lam=0.0, **kw):
    m, n = A.shape
    ctx = kk.B200Context(m, 16)
    try:
        sv = ctx.add_space(n, max(alg.krylovdim, 1) + 12, sharded=False)
        Ad = kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        used = (ctx.lib.b2k_debug_used_columns(ctx.h, 0), ctx.lib.b2k_debug_used_columns(ctx.h, sv))
        bd = ctx.from_host(b)
        x, info = kk.lssolve(Ad, bd, alg, lam, **kw)
        info.residual = info.residual.to_host()
        out = x.to_host(), info.residual, info
        del x, bd
        import gc
        gc.collect()
        # no slab column outlives the call: every work vector of the chain went back
        assert (ctx.lib.b2k_debug_used_columns(ctx.h, 0), ctx.lib.b2k_debug_used_columns(ctx.h, sv)) == used
        return out
    finally:
        ctx.close()


@pytest.mark.parametrize("orth,K", [("mgs", 1), ("mgs", 3), ("mgs2", 3), ("cgs2", 4), ("mgs2b", 3)])
@pytest.mark.parametrize("lam", [0.0, 0.4])
@pytest.mark.parametrize("chain_len,maxiter", [(5, 17), (1, 4), (17, 17), (32, 17)])
def test_chained_driver_matches_oracle(orth, K, lam, chain_len, maxiter, monkeypatch):
    """ring rotation over more iterations than krylovdim, batch lengths that divide maxiter, do not, and exceed it"""
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", chain_len)
    A = _matrix(120, 40, 3)
    b = np.random.default_rng(4).random(120)
    o = getattr(kk, orth)
    oo = ko.Orth(ko.MGS2 if orth == "mgs2b" else o.tag)
    with hostsim_lsmr.installed() as lib:
        x, res, info = _solve(A, b, kk.LSMR(orth=o, maxiter=maxiter, tol=0.0, krylovdim=K, verbosity=0), lam)
        assert lib.lsmr_calls == -(-maxiter // chain_len) and lib.lsmr_iters == maxiter
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=maxiter, tol=0.0, krylovdim=K, orth=oo, lam=lam)
    assert (info.numiter, info.numops, info.converged) == (oinfo["numiter"], oinfo["numops"], 0)
    np.testing.assert_allclose(x, ox, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-6)
    np.testing.assert_allclose(res, b - A @ x, atol=1e-10)


def test_convergence_in_a_batch_and_atol_rtol(monkeypatch):
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", 8)
    A = _matrix(150, 50, 5)
    b = np.random.default_rng(6).random(150)
    tol = 1e-9 * np.linalg.norm(A.T @ b)
    with hostsim_lsmr.installed() as lib:
        x, res, info = _solve(A, b, kk.LSMR(maxiter=200, krylovdim=5, verbosity=0), rtol=1e-9)
        assert lib.lsmr_calls >= 1
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=200, tol=tol, krylovdim=5)
    assert info.converged == 1 and abs(info.numiter - oinfo["numiter"]) <= 1
    assert np.linalg.norm(A.T @ (b - A @ x)) <= 10 * tol


@pytest.mark.parametrize("K", [1, 4])
def test_exhausted_krylov_space_stops_in_the_chain(K, monkeypatch):
    """three distinct singular values and b in the range: beta falls below tol at the third iteration, whose A'
    product is skipped (numops), and |zetabar| <= tol stops the chain there with the oracle's counts"""
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", 32)
    rng = np.random.default_rng(7)
    m, n = 60, 30
    U, _ = np.linalg.qr(rng.standard_normal((m, n)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = sp.csr_matrix(U @ np.diag(np.repeat([3.0, 2.0, 1.0], n // 3)) @ V.T)
    b = A @ rng.standard_normal(n)
    with hostsim_lsmr.installed() as lib:
        x, res, info = _solve(A, b, kk.LSMR(maxiter=8, tol=1e-8, krylovdim=K, verbosity=0))
        assert lib.lsmr_calls == 1 and lib.lsmr_iters == 3
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=8, tol=1e-8, krylovdim=K)
    assert (info.numiter, info.numops, info.converged) == (oinfo["numiter"], oinfo["numops"], oinfo["converged"])
    np.testing.assert_allclose(x, ox, rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("orth", ["cgsr", "mgsr", "cgs"])
def test_orthogonalizers_that_do_not_chain_take_the_literal_loop(orth):
    A = _matrix(80, 30, 8)
    b = np.random.default_rng(9).random(80)
    o = getattr(kk, orth)
    with hostsim_lsmr.installed() as lib:
        x, res, info = _solve(A, b, kk.LSMR(orth=o, maxiter=10, tol=0.0, krylovdim=4, verbosity=0))
        assert lib.lsmr_calls == 0
        x1, _, info1 = _solve(A, b, kk.LSMR(orth=o, maxiter=10, tol=0.0, krylovdim=1, verbosity=0))
        assert lib.lsmr_calls == 1                    # krylovdim <= 1: nothing to reorthogonalise, any orth chains
    oo = ko.Orth(o.tag, o.eta) if o.is_ir else ko.Orth(o.tag)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=10, tol=0.0, krylovdim=4, orth=oo)
    np.testing.assert_allclose(x, ox, rtol=1e-10, atol=1e-12)
    assert info.numops == oinfo["numops"]


def test_use_lsmr_chain_off_takes_the_literal_loop(monkeypatch):
    monkeypatch.setattr(lsq, "USE_LSMR_CHAIN", False)
    A = _matrix(80, 30, 10)
    b = np.random.default_rng(11).random(80)
    with hostsim_lsmr.installed() as lib:
        x, _, info = _solve(A, b, kk.LSMR(maxiter=6, tol=0.0, krylovdim=3, verbosity=0))
        assert lib.lsmr_calls == 0
    ox, _ = ko.lssolve_lsmr(A.toarray(), b, maxiter=6, tol=0.0, krylovdim=3)
    np.testing.assert_allclose(x, ox, rtol=1e-10, atol=1e-12)


def test_front_end_refusals():
    with hostsim_lsmr.installed():
        ctx = kk.B200Context(64, 8)
        try:
            b = ctx.from_host(np.ones(64))
            with pytest.raises(L.B200Error, match="matrix-free"):
                kk.lssolve(kk.B200CSR.stencil_free(ctx, 8, 8), b, kk.LSMR(verbosity=0))
            ctx.add_space(16, 8, sharded=False)
            A = kk.B200CSR.from_scipy(ctx, sp.random(64, 16, density=0.2, random_state=1).tocsr())
            with pytest.raises(ValueError, match="carry its spaces"):
                kk.lssolve(A, b, kk.LSMR(verbosity=0))
        finally:
            ctx.close()


def _breakdown_problem(kind, seed=7):
    rng = np.random.default_rng(seed)
    m, n = 400, 120
    U, _ = np.linalg.qr(rng.standard_normal((m, n)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = sp.csr_matrix(U @ np.diag(np.repeat([3.0, 2.0, 1.0], n // 3)) @ V.T)
    b = A @ rng.standard_normal(n)
    if kind == "alpha":
        w = rng.standard_normal(m)
        b = b + (w - U @ (U.T @ w))
    return A, 1e6 * b


@pytest.mark.parametrize("kind,code", [("beta", 2.0), ("alpha", 3.0)])
@pytest.mark.parametrize("orth,K", [("mgs", 1), ("mgs", 4), ("cgs2", 4)])
def test_breakdown_hands_over_to_the_literal_loop(kind, code, orth, K, monkeypatch):
    """b large, so |zetabar| is still above tol when beta (b in the range of A) or alpha (b with a part outside it)
    falls below tol: the chain stops with code 2 / 3 and the literal loop continues from the documented roles"""
    monkeypatch.setattr(lsq, "LSMR_CHAIN_LEN", 32)
    A, b = _breakdown_problem(kind)
    o = getattr(kk, orth)
    with hostsim_lsmr.installed() as lib:
        x, res, info = _solve(A, b, kk.LSMR(orth=o, maxiter=30, tol=1e-8, krylovdim=K, verbosity=0))
        assert lib.lsmr_calls == 1 and lib.lsmr_codes == [code]
        assert info.numiter > lib.lsmr_iters                  # the literal loop ran after the hand-over
    # after an alpha breakdown the reference's later iterates amplify rounding (v is left unnormalised): the
    # literal loop on the same arithmetic is the yardstick; the oracle agrees on the counts
    monkeypatch.setattr(lsq, "USE_LSMR_CHAIN", False)
    with hostsim_lsmr.installed() as lib:
        xl, _, infol = _solve(A, b, kk.LSMR(orth=o, maxiter=30, tol=1e-8, krylovdim=K, verbosity=0))
        assert lib.lsmr_calls == 0
    assert (info.numiter, info.numops, info.converged) == (infol.numiter, infol.numops, infol.converged)
    assert np.linalg.norm(x - xl) <= 1e-12 * np.linalg.norm(xl)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=30, tol=1e-8, krylovdim=K, orth=ko.Orth(o.tag))
    assert info.converged == 1 and oinfo["converged"] == 1
    assert (info.numiter, info.numops) == (oinfo["numiter"], oinfo["numops"])
    assert np.linalg.norm(x - ox) <= (1e-8 if code == 2.0 else 5e-2) * np.linalg.norm(ox)


def test_cgs2_ring_beyond_the_panel_falls_back(monkeypatch):
    """the library refuses a ring its cooperative sweep cannot hold (B2K_ENOTSUP, nothing written): literal loop"""
    A = _matrix(300, 120, 12)
    b = np.random.default_rng(13).random(300)
    with hostsim_lsmr.installed() as lib:
        x, _, info = _solve(A, b, kk.LSMR(orth=kk.cgs2, maxiter=5, tol=0.0, krylovdim=100, verbosity=0))
        assert lib.lsmr_calls == 0 and lib.lsmr_enotsup == 1
    ox, _ = ko.lssolve_lsmr(A.toarray(), b, maxiter=5, tol=0.0, krylovdim=100, orth=ko.Orth(ko.CGS2))
    np.testing.assert_allclose(x, ox, rtol=1e-10, atol=1e-12)


def test_non_csr_operator_is_refused():
    with hostsim_lsmr.installed():
        ctx = kk.B200Context(64, 8)
        try:
            sv = ctx.add_space(16, 8, sharded=False)
            D = kk.B200Dense.from_host(ctx, np.ones((64, 16)), sv)
            fake = object.__new__(kk.B200CSR)        # a dense operator handle dressed as a B200CSR
            fake.ctx, fake.h, fake.n_rows, fake.n_cols = ctx, D.h, 64, 16
            fake.space_in, fake.space_out, fake._explicit_spaces = sv, 0, True
            with pytest.raises(L.B200Error, match="not a stored CSR matrix"):
                kk.lssolve(fake, ctx.from_host(np.ones(64)), kk.LSMR(verbosity=0))
        finally:
            ctx.close()
