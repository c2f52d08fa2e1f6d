"""The one-iteration restatement of the chained LSMR step (tests/lsmr_restate.py), iterated on the host from the
reference loop's start, against the oracle's LSMR: its role rules (ring slots, the flush) and its rounding sequence
give the reference's iterates to rounding, with and without reorthogonalisation, with and without lambda."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

import lsmr_restate as LR

f64, f32 = np.float64, np.float32


def start(A, b, K, lam, dt):
    """lssolve.py::_lsmr's set-up, in T"""
    b = b.astype(dt)
    beta = float(np.linalg.norm(b.astype(f64)))
    u = (b * dt(1 / beta)).astype(dt)
    v = ((A.T @ b).astype(dt) * dt(1 / beta)).astype(dt)
    alpha = float(np.linalg.norm(v.astype(f64)))
    v = (v * dt(1 / alpha)).astype(dt)
    m, n = A.shape
    z = lambda k: np.zeros(k, dtype=dt)  # noqa: E731
    vec = {"x": z(n), "h": v.copy(), "hbar": z(n), "r": (u * dt(beta)).astype(dt), "Ah": z(m), "Ahbar": z(m),
           "u": u}
    ring = [v] + [z(n) for _ in range(max(K, 1) - 1)]
    st = [alpha, beta, alpha, 1.0, 1.0, 1.0, 0.0, 0.0, alpha * beta, lam]
    return vec, ring, st


@pytest.mark.parametrize("orth,K", [(L.MGS, 1), (L.MGS, 3), (L.MGS2, 3), (L.CGS2, 3)])
@pytest.mark.parametrize("lam", [0.0, 0.4])
def test_restatement_iterates_match_oracle(fma, orth, K, lam):
    rng = np.random.default_rng(2)
    A = (sp.random(300, 80, density=0.05, random_state=3) + sp.eye(300, 80)).tocsr()
    A.sort_indices()
    At = A.T.tocsr()
    At.sort_indices()
    b = rng.random(300)
    N = 12
    vec, ring, st = start(A, b, K, lam, f64)
    for k in range(1, N + 1):
        vec, ring, spare, a, bt, st, rec = LR.iteration(fma, f64, A, At, st, vec, ring, K, orth, 0.0, 132, k)
    ox, oinfo = ko.lssolve_lsmr(A.toarray(), b, maxiter=N, tol=0.0, krylovdim=K, orth=ko.Orth(orth), lam=lam)
    assert np.linalg.norm(vec["x"] - ox) <= 1e-9 * np.linalg.norm(ox)
    np.testing.assert_allclose(rec[6], oinfo["normres"], rtol=1e-6)


def _scalars_float(st, alpha, beta, bskip, tol):
    """lsmr_scalars as first written, in Python floats (which raise on a division by zero): the finite reference"""
    hyp = lambda a, b: math.sqrt(a * a + b * b)  # noqa: E731
    _, _, alphabar, rhoold, rhobarold, cbar0, sbar0, _, zetabar0, lam = st
    alphahat = hyp(alphabar, lam)
    rho = hyp(alphahat, beta)
    c, s = alphahat / rho, beta / rho
    theta = s * alpha
    alphabar = c * alpha
    thetabar = sbar0 * rho
    cbarrho = cbar0 * rho
    rhobar = hyp(cbarrho, theta)
    cbar, sbar = cbarrho / rhobar, theta / rhobar
    zeta = cbar * zetabar0
    zetabar = -sbar * zetabar0
    g = (-thetabar * rho) / (rhoold * rhobarold)
    cz = zeta / (rho * rhobar)
    askip = not bskip and not alpha > tol
    code = 1.0 if abs(zetabar) <= tol else 2.0 if bskip else 3.0 if askip else 0.0
    rec = [alpha, beta, rho, rhobar, theta, zeta, abs(zetabar), code, 0.0 if bskip else 1.0, alphabar, cbar, sbar, g,
           cz, 0.0, 0.0]
    return [alpha, beta, alphabar, rho, rhobar, cbar, sbar, theta, zetabar, lam], rec


# rho_old rho-bar_old underflows to 0: g = -theta-bar rho / 0 is infinite while alpha, beta and zeta-bar stay finite
CODE4_STATE = [1.3, 0.7, 0.9, 1e-200, 1e-200, 0.8, 0.6, 0.35, 0.5, 0.3]


def test_scalars_unchanged_on_finite_inputs():
    rng = np.random.default_rng(4)
    for i in range(2000):
        st = list(rng.uniform(-2.0, 2.0, 10))
        st[3], st[4] = abs(st[3]) + 0.1, abs(st[4]) + 0.1
        alpha, beta = rng.uniform(0.0, 3.0, 2)
        bskip, tol = bool(i % 5 == 0), float(rng.choice([0.0, 1e-8, 0.5]))
        want_st, want_rec = _scalars_float(st, float(alpha), float(beta), bskip, tol)
        got_st, got_rec = LR.lsmr_scalars(st, alpha, beta, bskip, tol)
        assert np.array(got_st, dtype=f64).tobytes() == np.array(want_st, dtype=f64).tobytes()
        assert np.array(got_rec, dtype=f64).tobytes() == np.array(want_rec, dtype=f64).tobytes()


def test_scalars_raise_code_4_on_a_non_finite_derived_scalar():
    st, rec = LR.lsmr_scalars(CODE4_STATE, 1.1, 0.9, False, 0.0)
    assert rec[7] == 4.0 and np.isinf(rec[12])
    assert all(np.isfinite(rec[i]) and rec[i] != 0.0 for i in (0, 1, 6))
    with pytest.raises(ZeroDivisionError):
        _scalars_float(CODE4_STATE, 1.1, 0.9, False, 0.0)


@pytest.mark.parametrize("nsm", [132, 114, 7])
@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("per_thread,unroll", [(4, 2), (8, 4)], ids=["pt4", "pt8"])
def test_edge_sizes_have_their_properties(per_thread, unroll, dt, nsm):
    """cap and trips as the GPU tests derive them from the SM count, for every streaming kernel's geometry"""
    for name in ("cap", "trips"):
        LR.check_edge(name, LR.edge_size(name, dt, per_thread, unroll, nsm), dt, per_thread, unroll, nsm)
    g, capped, trips, _, tail = LR.trip_profile(LR.edge_size("V+1", dt, per_thread, unroll, nsm), dt, per_thread,
                                                unroll, nsm)
    assert g == 1 and not capped and trips == 1 and tail == 1
