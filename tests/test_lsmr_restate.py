"""The one-iteration restatement of the chained LSMR step (tests/lsmr_restate.py), iterated on the host from the
reference loop's start, against the oracle's LSMR: its role rules (ring slots, the flush) and its rounding sequence
give the reference's iterates to rounding, with and without reorthogonalisation, with and without lambda."""
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
