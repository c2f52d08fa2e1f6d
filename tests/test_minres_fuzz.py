"""Seeded random symmetric problems through linsolve(MINRES) on the numpy stand-in, literal and chained, against the
float64 restatement: counts and solution."""
import importlib

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk

import hostsim_minres
import minres_oracle as mo

ls = importlib.import_module("krylovkit_jl_b200.linsolve")


@pytest.mark.parametrize("seed", range(24))
def test_random_symmetric_problem(seed, monkeypatch):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(20, 200))
    R = sp.random(n, n, density=rng.uniform(0.02, 0.2), random_state=seed)
    sign = np.where(rng.random(n) < rng.uniform(0.0, 0.6), -1.0, 1.0)            # some seeds are positive definite
    A = (sp.diags(rng.uniform(0.5, 3.0, n) * sign) + rng.uniform(0.0, 0.1) * (R + R.T)).tocsr()
    A.sort_indices()
    b = rng.standard_normal(n)
    a0, a1 = ((0.0, 1.0), (rng.uniform(-0.2, 0.2), rng.uniform(0.5, 2.0) * rng.choice([-1.0, 1.0])))[seed % 2]
    x0 = rng.standard_normal(n) if seed % 3 == 0 else None
    tol = 10.0 ** rng.uniform(-11, -6) * np.linalg.norm(b)
    maxiter = (400, 9)[seed % 8 == 7]
    o = mo.minres(A, b, x0, a0, a1, tol=tol, maxiter=maxiter)
    monkeypatch.setattr(ls, "MINRES_CHAIN_LEN", int(rng.integers(1, 40)))
    for chain in (False, True):
        monkeypatch.setattr(ls, "USE_MINRES_CHAIN", chain)
        with hostsim_minres.installed() as sim:
            ctx = kk.B200Context(n, 12)
            op = kk.B200CSR.from_scipy(ctx, A)
            used = sim.b2k_debug_used_columns(ctx.h, 0)
            xv = ctx.from_host(x0) if x0 is not None else None
            x, info = kk.linsolve(op, ctx.from_host(b), xv, kk.MINRES(maxiter=maxiter, tol=tol, verbosity=0), a0, a1)
            xh = x.to_host()
            del x, xv, info.residual
            assert sim.b2k_debug_used_columns(ctx.h, 0) == used
            ctx.close()
        assert (info.numiter, info.numops, info.converged) == (o.numiter, o.numops, o.converged)
        assert np.linalg.norm(xh - o.x) <= 1e-12 * np.linalg.norm(o.x)
        assert info.normres == pytest.approx(o.normres, rel=1e-6, abs=1e-300)
