"""GPU tests of b2k_minres_chain (k_minres_step of blas1.cu and the SpMV in front of it) against an exact host
restatement, in Float64 and Float32.

Contract.  One iteration k, from the unnormalised Lanczos vectors p_cur = p_{k-1}, p_prev = p_{k-2} and the state
{β_k, 1/β_k, 1/β_{k-1}, c, s, δ̄, ε, φ̄}:
  v_k = rn(p_cur·T(1/β_k)), v_{k-1} = rn(p_prev·T(1/β_{k-1}))                      [scale!!]
  q = (a0 + a1 A) v_k: the bits of a separate shifted apply to a stored v_k;  α = <v_k, q>
  p_k = fma(T(-β_k), v_{k-1}, fma(T(-α), v_k, q)), over p_prev;  β_{k+1} = sqrt(Σ p_k²)  [two add!!, norm]
  the scalar recurrence in plain Float64 arithmetic (tests/minres_oracle.py::givens_step) — bit for bit
  d = rn(fma(T(-ε), d2, fma(T(-δ), d1, v_k))·T(1/γ)), over d2;  x = fma(T(φ), d, x)   [two add!!, scale!!, add!!]
Elementwise results are compared with array_equal; α and β_{k+1} are per-CTA sums whose order is not pinned, so they
are held to 16·u·Σ|terms| (u the unit roundoff of T; a thread accumulates a handful of terms in T at these sizes, the
rest of the sum is formed in double) and the vectors are then restated from the α the device reported.
The direction / solution update is applied one launch late (by the next iteration's kernel, or by the flush launch
that ends a call): nsteps = k against k calls of nsteps = 1 compares the two placements bit for bit.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

import minres_oracle as mo

f64, f32 = np.float64, np.float32
VEC = {f64: 2, f32: 4}
U = {f64: 2.0 ** -53, f32: 2.0 ** -24}
NAMES = ("x", "p_prev", "p_cur", "q", "d1", "d2")


def random_coupling(n, per_row, seed):
    """n x n sparse matrix with about per_row random entries per row (index pairs drawn directly: scipy.sparse.random
    permutes all n² positions)"""
    rng = np.random.default_rng(seed)
    k = int(per_row * n)
    return sp.coo_matrix((rng.uniform(0.0, 1.0, k), (rng.integers(0, n, k), rng.integers(0, n, k))), shape=(n, n)).tocsr()


def make_op(ctx, kind, n, dt, seed=3):
    """(device operator, the same matrix on the host)"""
    if kind in ("stencil", "stencil_free"):
        A = ko.stencil_matrix(n, 1, dtype=dt)
        return (kk.B200CSR.stencil if kind == "stencil" else kk.B200CSR.stencil_free)(ctx, n, 1), A
    R = random_coupling(n, 3, seed)
    A = (R + R.T + sp.diags(np.where(np.arange(n) % 2 == 0, 1.5, -1.5))).tocsr().astype(dt)
    A.sort_indices()
    return kk.B200CSR.from_scipy(ctx, A), A


def make_vecs(ctx, n, dt, seed):
    rng = np.random.default_rng(seed)
    host = {k: rng.standard_normal(n).astype(dt) for k in NAMES}
    return {k: ctx.from_host(v) for k, v in host.items()}, host


def state0(seed):
    rng = np.random.default_rng(seed)
    beta, bprev, th = rng.uniform(0.5, 2.0), rng.uniform(0.5, 2.0), rng.uniform(0, 2 * np.pi)
    return [beta, 1.0 / beta, 1.0 / bprev, np.cos(th), np.sin(th), rng.standard_normal(), rng.standard_normal(),
            rng.uniform(0.5, 2.0)]


def chain(ctx, op, v, st, a0, a1, tol, nsteps, names=NAMES):
    rec, done = np.zeros((nsteps, 8)), C.c_int32(-1)
    sin, sout = (C.c_double * 8)(*st), (C.c_double * 8)()
    status = ctx.lib.b2k_minres_chain(ctx.h, op.h, *[v[k].handle for k in names], a0, a1, sin, tol, nsteps,
                                      rec.ctypes.data_as(C.POINTER(C.c_double)), sout, C.byref(done))
    return status, rec[:max(done.value, 0)], list(sout), done.value


def rotated(v, done):
    """the handles by role after `done` iterations"""
    if done & 1:
        return dict(v, p_prev=v["p_cur"], p_cur=v["p_prev"], d1=v["d2"], d2=v["d1"])
    return v


def download(v):
    return {k: v[k].to_host() for k in NAMES}


def sizes(dt):
    return [1, 7, 64 * VEC[dt] - 1, 64 * VEC[dt] + 1, 100003]


@pytest.mark.parametrize("shift", [(0.0, 1.0), (-0.37, 1.25)])
@pytest.mark.parametrize("kind", ["stencil", "stencil_free", "csr"])
@pytest.mark.parametrize("dt", [f64, f32])
def test_one_iteration_against_the_restatement(fma, dt, kind, shift):
    a0, a1 = shift
    for n in sizes(dt):
        ctx = kk.B200Context(n, 12, dtype=dt)
        op, A = make_op(ctx, kind, n, dt)
        v, h = make_vecs(ctx, n, dt, n)
        st = state0(n + 1)
        status, rec, st_out, done = chain(ctx, op, v, st, a0, a1, 0.0, 1)
        assert status == L.OK and done == 1
        got = download(v)
        vk, vp = h["p_cur"] * dt(st[1]), h["p_prev"] * dt(st[2])
        q = kk.apply(op, ctx.from_host(vk), a0, a1).to_host()
        assert np.array_equal(got["q"], q), (n, "q")
        assert np.array_equal(got["p_cur"], h["p_cur"]) and np.array_equal(got["d1"], h["d1"])
        alpha, beta_new = rec[0, 0], rec[0, 1]
        terms = np.abs(vk.astype(f64) * q.astype(f64))
        assert abs(alpha - np.dot(vk.astype(f64), q.astype(f64))) <= 16 * U[dt] * terms.sum() + 1e-300, (n, "alpha")
        p_new = fma(dt(-st[0]), vp, fma(dt(-alpha), vk, q, dt), dt)
        assert np.array_equal(got["p_prev"], p_new), (n, "p")
        ss = np.dot(p_new.astype(f64), p_new.astype(f64))
        assert abs(beta_new * beta_new - ss) <= 16 * U[dt] * ss, (n, "beta")
        ref = list(st)
        want = mo.givens_step(ref, alpha, beta_new)
        assert tuple(rec[0][:5]) == want[:5] and tuple(rec[0][6:]) == want[6:] and rec[0][5] == 0.0
        assert st_out == ref
        _, _, gamma, phi, _, _, delta, eps = want
        d_new = fma(dt(-eps), h["d2"], fma(dt(-delta), h["d1"], vk, dt), dt) * dt(1.0 / gamma)
        assert np.array_equal(got["d2"], d_new), (n, "d")
        assert np.array_equal(got["x"], fma(dt(phi), d_new, h["x"], dt)), (n, "x")
        ctx.close()


@pytest.mark.parametrize("compact", [0, 1])
@pytest.mark.parametrize("dt", [f64, f32])
def test_chained_iterations_equal_single_ones(dt, compact):
    """nsteps = 6 in one call == 6 calls of nsteps = 1 (vectors, records, state), twice over the same input; a tol
    between two recorded |φ̄| stops at that iteration and the launches behind it change nothing"""
    n, k = 20011, 6
    lib = L.load()
    lib.b2k_debug_set_csr_compact(compact)
    try:
        ctx = kk.B200Context(n, 36, dtype=dt)
        op, A = make_op(ctx, "csr", n, dt)
        rng = np.random.default_rng(5)
        r = rng.standard_normal(n).astype(dt)
        beta1 = float(np.linalg.norm(r.astype(f64)))

        def fresh():
            v = {key: ctx.zeros() for key in NAMES}
            v["p_cur"].upload(r)
            return v

        v1 = fresh()
        status, rec1, st1, done = chain(ctx, op, v1, mo.fresh_state(beta1), -0.2, 1.0, 0.0, k)
        assert status == L.OK and done == k and np.all(rec1[:, 5] == 0)
        assert np.all(np.diff(rec1[:, 4]) <= 0) and rec1[0, 4] <= beta1
        one = download(rotated(v1, k))
        v1b = fresh()
        _, rec1b, st1b, _ = chain(ctx, op, v1b, mo.fresh_state(beta1), -0.2, 1.0, 0.0, k)
        two = download(rotated(v1b, k))
        assert np.array_equal(rec1, rec1b) and st1 == st1b and all(np.array_equal(one[key], two[key]) for key in NAMES)

        v2, st, recs = fresh(), mo.fresh_state(beta1), []
        for _ in range(k):
            status, rec, st, done = chain(ctx, op, v2, st, -0.2, 1.0, 0.0, 1)
            assert status == L.OK and done == 1
            v2 = rotated(v2, 1)
            recs.append(rec[0])
        assert np.array_equal(np.array(recs), rec1) and st == st1
        single = download(v2)
        for key in NAMES:
            assert np.array_equal(one[key], single[key]), key

        # the iterate is the literal one: x_k = Σ φ_j d_j with the d recurrence restated in float64 to rounding
        tol = 0.5 * (rec1[3, 4] + rec1[4, 4])
        v3 = fresh()
        status, rec3, st3, done3 = chain(ctx, op, v3, mo.fresh_state(beta1), -0.2, 1.0, tol, k + 3)
        assert status == L.OK and done3 == 5 and rec3[-1, 5] == 1.0 and np.array_equal(rec3[:, :5], rec1[:5, :5])
        v4 = fresh()
        _, _, st4, _ = chain(ctx, op, v4, mo.fresh_state(beta1), -0.2, 1.0, 0.0, 5)
        stopped, plain = download(rotated(v3, 5)), download(rotated(v4, 5))
        assert st3 == st4 and all(np.array_equal(stopped[key], plain[key]) for key in NAMES)
        o = mo.minres(A.astype(f64), r.astype(f64), a0=-0.2, tol=0.0, maxiter=5)
        assert np.linalg.norm(plain["x"] - o.x) <= 256 * U[dt] * np.linalg.norm(o.x)
        ctx.close()
    finally:
        lib.b2k_debug_set_csr_compact(1)


def test_refusals_write_nothing():
    n = 300
    ctx = kk.B200Context(n, 12)
    op, _ = make_op(ctx, "csr", n, f64)
    dense = kk.B200Dense.from_host(ctx, np.eye(n), ctx.add_space(n, 2, sharded=False))
    v, h = make_vecs(ctx, n, f64, 1)
    long = ctx.zeros(ctx.add_space(n + 1, 2))
    st = state0(2)
    assert chain(ctx, op, v, st, 0.0, 1.0, 0.0, 0)[0] == L.EINVAL
    assert chain(ctx, dense, v, st, 0.0, 1.0, 0.0, 1)[0] == L.ENOTSUP
    assert chain(ctx, op, dict(v, d2=long), st, 0.0, 1.0, 0.0, 1)[0] == L.EDIM
    assert chain(ctx, op, dict(v, d2=v["p_prev"]), st, 0.0, 1.0, 0.0, 1)[0] == L.EINVAL
    assert chain(ctx, op, dict(v, q=v["x"]), st, 0.0, 1.0, 0.0, 1)[0] == L.EINVAL
    got = download(v)
    assert all(np.array_equal(got[key], h[key]) for key in NAMES)
    ctx.close()
