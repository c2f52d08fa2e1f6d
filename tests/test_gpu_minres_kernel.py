"""GPU tests of b2k_minres_chain (k_minres_step of blas1.cu and the SpMV in front of it) against an exact host
restatement, in Float64 and Float32.

Contract.  One iteration k, from the unnormalised Lanczos vectors p_cur = p_{k-1}, p_prev = p_{k-2} and the state
{β_k, 1/β_k, 1/β_{k-1}, c, s, δ̄, ε, φ̄}:
  v_k = rn(p_cur·T(1/β_k)), v_{k-1} = rn(p_prev·T(1/β_{k-1}))                      [scale!!]
  q = (a0 + a1 A) v_k: the bits of a separate shifted apply to a stored v_k;  α = <v_k, q>
  p_k = fma(T(-β_k), v_{k-1}, fma(T(-α), v_k, q)), over p_prev;  β_{k+1} = sqrt(Σ p_k²)  [two add!!, norm]
  the scalar recurrence in plain Float64 arithmetic (tests/minres_oracle.py::givens_step) — bit for bit
  d = rn(fma(T(-ε), d2, fma(T(-δ), d1, v_k))·T(1/γ)), over d2;  x = fma(T(φ), d, x)   [two add!!, scale!!, add!!]
Every result is compared bit for bit.  α is the SpMV epilogue's fused dot (spmv_restate.apply with xscale = 1/β_k,
dot_self and the shift, on the kernel, grid and tiles the device reports), β_{k+1} the square root of k_minres_step's
CTA-ordered sum on grid_for(n, 4) (lsmr_restate.blas1_sum); a Higham-style bound checks those restatements against
the exact sums.  The sizes take k_minres_step (two-slot trips, 4 elements a thread) through its edges: lengths 1, 2,
3, V ± 1, 255, 257, a grid exactly at its 4·SMs cap, and a capped grid with three trips per thread, a partly live
second slot in the last trip and a tail.
The direction / solution update is applied one launch late (by the next iteration's kernel, or by the flush launch
that ends a call): nsteps = k against k calls of nsteps = 1 compares the two placements bit for bit.  Stop codes 2
(γ = 0) and 3 (β_{k+1} = 0) are raised on the identity, where α and p_k are exact.
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

import lsmr_restate as LR
import minres_oracle as mo
import spmv_restate as R

f64, f32 = np.float64, np.float32
VEC = {f64: 2, f32: 4}
U = {f64: 2.0 ** -53, f32: 2.0 ** -24}
NAMES = ("x", "p_prev", "p_cur", "q", "d1", "d2")
KERNEL_NAMES = {1: "stream", 2: "pipe", 3: "compact", 4: "stencil"}     # b2k_debug_spmv_launch kernel ids
COEFFS = (4.0, -1.0, -1.0, -1.0, -1.0, -1.0, -1.0)                      # B200CSR.stencil's default


def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


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
    """(name, n): k_minres_step's edges (grid_for(n, 4), trips of 2 slots), plus the sizes first tested"""
    names = list(LR.SMALL) + [7, 64 * VEC[dt] - 1, 64 * VEC[dt] + 1, 100003, "cap", "trips"]
    out = []
    for name in names:
        n = LR.edge_size(name, dt, 4, 2, nsm())
        LR.check_edge(name, n, dt, 4, 2, nsm())
        out.append((name, n))
    return out


def launch():
    out = (C.c_int32 * 4)()
    assert L.load().b2k_debug_spmv_launch(out) == L.OK
    return tuple(out)


def device_tiles(op):
    lib, nblk = L.load(), C.c_int32()
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, None, C.byref(nblk)) == L.OK
    rb = np.empty(nblk.value + 1, dtype=np.int32)
    if nblk.value:
        assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, rb.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nblk)) == L.OK
    return rb.astype(np.int64)


def alpha_restated(fma, dt, kind, A, op, rec, p_cur, invb, a0, a1):
    """the SpMV epilogue's α = <v_k, (a0 + a1 A) v_k> as the launch `rec` (b2k_debug_spmv_launch) summed it"""
    kname = KERNEL_NAMES[rec[0]]
    n = len(p_cur)
    kw = dict(a0=a0, a1=a1, shifted=(a0 != 0.0 or a1 != 1.0), xscale=invb, dot_self=True)
    if kind == "stencil_free":
        assert kname == "stencil"
        return R.apply(fma, dt, "stencil", rec[2], p_cur, stencil=(n, 1, 1, COEFFS), **kw)[2]
    rowblk = device_tiles(op)
    assert np.array_equal(rowblk, R.tiles(A.indptr)) and rec[3] == len(rowblk) - 1
    return R.apply(fma, dt, kname, rec[2], p_cur, csr=(A.indptr, A.indices, A.data), rowblk=rowblk, **kw)[2]


@pytest.mark.parametrize("shift", [(0.0, 1.0), (-0.37, 1.25)], ids=["plain", "shifted"])
@pytest.mark.parametrize("kind", ["stencil", "stencil_free", "csr"])
@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("size", ["small", "cap", "trips"])
def test_one_iteration_against_the_restatement(fma, size, dt, kind, shift):
    a0, a1 = shift
    for name, n in sizes(dt):
        if (size == "small") == (name in ("cap", "trips")) or (size != "small" and name != size):
            continue
        ctx = kk.B200Context(n, 12, dtype=dt)
        op, A = make_op(ctx, kind, n, dt)
        v, h = make_vecs(ctx, n, dt, n)
        st = state0(n + 1)
        status, rec, st_out, done = chain(ctx, op, v, st, a0, a1, 0.0, 1)
        spmv = launch()                              # before any other apply replaces the record
        assert status == L.OK and done == 1
        got = download(v)
        vk, vp = h["p_cur"] * dt(st[1]), h["p_prev"] * dt(st[2])
        q = kk.apply(op, ctx.from_host(vk), a0, a1).to_host()
        assert np.array_equal(got["q"], q), (name, "q")
        assert np.array_equal(got["p_cur"], h["p_cur"]) and np.array_equal(got["d1"], h["d1"])
        alpha, beta_new = rec[0, 0], rec[0, 1]
        a_ref = alpha_restated(fma, dt, kind, A, op, spmv, h["p_cur"], st[1], a0, a1)
        assert f64(alpha).tobytes() == f64(a_ref).tobytes(), (name, "alpha", alpha, a_ref)
        terms = np.abs(vk.astype(f64) * q.astype(f64))
        assert abs(a_ref - np.dot(vk.astype(f64), q.astype(f64))) <= 16 * U[dt] * terms.sum() + 1e-300, (name, "α")
        p_new = fma(dt(-st[0]), vp, fma(dt(-alpha), vk, q, dt), dt)
        assert np.array_equal(got["p_prev"], p_new), (name, "p")
        b_ref = np.sqrt(LR.blas1_sum(fma, dt, p_new, p_new, LR.grid_for(n, 4, nsm())))
        assert f64(beta_new).tobytes() == f64(b_ref).tobytes(), (name, "beta", beta_new, b_ref)
        ss = np.dot(p_new.astype(f64), p_new.astype(f64))
        assert abs(b_ref * b_ref - ss) <= 16 * U[dt] * ss, (name, "β")
        ref = list(st)
        want = mo.givens_step(ref, alpha, beta_new)
        assert tuple(rec[0][:5]) == want[:5] and tuple(rec[0][6:]) == want[6:] and rec[0][5] == 0.0
        assert st_out == ref
        _, _, gamma, phi, _, _, delta, eps = want
        d_new = fma(dt(-eps), h["d2"], fma(dt(-delta), h["d1"], vk, dt), dt) * dt(1.0 / gamma)
        assert np.array_equal(got["d2"], d_new), (name, "d")
        assert np.array_equal(got["x"], fma(dt(phi), d_new, h["x"], dt)), (name, "x")
        ctx.close()


def bits(a):
    return np.asarray(a).tobytes()


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("a0,code", [(-1.0, 2), (0.0, 3)], ids=["code2-gamma0", "code3-beta0"])
def test_stop_codes(dt, a0, code):
    """The identity with v_k = e_1 and β_k = 1, tol = 0: a0 = -1 gives q = 0, α = 0, p_k = 0 and so γ = 0 (code 2, the
    pending update kept with zero weights); a0 = 0 gives q = v_k, α = 1, p_k = 0, so β_{k+1} = 0 with γ = 1 (code 3).
    nsteps = 4 stops after one iteration and leaves every vector as one call of nsteps = 1 does."""
    n = 1001
    ctx = kk.B200Context(n, 12, dtype=dt)
    A = sp.identity(n, format="csr", dtype=dt)
    op = kk.B200CSR.from_scipy(ctx, A)
    st = mo.fresh_state(1.0)
    outs = []
    for nsteps in (4, 1):
        v, h = make_vecs(ctx, n, dt, 7)
        e1 = np.zeros(n, dtype=dt)
        e1[0] = 1
        v["p_cur"].upload(e1)
        h["p_cur"] = e1
        status, rec, st_out, done = chain(ctx, op, v, st, a0, 1.0, 0.0, nsteps)
        assert status == L.OK and done == 1, (status, done)
        ref = list(st)
        want = mo.givens_step(ref, 1.0 + a0, 0.0)
        assert rec[0][0] == 1.0 + a0 and rec[0][1] == 0.0
        assert tuple(rec[0][:5]) == want[:5] and tuple(rec[0][6:]) == want[6:] and rec[0][5] == code
        assert st_out == ref
        got = download(rotated(v, 1))
        assert not np.any(got["p_cur"])                                # p_k = 0
        if code == 2:
            assert want[2] == 0.0 and not np.any(got["d1"])            # d = 0 after the flush
            assert bits(got["x"]) == bits(h["x"])                      # x unchanged
        else:
            _, _, gamma, phi, _, _, delta, eps = want
            assert gamma == 1.0 and phi == 1.0
            assert bits(got["d1"]) == bits(e1)                         # d = v_k exactly (δ = ε = 0)
            assert bits(got["x"]) == bits(fma_add(h["x"], e1))
        outs.append((rec, st_out, got))
    (r4, s4, g4), (r1, s1, g1) = outs
    assert bits(r4) == bits(r1) and s4 == s1
    for key in NAMES:
        assert bits(g4[key]) == bits(g1[key]), key
    ctx.close()


def fma_add(x, e):
    """x + 1·e, elementwise: fma(1, e, x) where e is 0 or 1 is exact rounding of x + e"""
    return (x + e).astype(x.dtype)


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
