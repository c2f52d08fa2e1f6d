"""GPU tests of the tall-skinny engine (csrc/tsk.cuh: k_phase, k_gs_fused, k_finalize, driven from csrc/basis.cu) against
the host restatement of its summation order in tsk_restate.py, bit for bit, in Float64 and Float32: project!! and
unproject!!, orthogonalize!! with every classical orthogonalizer (fused, per phase, unfused passes), the pipelined MGS
sweeps against their literal BLAS-1 sequence, one Lanczos step (fused, split sweeps, unfused; CGS2, CGSIR and the MGS
family) and the dense GEMV.

Every engine case checks three things: the outputs (h, the vector, ||v||, alpha, beta) have the restatement's bits; the
path that ran is the expected one (per-class launch counts of b2k_prof_read: fused sweeps, project and unproject
passes); and the cooperative launch and the launch per phase give the same bits.  A pinned single Lanczos step also
pins the device-chained batch, which test_gpu_lanczos_step_layout.py and test_gpu_solvers.py check against stepping.

Shapes.  n: 1, 2, 3, 255, 256, 257, 4099 (odd, n % 4 = 3), G·256 ± 1 and 2G·256 + 129 with G the device's SM count
(the last gives CTAs one, two and three tiles, the ragged tile on a CTA that has done full ones).  k: 1, C - 1, C, C + 1,
the coef_lanes steps (16/17, 32/33, 64/65, 128/129), the fused limit and one more, kcap and kcap + 1, 2 kcap + 3.
Column lists: contiguous, every other column, reversed, shuffled.

The module's CPU tests check the restatement itself: exact on small integers, within the Higham-Mary bound of the
float64 result on random data, and sensitive to the orders it pins.
"""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
import tsk_restate as ts
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.vectors import handles
from test_gpu_blas1 import fma, num_sms  # noqa: F401  (fma: module fixture)
from test_gpu_paths import LAM, PROJECT, SWEEP, UNPROJECT, coop, expected_orth_launches, profiled, unit

gpu = pytest.mark.gpu
f64, f32 = np.float64, np.float32
DT = [f64, f32]
DT_IDS = ["f64", "f32"]
EPS = {f64: 2.0 ** -52, f32: 2.0 ** -23}
NNAMES = ["1", "2", "3", "255", "256", "257", "4099", "G256-1", "G256+1", "2G256+129"]
LAYOUTS = ["strided", "reversed", "shuffled"]


def rows(name):
    G = num_sms()
    return {"G256-1": G * 256 - 1, "G256+1": G * 256 + 1, "2G256+129": 2 * G * 256 + 129}.get(name) or int(name)


def widths_k(dt):
    c, _, _, kcap, fused = ts.cfg(dt)
    return sorted({1, c - 1, c, c + 1, 16, 17, 32, 33, 64, 65, 128, 129, fused, fused + 1, kcap, kcap + 1,
                   2 * kcap + 3})


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(bits(a), bits(b))


def first_diff(got, want):
    bad = np.flatnonzero(bits(np.atleast_1d(got)) != bits(np.atleast_1d(want)))
    return f"{len(bad)} differ, first at {bad[0]}: {np.atleast_1d(got)[bad[0]]!r} != {np.atleast_1d(want)[bad[0]]!r}" \
        if len(bad) else "equal"


def column_list(ctx, k, layout, rng):
    """k basis vectors of the context's slab in the order of the column list"""
    if layout == "contiguous":
        return ctx.empty_range(k)
    if layout == "strided":
        return ctx.empty_range(2 * k)[::2]
    if layout == "reversed":
        return ctx.empty_range(2 * k)[::2][::-1]
    pool = ctx.empty_range(k + k // 2 + 1)
    return [pool[i] for i in rng.permutation(len(pool))[:k]]


def context(dt, n, k, layout):
    return kk.B200Context(n, (2 * k if layout != "contiguous" else k) + 12, dtype=dt)


def upload(vecs, Q):
    for j, v in enumerate(vecs):
        v.upload(Q[:, j])


def rand(rng, shape, dt):
    return rng.standard_normal(shape).astype(dt)


def passes_of(k, dt):
    return -(-k // ts.cfg(dt)[3])


# ------------------------------------------------------------------------------------------ CPU: the restatement ---

def test_restatement_exact_on_small_integers(fma):
    """integers in [-8, 8]: every partial sum is exact in T and in double, so projection, coefficients, update and norm
    are the exact integer results whatever the order"""
    rng = np.random.default_rng(1)
    for dt in DT:
        for n, k, nsm in ((3, 2, 132), (700, 20, 2), (1100, 70, 3), (600, 300, 2)):
            Qi = rng.integers(-8, 9, (n, k)).astype(dt)
            xi = rng.integers(-8, 9, n).astype(dt)
            h = ts.project(Qi, xi, nsm, fma)
            assert same(h, Qi.astype(f64).T @ xi.astype(f64))
            c = rng.integers(-4, 5, k).astype(f64)
            y = ts.update(Qi, xi, ts.coefs(c, -1.0, dt), fma)
            want = xi.astype(f64) - Qi.astype(f64) @ c
            assert np.abs(want).max() < 2 ** 22
            assert same(y, want.astype(dt))
            if 4 * (want ** 2).max() < 2 ** 24:      # each thread's squares then sum exactly in T
                assert ts.normsum(ts.norm_partials(y, nsm, fma)) == float(want @ want)


def test_restatement_within_the_float64_bound(fma):
    """random data: |restated - float64| <= LAM sqrt(m) u sum|terms| (Higham & Mary) for the projection (m = n products
    in T, then the double partial sums), the update (k + 1 terms) and the norm"""
    rng = np.random.default_rng(2)
    for dt in DT:
        u = unit(dt)
        for n, k, nsm in ((5000, 40, 7), (2 * 3 * 256 + 129, 270, 3)):
            Q, x = rand(rng, (n, k), dt), rand(rng, n, dt)
            Q64, x64 = Q.astype(f64), x.astype(f64)
            h = ts.project(Q, x, nsm, fma)
            S = np.abs(Q64).T @ np.abs(x64)
            assert np.all(np.abs(h - Q64.T @ x64) <= LAM * math.sqrt(n) * u * S)
            c = rng.standard_normal(k)
            cs = ts.coefs(c, -0.7, dt)
            y = ts.update(Q, x, cs, fma).astype(f64)
            cs64 = cs.astype(f64)
            assert np.all(np.abs(y - (x64 + Q64 @ cs64)) <= LAM * math.sqrt(k + 1) * u * (np.abs(x64) + np.abs(Q64) @ np.abs(cs64)))
            n2 = ts.normsum(ts.norm_partials(y.astype(dt), nsm, fma))
            assert abs(n2 - float(y @ y)) <= LAM * math.sqrt(n) * u * float(y @ y)


def test_restatement_tells_the_orders_apart(fma):
    """the bitwise contract can see the orders it pins: a reversed update, the prologue's v_prev / v added first and
    a reversed coefficient sum differ from the restatement"""
    rng = np.random.default_rng(3)
    dt = f32
    n, k = 3000, 40
    Q, x = rand(rng, (n, k), dt), rand(rng, n, dt)
    cs = ts.coefs(rng.standard_normal(k), -1.0, dt)
    y = ts.update(Q, x, cs, fma)
    assert not same(y, ts.update(Q[:, ::-1], x, cs[::-1], fma))
    V, v, w = Q[:, :k - 1], Q[:, k - 1], x
    Qp = np.column_stack([V, v])
    xp = ts.prologue(w, V[:, -1], v, 1.3, 0.7, fma)
    h = ts.project(Qp, xp, 5, fma)
    out = ts.update(Qp, xp, ts.coefs(h, -1.0, dt), fma)
    order = [k - 2, k - 1] + list(range(k - 2))            # v_prev and v first
    first = ts.update(Qp[:, order], xp, ts.coefs(h, -1.0, dt)[order], fma)
    assert not same(out, first)
    P = rng.standard_normal((132, 40)) * 10.0 ** rng.integers(-8, 8, (132, 40))
    assert not same(ts.colsum(P), ts.colsum(P[::-1]))
    assert ts.coef_lanes(16) == 16 and ts.coef_lanes(17) == 8 and ts.coef_lanes(129) == 1


# ------------------------------------------------------------------------------------------ GPU: project / unproject

def pu_cases():
    out = []
    for dt in DT:
        c, _, _, kcap, _ = ts.cfg(dt)
        out += [(dt, nn, k, "contiguous") for nn in NNAMES for k in (c + 1, 65)]
        out += [(dt, "2G256+129", k, "contiguous") for k in widths_k(dt)]
        out += [(dt, nn, k, lay) for lay in LAYOUTS for nn, k in (("G256+1", 2 * c + 3), ("257", kcap + 1))]
    return out


PU = pu_cases()


@gpu
@pytest.mark.parametrize("dt,nn,k,layout", PU, ids=[f"{np.dtype(d).name}-n{nn}-k{k}-{lay}" for d, nn, k, lay in PU])
def test_project_and_unproject(dt, nn, k, layout, fma):
    """b2k_basis_project with the host's alpha / beta fold, b2k_basis_unproject with beta = 0, 1 and general and
    alpha = 0.7 (T(alpha) * T(c_j) rounds twice in Float32)"""
    n = rows(nn)
    nsm = num_sms()
    rng = np.random.default_rng([n, k, len(layout)])
    ctx = context(dt, n, k, layout)
    try:
        vecs = column_list(ctx, k, layout, rng)
        Q, x = rand(rng, (n, k), dt), rand(rng, n, dt)
        upload(vecs, Q)
        xv = ctx.from_host(x)
        h0 = rng.standard_normal(k)
        h = h0.copy()
        with profiled(ctx) as cnt:
            ctx.check(ctx.lib.b2k_basis_project(ctx.h, handles(vecs), k, xv.handle, 0.7, -1.3,
                                                h.ctypes.data_as(C.POINTER(C.c_double))))
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == (0, passes_of(k, dt), 0), cnt
        want = -1.3 * h0 + 0.7 * ts.project(Q, x, nsm, fma)
        assert same(h, want), first_diff(h, want)
        c = rng.standard_normal(k)
        for beta, mode in ((0.0, 0), (1.0, 1), (-1.3, 2)):
            y = rand(rng, n, dt)
            yv = ctx.from_host(y)
            with profiled(ctx) as cnt:
                ctx.check(ctx.lib.b2k_basis_unproject(ctx.h, yv.handle, handles(vecs), k,
                                                      c.ctypes.data_as(C.POINTER(C.c_double)), 0.7, beta))
            assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == (0, 0, passes_of(k, dt)), cnt
            want = ts.update(Q, y, ts.coefs(c, 0.7, dt), fma, mode, beta)
            got = yv.to_host()
            assert same(got, want), (beta, first_diff(got, want))
            yv.free()
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ GPU: orthogonalize -----

CLASSICAL = [(L.CGS, None), (L.CGS2, None), (L.MGS2B, None), (L.CGSIR, 0.75)]


def orth_cases():
    out = []
    for dt in DT:
        c = ts.cfg(dt)[0]
        out += [(dt, "G256+1", k, "contiguous") for k in widths_k(dt)]
        out += [(dt, nn, c + 1, "contiguous") for nn in NNAMES]
        out += [(dt, "2G256+129", 65, "contiguous")]
        out += [(dt, "G256-1", 2 * c + 3, lay) for lay in LAYOUTS]
    return out


ORTH = orth_cases()


def orthogonalize(ctx, v, vecs, tag, eta):
    k = len(vecs)
    h = np.empty(k)
    nrm, passes = C.c_double(), C.c_int32()
    ctx.check(ctx.lib.b2k_basis_orthogonalize(ctx.h, v.handle, handles(vecs), k, h.ctypes.data_as(C.POINTER(C.c_double)),
                                              tag, eta, C.byref(nrm), C.byref(passes)))
    return h, nrm.value, passes.value


def restate_orth(Q, v, tag, eta, nold, nsm, fma):
    """(h, v, ||v||, passes) of the classical orthogonalizers; CGSIR loops while eps < nnew < eta nold"""
    dt = Q.dtype.type
    if tag in (L.CGS, L.CGS2, L.MGS2B):
        h, out, n2 = ts.cgs(Q, v, 1 if tag == L.CGS else 2, nsm, fma)
        return h, out, math.sqrt(n2), 1 if tag == L.CGS else 2
    hsum, passes = np.zeros(Q.shape[1]), 0
    while True:
        h, v, n2 = ts.cgs(Q, v, 1, nsm, fma)
        passes += 1
        hsum = hsum + h
        nnew = math.sqrt(n2)
        if not (EPS[dt] < nnew < eta * nold):
            return hsum, v, nnew, passes
        nold = nnew


@gpu
@pytest.mark.parametrize("dt,nn,k,layout", ORTH, ids=[f"{np.dtype(d).name}-n{nn}-k{k}-{lay}" for d, nn, k, lay in ORTH])
def test_orthogonalize_classical(dt, nn, k, layout, fma):
    """CGS, CGS2, MGS2B (two classical passes) and CGSIR: fused cooperative, one launch per phase, and the unfused
    passes past the fused limit.  v has half its norm outside the basis: CGSIR takes two passes."""
    n = rows(nn)
    nsm = num_sms()
    rng = np.random.default_rng([n, k, len(layout), 7])
    ctx = context(dt, n, k + 2, layout)
    try:
        vecs = column_list(ctx, k, layout, rng)
        Q = (rng.standard_normal((n, k)) / math.sqrt(n)).astype(dt)
        upload(vecs, Q)
        for tag, eta in CLASSICAL:
            vh = (Q.astype(f64) @ rng.standard_normal(k) + 0.5 * math.sqrt(k / n) * rng.standard_normal(n)
                  ).astype(dt)
            runs = {}
            for on in (True, False):
                v = ctx.from_host(vh)
                nold = v.norm()
                with coop(on):
                    l0 = ctx.launches
                    with profiled(ctx) as cnt:
                        h, nrm, passes = orthogonalize(ctx, v, vecs, tag, eta or 0.0)
                    runs[on] = (h, nrm, passes, v.to_host(), ctx.launches - l0, dict(cnt))
                v.free()
            h, nrm, passes, out, nl, cnt = runs[True]
            assert same(h, runs[False][0]) and same(out, runs[False][3]) and nrm == runs[False][1], tag
            wh, wv, wn, wp = restate_orth(Q, vh, tag, eta, nold, nsm, fma)
            assert passes == wp, (tag, passes, wp)
            assert same(h, wh), (tag, first_diff(h, wh))
            assert same(out, wv), (tag, first_diff(out, wv))
            assert nrm == wn, (tag, nrm, wn)
            sweeps, proj, unproj, saved = expected_orth_launches(tag, k, dt, passes)
            assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == (sweeps, proj, unproj), (tag, cnt)
            assert runs[False][4] - nl == saved, (tag, runs[False][4], nl)
    finally:
        ctx.close()


def literal_mgs(v, vecs, passes):
    """the reference's modified Gram-Schmidt loop through b2k_vec_inner / b2k_vec_axpby: h summed over the passes"""
    h = np.zeros(len(vecs))
    for _ in range(passes):
        for j, q in enumerate(vecs):
            s = q.inner(v)
            v.add_(q, -s)
            h[j] += s
    return h


MGS_CASES = [(dt, nn, k) for dt in DT for nn, k in (("G256+1", 1), ("G256+1", 3), ("G256+1", 4), ("257", 9),
                                                    ("2G256+129", 5), ("3", 2))]


@gpu
@pytest.mark.parametrize("tag", [L.MGS, L.MGS2, L.MGSIR], ids=["MGS", "MGS2", "MGSIR"])
@pytest.mark.parametrize("dt,nn,k", MGS_CASES, ids=[f"{np.dtype(d).name}-n{nn}-k{k}" for d, nn, k in MGS_CASES])
def test_orthogonalize_mgs_equals_the_literal_loop(dt, nn, k, tag):
    """the pipelined k_dot<UPDATE> sweep (L2 hints from k = 4 on) gives the bits of inner / add!!(v, q_j, -s_j, 1)
    called in turn; MGSIR loops on the same norms"""
    n = rows(nn)
    rng = np.random.default_rng([n, k, tag])
    ctx = kk.B200Context(n, k + 8, dtype=dt)
    try:
        vecs = ctx.empty_range(k)
        Q = (rng.standard_normal((n, k)) / math.sqrt(n)).astype(dt)
        upload(vecs, Q)
        vh = (Q.astype(f64) @ rng.standard_normal(k) + 0.5 * math.sqrt(k / n) * rng.standard_normal(n)
              ).astype(dt)
        res = {}
        for on in (True, False):
            v = ctx.from_host(vh)
            with coop(on), profiled(ctx) as cnt:
                h, nrm, passes = orthogonalize(ctx, v, vecs, tag, 0.75)
            assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == (0, 0, 0), cnt
            res[on] = (h, nrm, passes, v.to_host())
            v.free()
        assert all(same(a, b) for a, b in zip(res[True], res[False]))
        h, nrm, passes, out = res[True]
        vl = ctx.from_host(vh)
        if tag == L.MGSIR:
            nold = vl.norm()
            hl, lp = literal_mgs(vl, vecs, 1), 1
            nnew = vl.norm()
            while EPS[dt] < nnew < 0.75 * nold:
                nold = nnew
                hl = hl + literal_mgs(vl, vecs, 1)
                lp += 1
                nnew = vl.norm()
        else:
            lp = 1 if tag == L.MGS else 2
            h1 = literal_mgs(vl, vecs, 1)
            hl = h1 if lp == 1 else h1 + literal_mgs(vl, vecs, 1)
            nnew = vl.norm()
        assert passes == lp
        assert same(h, hl), first_diff(h, hl)
        assert same(out, vl.to_host()) and nrm == nnew
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ GPU: a Lanczos step ----

def tridiag(n, dt, rng):
    d, e = rng.standard_normal(n), rng.standard_normal(max(n - 1, 0))
    return sp.diags([e, d, e], [-1, 0, 1], shape=(n, n), format="csr").astype(dt)


def lanczos_setup(dt, n, k, rng):
    """context, operator, basis V (k columns: q_0 ... q_{k-2}, v_prev), the residual r and beta_old"""
    ctx = kk.B200Context(n, k + 12, dtype=dt)
    op = kk.B200CSR.from_scipy(ctx, tridiag(n, dt, rng))
    vecs = ctx.empty_range(k + 1)
    V = (rng.standard_normal((n, k)) / math.sqrt(n)).astype(dt)
    upload(vecs[:k], V)
    r = rng.standard_normal(n)
    rh = (1.7 * r / np.linalg.norm(r)).astype(dt)     # v = r / beta_old of unit length
    return ctx, op, vecs[:k], vecs[k], V, rh, 1.7


def expand(ctx, op, V, r, w, beta_old, tag, eta):
    a, b = C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_lanczos_expand(ctx.h, op.h, handles(V + [r]), len(V), r.handle, w.handle, beta_old, tag,
                                         eta, C.byref(a), C.byref(b)))
    return a.value, b.value


def run_expand(ctx, op, Vv, r, rh, beta_old, tag, eta):
    """the step with the cooperative sweep on and off: both give the same bits; returns (alpha, beta, w, v, counts,
    launches saved)"""
    runs = {}
    for on in (True, False):
        r.upload(rh)
        w = ctx.empty()
        with coop(on):
            l0 = ctx.launches
            with profiled(ctx) as cnt:
                a, b = expand(ctx, op, Vv, r, w, beta_old, tag, eta)
            runs[on] = (a, b, w.to_host(), r.to_host(), dict(cnt), ctx.launches - l0)
        w.free()
    for x, y in zip(runs[True][:4], runs[False][:4]):
        assert same(x, y), tag
    a, b, wd, vd, cnt, nl = runs[True]
    return a, b, wd, vd, cnt, runs[False][5] - nl


def step_inputs(ctx, op, rh, beta_old, dt):
    """v = scale!!(r, 1/beta_old) and (w, alpha0) from b2k_op_apply_dot(op, v, w, v), the SpMV + fused dot the step uses"""
    v = (dt(1.0 / beta_old) * rh).astype(dt)
    vv, wv = ctx.from_host(v), ctx.empty()
    a0 = op.apply_dot_into(wv, vv, vv)
    w = wv.to_host()
    vv.free()
    wv.free()
    return v, w, a0


def band(K1, dt):
    _, _, _, kcap, fused = ts.cfg(dt)
    return "fused" if K1 <= fused else ("split" if K1 <= kcap else "unfused")


def lanczos_cases():
    out = []
    for dt in DT:
        c, _, _, kcap, fused = ts.cfg(dt)
        out += [(dt, "G256+1", K1) for K1 in (2, c + 1, 33, fused, fused + 1, kcap, kcap + 1)]
        out += [(dt, nn, c + 1) for nn in ("3", "257", "4099", "G256-1", "2G256+129")]
        out += [(dt, "2G256+129", 65)]
    return out


LZ = lanczos_cases()


@gpu
@pytest.mark.parametrize("dt,nn,K1", LZ, ids=[f"{np.dtype(d).name}-n{nn}-K{K1}" for d, nn, K1 in LZ])
def test_lanczos_step_cgs2_and_cgsir(dt, nn, K1, fma):
    """b2k_lanczos_expand with CGS2 (fused sweep, split sweeps with alpha deferred on the device, unfused passes) and
    CGSIR: w, v = r / beta_old, alpha and beta bit for bit.  alpha0 comes from the SpMV's fused dot; alpha adds h[k]
    of every pass on the host."""
    n, k = rows(nn), K1 - 1
    nsm = num_sms()
    rng = np.random.default_rng([n, K1, 11])
    ctx, op, Vv, r, V, rh, beta_old = lanczos_setup(dt, n, k, rng)
    try:
        v, w0, a0 = step_inputs(ctx, op, rh, beta_old, dt)
        Q = np.column_stack([V, v])
        nch = passes_of(K1, dt)
        # CGS2: the prologue, one classical pass over [V, v]
        a, b, wd, vd, cnt, saved = run_expand(ctx, op, Vv, r, rh, beta_old, L.CGS2, 0.0)
        assert same(vd, v)
        ww, wa, wn2, _ = ts.lanczos_step(V, v, w0, beta_old, a0, 1, nsm, fma)
        assert same(wd, ww), first_diff(wd, ww)
        assert a == wa and b == math.sqrt(wn2), (a, wa, b, math.sqrt(wn2))
        want = {"fused": (1, 0, 0, 1), "split": (1, 0, 0, 0), "unfused": (0, nch, nch, 0)}[band(K1, dt)]
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT], saved) == want, (cnt, saved)
        # CGSIR: w' = axpy2, beta = ||w'|| (BLAS-1 norm), then classical passes without the prologue while
        # eps < beta < eta nold
        eta = 0.9
        xp = ts.prologue(w0, V[:, -1], v, beta_old, a0, fma)
        tmp = ctx.from_host(xp)
        beta = tmp.norm()
        tmp.free()
        nold = math.sqrt(beta * beta + (a0 * a0 + beta_old * beta_old))
        alpha, x, npass = a0, xp, 0
        while EPS[dt] < beta < eta * nold:
            nold = beta
            h, x, n2 = ts.cgs(Q, x, 1, nsm, fma)
            alpha = alpha + h[k]
            beta = math.sqrt(n2)
            npass += 1
        a, b, wd, vd, cnt, saved = run_expand(ctx, op, Vv, r, rh, beta_old, L.CGSIR, eta)
        assert npass >= 1
        assert same(wd, x), first_diff(wd, x)
        assert a == alpha and b == beta, (a, alpha, b, beta)
        want = {"fused": (npass, 0, 0, npass), "split": (npass, 0, 0, 0),
                "unfused": (0, nch * npass, nch * npass, 0)}[band(K1, dt)]
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT], saved) == want, (cnt, saved, npass)
    finally:
        ctx.close()


def literal_lanczos_mgs(op, V, r, w, beta_old, tag, eta, dt):
    """lanczos.jl:304-312, 325-338, 357-376 as BLAS-1 calls: (alpha, beta)"""
    r.scale_(1.0 / beta_old)
    op.apply_into(w, r)
    w.add_(V[-1], -beta_old)
    alpha = r.inner(w)
    w.add_(r, -alpha)
    beta = w.norm()
    if tag == L.MGS:
        return alpha, beta
    if tag == L.MGS2:
        s = literal_mgs(w, V + [r], 1)
        return alpha + s[-1], w.norm()
    nold = math.sqrt(beta * beta + alpha * alpha + beta_old * beta_old)
    while EPS[dt] < beta < eta * nold:
        nold = beta
        s = literal_mgs(w, V + [r], 1)
        alpha += s[-1]
        beta = w.norm()
    return alpha, beta


LZM = [(dt, nn, K1) for dt in DT for nn, K1 in (("G256+1", 2), ("G256+1", 4), ("G256+1", 5), ("2G256+129", 9),
                                                ("257", 3))]


@gpu
@pytest.mark.parametrize("tag", [L.MGS, L.MGS2, L.MGSIR], ids=["MGS", "MGS2", "MGSIR"])
@pytest.mark.parametrize("dt,nn,K1", LZM, ids=[f"{np.dtype(d).name}-n{nn}-K{K1}" for d, nn, K1 in LZM])
def test_lanczos_step_mgs_equals_the_literal_sequence(dt, nn, K1, tag):
    n, k = rows(nn), K1 - 1
    rng = np.random.default_rng([n, K1, tag])
    ctx, op, Vv, r, V, rh, beta_old = lanczos_setup(dt, n, k, rng)
    try:
        a, b, wd, vd, cnt, saved = run_expand(ctx, op, Vv, r, rh, beta_old, tag, 0.9)
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT], saved) == (0, 0, 0, 0), cnt
        rl, wl = ctx.from_host(rh), ctx.empty()
        al, bl = literal_lanczos_mgs(op, Vv, rl, wl, beta_old, tag, 0.9, dt)
        assert same(vd, rl.to_host()) and same(wd, wl.to_host()), first_diff(wd, wl.to_host())
        assert a == al and b == bl, (a, al, b, bl)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ GPU: dense GEMV --------

GEMV = [(dt, m, nc) for dt in DT for m in ("33", "G256+1")
        for nc in ([1, 127, 128, 129, 300] + ([511, 512, 513] if dt == f32 else []))]


@gpu
@pytest.mark.parametrize("dt,mm,ncols", GEMV, ids=[f"{np.dtype(d).name}-m{m}-c{c}" for d, m, c in GEMV])
def test_dense_gemv(dt, mm, ncols, fma):
    """apply_normal: y = fold_j fma(A[:, j], x_j, acc) from +0 (unproject passes, coefficients T(1) x_j);
    apply_adjoint: z = T(project(A, u)) (project passes, then the result cast to T)"""
    m = rows(mm)
    nsm = num_sms()
    rng = np.random.default_rng([m, ncols])
    ctx = kk.B200Context(m, 8, dtype=dt)
    try:
        sv = ctx.add_space(ncols, 8, sharded=False)
        A = rand(rng, (m, ncols), dt)
        op = kk.B200Dense.from_host(ctx, A, sv)
        x, u = rand(rng, ncols, dt), rand(rng, m, dt)
        with profiled(ctx) as cnt:
            y = kk.apply_normal(op, ctx.from_host(x, sv)).to_host()
        assert cnt[UNPROJECT] == passes_of(ncols, dt) and cnt[PROJECT] == 0
        want = ts.update(A, np.zeros(m, dtype=dt), x, fma, beta_mode=0)
        assert same(y, want), first_diff(y, want)
        with profiled(ctx) as cnt:
            z = kk.apply_adjoint(op, ctx.from_host(u)).to_host()
        assert cnt[PROJECT] == passes_of(ncols, dt) and cnt[UNPROJECT] == 0
        want = ts.project(A, u, nsm, fma).astype(dt)
        assert same(z, want), first_diff(z, want)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ GPU: edges -------------

@gpu
@pytest.mark.parametrize("dt", DT, ids=DT_IDS)
def test_stale_ring_rows_of_the_ragged_tile(dt, fma):
    """One Inf in basis column i, at a row of CTA 0's first tile that lies past the end of its ragged last tile (n =
    G 256 + 100: CTA 0 owns tiles 0 and G).  With 8 chunks per tile the ring (12 slots) wraps: tile G's chunk 5 lands
    in the slot that held column i's chunk at tile 0, and the bulk copy of the ragged tile leaves the slot's rows >= 100
    as tile 0 left them.  Those rows are multiplied by x = 0: the column now at the Inf's slot position must still get a
    finite coefficient, the one of the restatement (only h_i is infinite)."""
    c, _, _, _, _ = ts.cfg(dt)
    nsm = num_sms()
    G = nsm
    rt, bad_row = 100, 200
    n = G * 256 + rt
    k = 8 * c
    nch = k // c
    i = 1 * c + 3                                       # chunk 1, slot position 3
    s = ts.slot_of(0, 1, nch)
    c2 = next(cc for cc in range(nch) if ts.slot_of(1, cc, nch) == s)
    j = c2 * c + 3
    assert (n - 1) // 256 % ts.grid(n, nsm) == 0 and c2 != 1 and j != i
    rng = np.random.default_rng(5)
    ctx = kk.B200Context(n, k + 4, dtype=dt)
    try:
        vecs = ctx.empty_range(k)
        Q = rand(rng, (n, k), dt)
        Q[bad_row, i] = np.inf
        upload(vecs, Q)
        x = rand(rng, n, dt)
        xv = ctx.from_host(x)
        h = np.empty(k)
        ctx.check(ctx.lib.b2k_basis_project(ctx.h, handles(vecs), k, xv.handle, 1.0, 0.0,
                                            h.ctypes.data_as(C.POINTER(C.c_double))))
        want = ts.project(Q, x, nsm, fma)
        assert np.isinf(want[i]) and np.isfinite(np.delete(want, i)).all()
        assert np.isfinite(h[j]), (i, j, h[j])
        assert same(h, want), first_diff(h, want)
    finally:
        ctx.close()


@gpu
def test_ir_threshold_is_eps_of_float32():
    """||v'|| = sqrt(2^-46 + 2^-76) lies in (2^-23, 1.1920929e-07]: above eps(Float32) = 2^-23, so CGSIR and MGSIR
    take a second pass (orthonormal.jl: eps(T) < nnew < eta nold), both in orthogonalize!! and in a Lanczos step.  The
    two squares sit in different rows (threads) and are added in double, so the sum is exact."""
    nnew = math.sqrt(2.0 ** -46 + 2.0 ** -76)
    assert 2.0 ** -23 < nnew <= 1.1920929e-07
    n = 3
    ctx = kk.B200Context(n, 8, dtype=f32)
    try:
        q = ctx.from_host(np.array([1.0, 0.0, 0.0]))
        for tag in (L.CGSIR, L.MGSIR):
            v = ctx.from_host(np.array([1.0, 2.0 ** -23, 2.0 ** -38]))
            h, nrm, passes = orthogonalize(ctx, v, [q], tag, 0.75)
            assert passes == 2 and nrm == nnew and h[0] == 1.0, (tag, passes, nrm)
        # Lanczos: V = [e0], r = e1, A e1 = (1 + 2^-23, a11, 2^-38): w' = (2^-23, 0, 2^-38) after the prologue
        A = sp.csr_matrix(np.array([[0.0, 1.0 + 2.0 ** -23, 0.0], [1.0 + 2.0 ** -23, 0.5, 2.0 ** -38],
                                    [0.0, 2.0 ** -38, 0.0]]))
        op = kk.B200CSR.from_scipy(ctx, A)
        for tag in (L.CGSIR, L.MGSIR):
            r = ctx.from_host(np.array([0.0, 1.0, 0.0]))
            w = ctx.empty()
            a, b = expand(ctx, op, [q], r, w, 1.0, tag, 0.9)
            # the reorthogonalisation pass removes 2^-23 e0: beta = 2^-38, alpha = 0.5 + 0
            assert b == 2.0 ** -38 and a == 0.5, (tag, a, b)
            assert np.array_equal(w.to_host(), np.array([0.0, 0.0, 2.0 ** -38], dtype=f32))
            r.free()
            w.free()
    finally:
        ctx.close()
