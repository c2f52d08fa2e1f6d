"""GPU tests of the dispatcher branches behind the default ones: Gram-Schmidt and Lanczos steps on both sides of every
width threshold (fused / split sweeps / unfused chunked passes), the device-chained batch at its width limit, solvers
with krylovdim past 128, the SpMV arithmetic contract (rounded products summed in CSR order) for all three CSR kernels
in Float64 and Float32, SpMM against single applies on long rows, the Float32 stencils and chains, and the dense GEMV
at its chunk edges.

Every boundary test asserts which branch ran, from the per-class launch counts of b2k_prof_read (0 = SpMV, 1 = fused
Gram-Schmidt sweep, 2 = basis transform, 3 = project pass, 4 = unproject pass, 7 = SpMM) and from ctx.launches.

Tolerances.  u is the unit roundoff of the vector type (2^-53 / 2^-24).  Unless a test states otherwise, a sum of m
rounded terms is allowed to be off by LAM * sqrt(m) * u * sum(|terms|): the probabilistic bound of Higham & Mary
(SIAM J. Sci. Comput. 41(5), 2019), which a sum violates with probability below 2 m exp(-LAM^2 / 2) (< 1e-9 here).
"""
import contextlib
import ctypes as C
import gc
import math

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.factorizations import lanczos as lz
from krylovkit_jl_b200.vectors import handles
from oracle import krylov_oracle as ko

SEED = 20260923
LAM = 8.0
SPMV, SWEEP, TRANSFORM, PROJECT, UNPROJECT, SPMM = 0, 1, 2, 3, 4, 7
SP_NNZ = 1536            # nonzeros of one CSR row tile (spmv.cu); longer rows get a CTA of their own
f64, f32 = np.float64, np.float32


def unit(dtype):
    return 2.0 ** -53 if dtype == f64 else 2.0 ** -24


def widths(dtype):
    """(fused limit, columns per unfused pass): the resident ring holds 12 chunks of 8 (f64) / 16 (f32) columns, an
    unfused pass takes 16 chunks (tsk.cuh NS, MAXCH)."""
    c = 8 if dtype == f64 else 16
    return 12 * c, 16 * c


@contextlib.contextmanager
def profiled(ctx):
    """launch counts per profile class of what runs inside the block"""
    counts = {}
    ctx.check(ctx.lib.b2k_prof_reset(ctx.h))
    ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 1))
    try:
        yield counts
    finally:
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 0))
        for cls in (SPMV, SWEEP, TRANSFORM, PROJECT, UNPROJECT, SPMM):
            c = C.c_int64()
            ctx.check(ctx.lib.b2k_prof_read(ctx.h, cls, C.byref(c), None, None))
            counts[cls] = c.value


@contextlib.contextmanager
def coop(on):
    lib = L.load()
    lib.b2k_debug_set_coop(1 if on else 0)
    try:
        yield
    finally:
        lib.b2k_debug_set_coop(1)


_Q = {}


def qbasis(n, k):
    """n x k orthonormal columns (float64), reused across tests: a prefix of the columns of one QR factor"""
    if n not in _Q or _Q[n].shape[1] < k:
        kq = max(k, 513) if n >= 4 * 513 else k
        _Q[n] = np.linalg.qr(np.random.default_rng(n).standard_normal((n, kq)))[0]
    return _Q[n][:, :k]


def upload_basis(ctx, Q, contiguous=True):
    """Q's columns as device vectors (one slab range, or every other column of a range); returns the stored values
    as float64 (Float32 contexts round them) and the vectors"""
    k = Q.shape[1]
    if contiguous:
        vecs = ctx.empty_range(k)
    else:
        vecs = [ctx.empty() for _ in range(2 * k)][::2]
    Qt = np.ascontiguousarray(Q.T, dtype=ctx.np_dtype)
    for j, v in enumerate(vecs):
        v.upload(Qt[j])
    return Qt.T.astype(f64), vecs


def orthogonalize(ctx, v, vecs, alg):
    """orthogonalize!!(v, b, alg) as kk.orthogonalize_ calls it, also returning the number of passes"""
    k = len(vecs)
    h = np.empty(k)
    nrm, passes = C.c_double(), C.c_int32()
    ctx.check(ctx.lib.b2k_basis_orthogonalize(ctx.h, v.handle, handles(vecs), k, h.ctypes.data_as(C.POINTER(C.c_double)),
                                              alg.tag, alg.eta, C.byref(nrm), C.byref(passes)))
    return h, nrm.value, passes.value


def oracle_orth(alg):
    # the flagged blocked MGS2 of orthogonalize!! is two classical passes
    return ko.Orth(ko.CGS2 if alg.tag == L.MGS2B else alg.tag, alg.eta)


ALGS = [kk.cgs, kk.mgs, kk.cgs2, kk.mgs2, kk.ClassicalGramSchmidtIR(eta=0.75), kk.ModifiedGramSchmidtIR(eta=0.75),
        kk.mgs2b]
CLASSICAL = (L.CGS, L.CGS2, L.CGSIR, L.MGS2B)


# ------------------------------------------------------------------------------------------ 1. Gram-Schmidt --------

def gs_tols(n, k, u, nv, passes):
    """Bounds on |device - oracle| after `passes` Gram-Schmidt passes of v (norm nv) against k orthonormal columns of
    length n.  Per pass, for the vector w it starts from (|w| <= nv, |h| <= |w|):
      coefficient <q_j, w>, n terms:        |dh_j| <= LAM sqrt(n) u nv                 (sum |q_ij w_i| <= |q_j| |w|)
      update w - sum_j h_j q_j, k+1 terms:  |dw|   <= LAM sqrt(k+1) u (1 + sqrt(k)) nv   (| |Q| |_2 <= sqrt(k))
                                                      + sqrt(k) max_j |dh_j|             (|Q dh| <= sqrt(k) max |dh|)
    A coefficient of a later pass sees the earlier update's rounding but not its coefficient errors (q_j' Q dh =
    dh_j, cancelled by the pass).  Summed over the passes, doubled for the float64 oracle's own rounding.
    Returns (max |dx_j|, |d out|_2)."""
    eh = LAM * math.sqrt(n) * u * nv
    eu = LAM * math.sqrt(k + 1) * u * (1 + math.sqrt(k)) * nv
    return 2 * passes * (eh + eu), 2 * passes * (math.sqrt(k) * eh + eu)


def expected_orth_launches(tag, k, dtype, passes):
    """(sweeps, project passes, unproject passes, launches saved by the cooperative sweep) of one orthogonalize"""
    fused_max, per_pass = widths(dtype)
    if tag not in CLASSICAL:
        return 0, 0, 0, 0
    if k <= fused_max:
        # one fused call per classical pass set: CGS = phases (project, update), CGS2 = (project, update+project,
        # update); CGSIR runs one CGS call per pass.  Cooperative: one launch per call instead of one per phase.
        if tag == L.CGSIR:
            return passes, 0, 0, passes
        return 1, 0, 0, (1 if tag == L.CGS else 2)
    nch = -(-k // per_pass)
    return 0, passes * nch, passes * nch, 0


ORTH_CASES = [(f64, k) for k in (96, 97, 128, 129, 256, 257)] + [(f32, k) for k in (192, 193, 256, 257, 513)]


@pytest.mark.parametrize("contiguous", [True, False], ids=["contiguous", "strided"])
@pytest.mark.parametrize("dtype,k", ORTH_CASES, ids=[f"{np.dtype(d).name}-k{k}" for d, k in ORTH_CASES])
def test_orthogonalize_across_width_thresholds(dtype, k, contiguous):
    """orthogonalize!! with each orthogonalizer on both sides of the fused limit (96 / 192 columns) and of the chunk
    width of the unfused passes (128 / 256), against the float64 restatement on the downloaded basis and vector.  v has
    half its norm outside the basis, so the IR variants take exactly two passes (0.45 < eta = 0.75 after the first,
    ~1 after the second)."""
    n = 9973                             # ragged: 38 row tiles of 256 and 245 rows
    u = unit(dtype)
    ctx = kk.B200Context(n, 2 * k + 8, dtype=dtype)
    Q, vecs = upload_basis(ctx, qbasis(n, k), contiguous)
    Qrows = list(np.ascontiguousarray(Q.T))
    rng = np.random.default_rng(k + contiguous)
    for alg in ALGS:
        name = type(alg).__name__ + ("B" if alg.tag == L.MGS2B else "")
        vh = (Q @ rng.standard_normal(k) + 0.5 * math.sqrt(k / n) * rng.standard_normal(n)).astype(dtype)
        v64 = vh.astype(f64)
        runs = {}
        for on in (True, False):
            v = ctx.from_host(vh)
            with coop(on):
                l0 = ctx.launches
                with profiled(ctx) as cnt:
                    h, nrm, passes = orthogonalize(ctx, v, vecs, alg)
                runs[on] = (h, nrm, passes, v.to_host(), ctx.launches - l0, cnt)
            v.free()
        h, nrm, passes, out, nl, cnt = runs[True]
        assert passes == {L.CGS: 1, L.MGS: 1}.get(alg.tag, 2), (name, passes)
        # the cooperative launch and the launch per phase compute the same bits
        assert np.array_equal(h, runs[False][0]) and nrm == runs[False][1] and np.array_equal(out, runs[False][3]), name
        sweeps, proj, unproj, saved = expected_orth_launches(alg.tag, k, dtype, passes)
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == (sweeps, proj, unproj), (name, cnt)
        assert runs[False][4] - nl == saved, (name, runs[False][4], nl)
        oout, ox = ko.orthogonalize(v64.copy(), Qrows, np.zeros(k), oracle_orth(alg))
        out = out.astype(f64)
        nv = float(np.linalg.norm(v64))
        tx, tv = gs_tols(n, k, u, nv, passes)
        assert np.abs(h - ox).max() <= tx, (name, np.abs(h - ox).max(), tx)
        assert np.linalg.norm(out - oout) <= tv, (name, np.linalg.norm(out - oout), tv)
        assert np.abs(Q.T @ out).max() <= tv + np.abs(Q.T @ oout).max(), name
        # ||v|| from the last update's partial sums: n squares (the row values are the downloaded ones)
        assert abs(nrm - np.linalg.norm(out)) <= 2 * LAM * math.sqrt(n) * u * nv, name
        # |v|^2 = |x|^2 + |v - Q x|^2 up to the errors of x and of the result
        assert abs(math.hypot(np.linalg.norm(h), nrm) - nv) <= math.sqrt(k) * tx + tv, name
    ctx.close()


def test_orthogonalize_at_the_width_limit():
    """k = 2040 (the most the result buffer takes) runs the chunked unfused passes; 2041 is refused.  The basis is a
    permuted set of unit vectors, so every coefficient and every entry of the result is exact: bit-for-bit checks."""
    n, k = 2053, 2040
    rng = np.random.default_rng(2040)
    perm = rng.permutation(n)
    ctx = kk.B200Context(n, k + 8)
    vecs = ctx.empty_range(k + 1)
    for j, q in enumerate(vecs):
        e = np.zeros(n)
        e[perm[j]] = 1.0
        q.upload(e)
    vh = rng.standard_normal(n)
    want = vh.copy()
    want[perm[:k]] = 0.0
    _, per_pass = widths(f64)
    nch = -(-k // per_pass)
    for alg, launches in ((kk.cgs2, (0, 2 * nch, 2 * nch)), (kk.mgs, (0, 0, 0))):
        v = ctx.from_host(vh)
        with profiled(ctx) as cnt:
            h, nrm, passes = orthogonalize(ctx, v, vecs[:k], alg)
        assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT]) == launches, cnt
        assert np.array_equal(h, vh[perm[:k]])
        assert np.array_equal(v.to_host(), want)
        assert abs(nrm - np.linalg.norm(want)) <= 2 * LAM * math.sqrt(n) * unit(f64) * np.linalg.norm(vh)
        v.free()
    v = ctx.from_host(vh)
    with pytest.raises(kk.B200Error):
        orthogonalize(ctx, v, vecs, kk.cgs2)
    assert np.array_equal(v.to_host(), vh)           # refused before anything ran
    ctx.close()


def test_project_at_the_result_buffer_limit():
    """project!! of 8184 columns (the result buffer less its 8 scalar slots) in 64 chunked passes; 8185 is refused."""
    n, k = 33, 8184
    rng = np.random.default_rng(8184)
    B = rng.standard_normal((k + 1, n))
    ctx = kk.B200Context(n, k + 4)
    vecs = ctx.empty_range(k + 1)
    for j, q in enumerate(vecs):
        q.upload(B[j])
    xh = rng.standard_normal(n)
    x = ctx.from_host(xh)
    y = np.zeros(k)
    with profiled(ctx) as cnt:
        kk.project_(y, kk.OrthonormalBasis(vecs[:k]), x)
    assert cnt[PROJECT] == -(-k // widths(f64)[1]) == 64
    # n products summed per column, doubled for the float64 reference
    bound = 2 * LAM * math.sqrt(n) * unit(f64) * (np.abs(B[:k]) @ np.abs(xh))
    assert np.all(np.abs(y - B[:k] @ xh) <= bound)
    with pytest.raises(ValueError):
        kk.project_(np.zeros(k + 1), kk.OrthonormalBasis(vecs), x)
    ctx.close()


@pytest.mark.parametrize("dtype,k", [(f64, 257), (f32, 513)])
def test_unproject_applies_beta_once_across_chunks(dtype, k):
    """unproject!!(y, b, c, alpha, beta) with beta not in {0, 1} and three chunked passes: beta scales y once (in the
    first pass), the later passes add to it."""
    n = 4099
    rng = np.random.default_rng(k)
    ctx = kk.B200Context(n, k + 8, dtype=dtype)
    Q, vecs = upload_basis(ctx, qbasis(n, k))
    c = rng.standard_normal(k)
    yh = rng.standard_normal(n).astype(dtype)
    y = ctx.from_host(yh)
    alpha, beta = 0.7, -1.3
    with profiled(ctx) as cnt:
        kk.unproject_(y, kk.OrthonormalBasis(vecs), c, alpha, beta)
    assert cnt[UNPROJECT] == 3 and cnt[PROJECT] == 0
    y64 = yh.astype(f64)
    ref = beta * y64 + alpha * (Q @ c)
    # per row: beta*y, then k fused multiply-adds (coefficients alpha*c_j rounded to the vector type): k + 2 roundings
    u = unit(dtype)
    bound = 2 * LAM * math.sqrt(k + 2) * u * (abs(beta) * np.abs(y64) + abs(alpha) * (np.abs(Q) @ np.abs(c)))
    assert np.all(np.abs(y.to_host().astype(f64) - ref) <= bound)
    ctx.close()


# ------------------------------------------------------------------------------------------ 2. one Lanczos step ----

def lanczos_expand(ctx, op, V, r, w, beta_old, alg):
    a, b = C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_lanczos_expand(ctx.h, op.h, handles(V + [r]), len(V), r.handle, w.handle, beta_old, alg.tag,
                                         alg.eta, C.byref(a), C.byref(b)))
    return a.value, b.value


STEP_CASES = [(f64, K1) for K1 in (96, 97, 128, 129, 257)] + [(f32, K1) for K1 in (192, 193, 256, 257)]


@pytest.mark.parametrize("dtype,K1", STEP_CASES, ids=[f"{np.dtype(d).name}-K{K1}" for d, K1 in STEP_CASES])
def test_lanczos_step_at_each_width_boundary(dtype, K1):
    """b2k_lanczos_expand with K1 = k + 1 basis vectors after push!, around the fused limit (96 / 192), the split-sweep
    band (up to 128 / 256, alpha deferred on the device for CGS2) and the unfused chunked passes, for every
    orthogonalizer with the cooperative sweep on and off, against lanczosrecurrence on the same host data."""
    nx, ny = 61, 53
    n = nx * ny
    u = unit(dtype)
    A = ko.stencil_matrix(nx, ny)
    k = K1 - 1
    Qf = qbasis(n, K1)
    ctx = kk.B200Context(n, K1 + 8, dtype=dtype)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    V, Vvecs = upload_basis(ctx, Qf[:, :k])
    Vrows = list(np.ascontiguousarray(V.T))
    beta_old = 2.5
    rh = (beta_old * Qf[:, k]).astype(dtype)
    r = ctx.from_host(rh)
    fused_max, per_pass = widths(dtype)
    nch = -(-K1 // per_pass)
    for alg in ALGS:
        name = type(alg).__name__ + ("B" if alg.tag == L.MGS2B else "")
        runs = {}
        for on in (True, False):
            r.upload(rh)
            w = ctx.empty()
            with coop(on):
                l0 = ctx.launches
                with profiled(ctx) as cnt:
                    a, b = lanczos_expand(ctx, op, Vvecs, r, w, beta_old, alg)
                runs[on] = (a, b, w.to_host(), r.to_host(), ctx.launches - l0, cnt)
            w.free()
        a, b, wd, vd, nl, cnt = runs[True]
        assert (a, b) == runs[False][:2] and np.array_equal(wd, runs[False][2]), name
        saved = runs[False][4] - nl
        assert cnt[SPMV] == 1, (name, cnt)
        tag = alg.tag
        if tag in (L.CGS, L.MGS, L.MGS2, L.MGSIR):
            assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT], saved) == (0, 0, 0, 0), (name, cnt, saved)
        elif tag == L.MGS2B:                       # no split band: fused, or the unfused pass
            want = (1, 0, 0, 1) if K1 <= fused_max else (0, nch, nch, 0)
            assert (cnt[SWEEP], cnt[PROJECT], cnt[UNPROJECT], saved) == want, (name, cnt, saved)
        elif K1 <= fused_max:                      # fused: one cooperative launch instead of two per sweep
            assert cnt[SWEEP] >= 1 and cnt[PROJECT] == cnt[UNPROJECT] == 0 and saved == cnt[SWEEP], (name, cnt, saved)
        elif K1 <= per_pass:                       # split sweeps: one launch per sweep either way
            assert cnt[SWEEP] >= 1 and cnt[PROJECT] == cnt[UNPROJECT] == 0 and saved == 0, (name, cnt, saved)
        else:                                      # unfused: nch project and unproject launches per pass
            assert cnt[SWEEP] == 0 and cnt[PROJECT] == cnt[UNPROJECT] and cnt[PROJECT] % nch == 0, (name, cnt)
            assert cnt[PROJECT] >= nch and saved == 0, (name, cnt, saved)
        if tag == L.CGS2:
            assert cnt[SWEEP] + cnt[PROJECT] // nch == 1, (name, cnt)
        v64 = vd.astype(f64)                       # r / beta_old as the device rounded it
        ow, oa, ob = ko.lanczos_recurrence(A, Vrows + [v64], beta_old, oracle_orth(alg) if tag != L.MGS2B
                                           else ko.Orth(ko.MGS2))
        s = float(np.linalg.norm(A @ v64)) + beta_old
        if dtype == f64:
            # one step from identical inputs: no accumulated drift
            ta = tw = 1e-13 * s
        else:
            # the SpMV (5 products a row, |A| <= 8) is below the Gram-Schmidt bound of gs_tols for two passes of |w| <= s
            ta, tw = gs_tols(n, K1, u, s, 2)
        assert abs(a - oa) <= ta and abs(b - ob) <= ta, (name, a, oa, b, ob, ta)
        assert np.linalg.norm(wd.astype(f64) - ow) <= tw, (name, np.linalg.norm(wd.astype(f64) - ow), tw)
    ctx.close()


# ------------------------------------------------------------------------------------------ 3. chained batches -----

def run_batch(chain, dtype, nsteps, orth, nx=97, ny=61):
    """initialize + one b2k_lanczos_expand_many batch of nsteps steps; (alphas, betas, V, r, launches of the batch)"""
    lib = L.load()
    lib.b2k_debug_set_chain(1 if chain else 0)
    try:
        n = nx * ny
        ctx = kk.B200Context(n, nsteps + 8, dtype=dtype)
        op = kk.B200CSR.stencil(ctx, nx, ny)
        x0 = ctx.from_host(ko.splitmix_vector(SEED, n, dtype=dtype))
        it = lz.LanczosIterator(op, x0, orth)
        used = lambda: lib.b2k_debug_used_columns(ctx.h, 0)
        f = lz.initialize(it)
        assert used() == 3
        l0 = ctx.launches
        done = lz.expand_many_(it, f, nsteps, 0.0)
        nl = ctx.launches - l0
        # x0, the basis, the residual — and nothing else
        assert done == nsteps and used() == 1 + len(f.V) + 1, (done, used(), len(f.V))
        out = (np.array(f.alphas), np.array(f.betas), np.column_stack([v.to_host() for v in f.V]).astype(f64),
               f.r.to_host().astype(f64), nl)
        del f, it, x0
        gc.collect()
        assert used() == 0
        ctx.close()
        return out
    finally:
        lib.b2k_debug_set_chain(1)


CHAIN_CASES = [(f64, 96), (f64, 97), (f32, 192), (f32, 193)]


@pytest.mark.parametrize("orth", [kk.cgs2, kk.mgs2b], ids=["cgs2", "mgs2b"])
@pytest.mark.parametrize("dtype,K1", CHAIN_CASES, ids=[f"{np.dtype(d).name}-K{K1}" for d, K1 in CHAIN_CASES])
def test_chained_batch_at_the_chain_limit(dtype, K1, orth):
    """b2k_lanczos_expand_many from k = 1 with k + nsteps = K1: at the limit the steps are chained on the device (two
    launches a step), one past it the batch is the loop of synchronous steps.  Either way the result is the one of the
    stepping loop: bit for bit for cgs2, to rounding for mgs2b (its synchronous alpha is a separate dot product)."""
    fused_max, _ = widths(dtype)
    nsteps = K1 - 1
    a1, b1, V1, r1, nl1 = run_batch(True, dtype, nsteps, orth)
    a0, b0, V0, r0, nl0 = run_batch(False, dtype, nsteps, orth)
    if K1 <= fused_max:
        assert nl1 <= 2 * nsteps + 2, nl1     # seed record (+ the first normalisation), then SpMV + sweep per step
    else:
        assert nl1 >= 3 * nsteps, nl1
    assert nl0 >= 3 * nsteps, nl0
    if orth is kk.cgs2:
        assert np.array_equal(a1, a0) and np.array_equal(b1, b0)
        assert np.array_equal(V1, V0) and np.array_equal(r1, r0)
    else:
        # rounding differences of one dot product per step, carried through at most K1 steps
        n = V1.shape[0]
        tol = K1 * LAM * math.sqrt(n) * unit(dtype)
        np.testing.assert_allclose(a1, a0, rtol=tol, atol=tol)
        np.testing.assert_allclose(b1, b0, rtol=tol, atol=tol)
        np.testing.assert_allclose(V1, V0, atol=tol)
    n = V1.shape[0]
    assert np.abs(V1.T @ V1 - np.eye(V1.shape[1])).max() <= K1 * LAM * math.sqrt(n) * unit(dtype)


# ------------------------------------------------------------------------------------------ 4. wide krylovdim -----

@pytest.mark.parametrize("krylovdim", [130, 256])
@pytest.mark.parametrize("orth,oorth", [(kk.cgs2, ko.Orth(ko.CGS2)), (kk.mgs2, ko.Orth(ko.MGS2))], ids=["cgs2", "mgs2"])
def test_lanczos_eigsolve_wide_krylovdim(orth, oorth, krylovdim):
    """eigsolve with krylovdim past the fused and the one-pass widths, two restart cycles far from convergence: the
    Ritz values within 1e-10 relative of the oracle's, same numops."""
    nx, ny = 60, 50
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(SEED, n)
    ctx = kk.B200Context(n, krylovdim + 24)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    alg = kk.Lanczos(orth=orth, krylovdim=krylovdim, maxiter=2, tol=1e-14, verbosity=0)
    with profiled(ctx) as cnt:
        vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0), 4, "SR", alg)
    ovals, _, oinfo = ko.eigsolve_lanczos(A, x0, 4, "SR", krylovdim=krylovdim, maxiter=2, tol=1e-14, orth=oorth)
    assert info.numiter == oinfo["numiter"] == 2 and info.numops == oinfo["numops"]
    np.testing.assert_allclose(vals[:4], ovals[:4], rtol=1e-10)
    assert cnt[TRANSFORM] >= 1                          # the restart transformed a basis of krylovdim vectors
    if orth is kk.cgs2:
        assert cnt[PROJECT] > 0 and cnt[PROJECT] == cnt[UNPROJECT]     # steps past K1 = 128 ran the unfused passes
    ctx.close()


def test_lanczos_eigsolve_krylovdim_257_is_refused_at_the_first_restart():
    """The restart's basis transform supports at most 256 vectors: krylovdim = 257 builds the factorization and then
    raises B200Error (not a CUDA error, not a wrong answer); the context stays usable."""
    nx, ny = 60, 50
    n = nx * ny
    ctx = kk.B200Context(n, 257 + 24)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=257, maxiter=2, tol=1e-14, verbosity=0)
    with profiled(ctx) as cnt:
        with pytest.raises(kk.B200Error, match="supported basis width"):
            kk.eigsolve(op, ctx.from_host(ko.splitmix_vector(SEED, n)), 4, "SR", alg)
    assert cnt[SPMV] >= 257 and cnt[PROJECT] > 0 and cnt[TRANSFORM] == 0
    xh = ko.splitmix_vector(SEED + 1, n)
    y = kk.apply(op, ctx.from_host(xh)).to_host()
    assert np.abs(y - ko.stencil_matrix(nx, ny) @ xh).max() <= 1e-14
    ctx.close()


def nearly_normal(n):
    """nonsymmetric, eigenvalues well conditioned: diag(1..10) plus a small random part"""
    return (sp.diags(np.linspace(1.0, 10.0, n)) + 0.01 * sp.random(n, n, density=5.0 / n, random_state=3)).tocsr()


def test_arnoldi_schursolve_wide_krylovdim():
    n = 4800
    A = nearly_normal(n)
    x0 = ko.splitmix_vector(SEED, n)
    ctx = kk.B200Context(n, 130 + 40)
    op = kk.B200CSR.from_scipy(ctx, A)
    alg = kk.Arnoldi(orth=kk.cgs2, krylovdim=130, maxiter=2, tol=1e-14, verbosity=0)
    with profiled(ctx) as cnt:
        T, Q, vals, info = kk.schursolve(op, ctx.from_host(x0), 4, "LR", alg)
    oT, _, ovals, oinfo = ko.schursolve_arnoldi(A, x0, 4, "LR", krylovdim=130, maxiter=2, tol=1e-14,
                                                orth=ko.Orth(ko.CGS2))
    assert info.numiter == oinfo["numiter"] == 2 and info.numops == oinfo["numops"]
    np.testing.assert_allclose(vals[:4], ovals[:4], rtol=1e-10)
    assert cnt[PROJECT] > 0 and cnt[TRANSFORM] >= 1
    ctx.close()


@pytest.mark.parametrize("orth,oorth", [(kk.cgs2, ko.Orth(ko.CGS2)), (kk.mgs2, ko.Orth(ko.MGS2))], ids=["cgs2", "mgs2"])
def test_gmres_wide_krylovdim(orth, oorth):
    nx, ny = 80, 50
    n = nx * ny
    A = ko.stencil_matrix(nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0, 0))
    b = A @ np.ones(n)
    ctx = kk.B200Context(n, 130 + 24)
    op = kk.B200CSR.from_scipy(ctx, A)
    alg = kk.GMRES(orth=orth, krylovdim=130, maxiter=2, tol=1e-14, verbosity=0)
    with profiled(ctx) as cnt:
        x, info = kk.linsolve(op, ctx.from_host(b), None, alg)
    ox, oinfo = ko.linsolve_gmres(A, b, None, krylovdim=130, maxiter=2, tol=1e-14, orth=oorth)
    assert info.numiter == oinfo["numiter"] and info.numops == oinfo["numops"] and info.numops > 129
    xh = x.to_host()
    np.testing.assert_allclose(A @ xh + info.residual.to_host(), b, atol=1e-10)
    np.testing.assert_allclose(info.normres, oinfo["normres"], rtol=1e-6, atol=1e-13)
    np.testing.assert_allclose(xh, ox, rtol=1e-8, atol=1e-10)
    if orth is kk.cgs2:
        assert cnt[PROJECT] > 0          # steps past K = 128 ran the unfused passes (the solution update unprojects too)
    ctx.close()


# ------------------------------------------------------------------------------------------ 5. SpMV contract -------

@pytest.fixture(params=[(1, 1), (1, 0), (0, 1)], ids=["pipe-2x4", "pipe-3x3", "stream"])
def spmv_kernel(request):
    """the TMA-pipelined SpMV in its two stage/occupancy variants and the plain streaming kernel"""
    lib = L.load()
    lib.b2k_debug_set_spmv_pipe(request.param[0])
    lib.b2k_debug_set_spmv_variant(request.param[1])
    yield request.param[0]
    lib.b2k_debug_set_spmv_pipe(1)
    lib.b2k_debug_set_spmv_variant(1)


def csr_in_order(A, x, dtype):
    """y_i = (((0 + p_0) + p_1) + ...) + p_last with p_j = a_ij x_j rounded in `dtype`, nonzeros in CSR order, each
    addition an elementwise numpy add in `dtype`.  Returns (y, row lengths, sum_j |p_j| in float64)."""
    A = A.tocsr()
    A.sort_indices()
    prod = A.data.astype(dtype) * x.astype(dtype)[A.indices]
    lens = np.diff(A.indptr)
    y = np.zeros(A.shape[0], dtype=dtype)
    for t in range(int(lens.max(initial=0))):
        rows = np.nonzero(lens > t)[0]
        y[rows] = y[rows] + prod[A.indptr[rows] + t]
    absum = np.zeros(A.shape[0])
    np.add.at(absum, np.repeat(np.arange(A.shape[0]), lens), np.abs(prod.astype(f64)))
    return y, lens, absum


_EDGE = {}


def edge_matrix():
    """rows of exactly 1536 and 1537 nonzeros and one of 3000; runs of 1025 and 2049 empty rows (past the staged
    rowptr segment of the pipelined kernel and past the rows of one tile); 0-8 nonzeros elsewhere"""
    if "A" not in _EDGE:
        n = 9000
        rng = np.random.default_rng(1536)
        lens = rng.integers(0, 9, size=n)
        lens[5], lens[6], lens[7] = SP_NNZ, SP_NNZ + 1, 3000
        lens[100:100 + 1025] = 0
        lens[4000:4000 + 2049] = 0
        cols = [np.sort(rng.choice(n, size=m, replace=False)) for m in lens]
        indptr = np.concatenate([[0], np.cumsum(lens)])
        _EDGE["A"] = sp.csr_matrix((rng.standard_normal(indptr[-1]), np.concatenate(cols), indptr), shape=(n, n))
    return _EDGE["A"]


def check_spmv_contract(ctx, op, A, dtype, seed):
    """apply, shifted apply and the fused dot of one operator against csr_in_order"""
    n = A.shape[0]
    u = unit(dtype)
    rng = np.random.default_rng(seed)
    xh = rng.standard_normal(n).astype(dtype)
    vh = rng.standard_normal(n).astype(dtype)
    x, v = ctx.from_host(xh), ctx.from_host(vh)
    ref, lens, absum = csr_in_order(A, xh, dtype)
    short = lens <= SP_NNZ
    with profiled(ctx) as cnt:
        y = kk.apply(op, x).to_host()
    assert cnt[SPMV] == 1
    bad = np.nonzero(short & (y != ref))[0]
    assert bad.size == 0, f"{bad.size} rows of <= {SP_NNZ} nonzeros differ, e.g. rows {bad[:8]} (lengths {lens[bad[:8]]})"
    # a long row: the same rounded products in another order (double partial sums, one rounding at the end)
    rowb = np.where(short, 0.0, lens * u * absum)
    assert np.all(np.abs(y.astype(f64) - ref.astype(f64)) <= rowb)
    # shifted: fma(a0, x, a1 * s) with a0, a1 rounded to the vector type — two roundings on top of the row error, two
    # more in the float64 reference
    a0, a1 = dtype(0.3), dtype(-1.5)
    x64, r64 = xh.astype(f64), ref.astype(f64)
    ysh = kk.apply(op, x, 0.3, -1.5).to_host().astype(f64)
    want = float(a1) * r64 + float(a0) * x64
    assert np.all(np.abs(ysh - want) <= 4 * u * (abs(float(a1)) * np.abs(r64) + abs(float(a0)) * np.abs(x64))
                  + abs(float(a1)) * rowb * (1 + 2 * u))
    # fused <v, A x>: n products accumulated (plus the row errors weighted by |v|)
    y2 = ctx.empty()
    d = op.apply_dot_into(y2, x, v)
    assert np.array_equal(y2.to_host(), y)
    v64 = vh.astype(f64)
    dref = math.fsum(v64 * r64)
    assert abs(d - dref) <= 2 * LAM * math.sqrt(n) * u * float(np.abs(v64 * r64).sum()) + float(np.abs(v64) @ rowb)


STENCILS = [(100, 100), (125, 80), (1, 7), (2048, 3), (37, 1), (1000, 700)]


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("matrix", ["edges", "n1"] + [f"stencil{nx}x{ny}" for nx, ny in STENCILS])
def test_spmv_rounds_products_and_sums_in_csr_order(matrix, dtype, spmv_kernel):
    """spmv.cu's contract: products rounded in the vector type and each row summed in CSR order — every row of at most
    1536 nonzeros bit-identical to the host restatement, longer rows within nnz u sum|a_ij x_j|."""
    if matrix == "edges":
        A = edge_matrix()
        assert {SP_NNZ, SP_NNZ + 1, 3000} <= set(np.diff(A.indptr).tolist())
    elif matrix == "n1":
        A = sp.csr_matrix(np.array([[1.7]]))
    else:
        nx, ny = (int(s) for s in matrix[len("stencil"):].split("x"))
        A = None
    n = A.shape[0] if A is not None else nx * ny
    ctx = kk.B200Context(n, 8, dtype=dtype)
    if A is None:
        ops = [kk.B200CSR.stencil(ctx, nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0))]
        A = ops[0].to_scipy()[:, :n]               # the device-assembled matrix, as stored
        ops.append(kk.B200CSR.from_scipy(ctx, A))
    else:
        ops = [kk.B200CSR.from_scipy(ctx, A)]
        A = sp.csr_matrix(A.astype(dtype))
    for i, op in enumerate(ops):
        check_spmv_contract(ctx, op, A, dtype, n + i)
    ctx.close()


# ------------------------------------------------------------------------------------------ 6. SpMM ----------------

@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("p", [2, 7, 8, 9, 16, 17])
def test_spmm_equals_single_applies_on_long_rows(p, dtype):
    """b2k_op_apply_block (one pass over the matrix per 8 vectors) is bit-identical to p calls of apply, long rows
    included: both round every product before it is added."""
    A = edge_matrix()
    n = A.shape[0]
    rng = np.random.default_rng(p)
    ctx = kk.B200Context(n, 2 * p + 6, dtype=dtype)
    op = kk.B200CSR.from_scipy(ctx, A)
    X = [ctx.from_host(rng.standard_normal(n)) for _ in range(p)]
    Y = [ctx.empty() for _ in range(p)]
    with profiled(ctx) as cnt:
        ctx.check(ctx.lib.b2k_op_apply_block(ctx.h, op.h, handles(X), handles(Y), p))
    assert cnt[SPMM] == -(-p // 8) and cnt[SPMV] == 0, cnt
    lens = np.diff(A.indptr)
    for i in range(p):
        bad = np.nonzero(Y[i].to_host() != kk.apply(op, X[i]).to_host())[0]
        assert bad.size == 0, f"vector {i}: rows {bad[:8]} (lengths {lens[bad[:8]]}) differ from the single apply"
    ctx.close()


# ------------------------------------------------------------------------------------------ 7. Float32 and dense ---

@pytest.mark.parametrize("grid,coeffs", [((97, 61, 1), (4.0, -1.0, -1.0, -1.0, -1.0, 0.0, 0.0)),
                                          ((64, 50, 1), (4.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0)),
                                          ((23, 17, 13), (6.0, -1.0, -1.1, -0.9, -1.0, -1.2, -0.8))])
def test_float32_stencils_match_each_other_and_the_restatement(grid, coeffs):
    """Float32: the assembled stencil and the matrix-free one give the same bits for apply and shifted apply, both equal
    to the CSR-order restatement of the assembled matrix."""
    nx, ny, nz = grid
    n = nx * ny * nz
    ctx = kk.B200Context(n, 16, dtype=f32)
    Aop = kk.B200CSR.stencil(ctx, nx, ny, nz, coeffs)
    Fop = kk.B200CSR.stencil_free(ctx, nx, ny, nz, coeffs)
    A = Aop.to_scipy()[:, :n]
    check_spmv_contract(ctx, Aop, A, f32, 5)
    check_spmv_contract(ctx, Fop, A, f32, 5)
    rng = np.random.default_rng(6)
    x = ctx.from_host(rng.standard_normal(n))
    assert np.array_equal(kk.apply(Fop, x).to_host(), kk.apply(Aop, x).to_host())
    assert np.array_equal(kk.apply(Fop, x, 0.3, 1.7).to_host(), kk.apply(Aop, x, 0.3, 1.7).to_host())
    ctx.close()


def test_float32_cg_chain_equals_stepwise():
    """b2k_cg_chain in a Float32 context: same numiter / numops / converged and the same x, bit for bit, as one
    b2k_cg_step per iteration."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    nx, ny = 181, 97
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    b = (A @ np.ones(n) + 0.01 * ko.splitmix_vector(3, n)).astype(f32)
    nb = float(np.linalg.norm(b.astype(f64)))
    ctx = kk.B200Context(n, 16, dtype=f32)
    op = kk.B200CSR.from_scipy(ctx, A)
    out = {}
    try:
        for chain in (True, False):
            ls.USE_CG_CHAIN = chain
            res = []
            for alg in (kk.CG(maxiter=2000, tol=1e-4 * nb, verbosity=0), kk.CG(maxiter=45, tol=1e-300, verbosity=0)):
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


def test_float32_bicgstab_chain_equals_stepwise():
    """b2k_bicgstab_chain in a Float32 context against b2k_bicgstab_half/_full called in turn: same numiter / numops /
    converged, the same x bit for bit, for converging runs and a fixed iteration budget."""
    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    rng = np.random.default_rng(5)
    n = 6000
    A = (sp.diags([-1.3, 2.6, -0.7], [-1, 0, 1], shape=(n, n)) +
         sp.random(n, n, density=1e-3, random_state=4) * 0.05).tocsr()
    b = rng.random(n).astype(f32)
    nb = float(np.linalg.norm(b.astype(f64)))
    ctx = kk.B200Context(n, 20, dtype=f32)
    op = kk.B200CSR.from_scipy(ctx, A)
    algs = [kk.BiCGStab(maxiter=4 * n, tol=1e-4 * nb, verbosity=0), kk.BiCGStab(maxiter=37, tol=1e-300, verbosity=0),
            kk.BiCGStab(maxiter=4 * n, tol=3e-3 * nb, verbosity=0), kk.BiCGStab(maxiter=4 * n, tol=1e-3 * nb, verbosity=0)]
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
    ctx.close()


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("m", [31, 33, 20011])
@pytest.mark.parametrize("ncols", [1, 127, 128, 129, 300])
def test_dense_gemv_at_the_chunk_edges(ncols, m, dtype):
    """apply_normal (y = A x: the unproject passes, 128 / 256 columns each) and apply_adjoint (z = A' u: the project
    passes) of a dense column-major m x ncols operator, against float64 products."""
    u = unit(dtype)
    rng = np.random.default_rng(m + ncols)
    ctx = kk.B200Context(m, 8, dtype=dtype)
    sv = ctx.add_space(ncols, 8, sharded=False)
    A = (rng.random((m, ncols)) - 0.5).astype(dtype)
    op = kk.B200Dense.from_host(ctx, A, sv)
    xh = rng.standard_normal(ncols).astype(dtype)
    uh = rng.standard_normal(m).astype(dtype)
    A64, x64, u64 = A.astype(f64), xh.astype(f64), uh.astype(f64)
    nch = -(-ncols // widths(dtype)[1])
    with profiled(ctx) as cnt:
        y = kk.apply_normal(op, ctx.from_host(xh, sv)).to_host().astype(f64)
    assert cnt[UNPROJECT] == nch and cnt[PROJECT] == 0
    # row i: ncols fused multiply-adds in the vector type
    assert np.all(np.abs(y - A64 @ x64) <= 2 * LAM * math.sqrt(ncols + 1) * u * (np.abs(A64) @ np.abs(x64)))
    with profiled(ctx) as cnt:
        z = kk.apply_adjoint(op, ctx.from_host(uh)).to_host().astype(f64)
    assert cnt[PROJECT] == nch and cnt[UNPROJECT] == 0
    # column j: m products summed
    assert np.all(np.abs(z - A64.T @ u64) <= 2 * LAM * math.sqrt(m) * u * (np.abs(A64).T @ np.abs(u64)))
    ctx.close()
