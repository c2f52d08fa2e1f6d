"""GPU tests of the BLAS-1 and short-recurrence kernels of blas1.cu against exact host restatements, in Float64 and
Float32: fill, scale, axpby (all three modes and the aliased add!!(y, y, α, β)), axpy2, Givens, rank1update! and the
Householder reflection, inner / norm, the single-vector orthogonalize!!, and the fused CG and BiCGStab iterations with
their device chains.

Rounding contracts.  Every elementwise kernel gives the bits of the literal VectorInterface calls it stands for, with
the scalars cast to the vector type T first:
  scale!!(y, x, α) = rn(α·x);  add!!(y, x, α, 0) = rn(α·x) (y never read);  add!!(y, x, α, 1) = fma(α, x, y);
  add!!(y, x, α, β) = fma(α, x, rn(β·y)), also when x is y;  axpy2 = two add!!(·, ·, a, 1) in turn;
  rmul!(b, Givens(c, s)) = (add(q1, q2, -s, c), add!!(q2, q1, s, c)) = (fma(-s, q2, rn(c·q1)), fma(s, q1, rn(c·q2))).
The host restates them with numpy arithmetic in float32 / float64 (correctly rounded per operation) and with libm's
fma / fmaf through a small C helper built by the module fixture (Python and numpy have no fused multiply-add), and
compares with array_equal.  A SpMV output inside a fused step is compared with a separate kk.apply of the same input,
whose own contract test_gpu_paths.py pins.

Launch geometry (blas1.cu): grid_for(n, 8) = min(ceil(n / 2048), 4·SMs) CTAs of 256 threads; a thread visits its
128-bit vectors (V = 2 doubles or 4 floats) in trips of 4 vectors (2 in k_cg_xr and k_bicg_xr); the n % V tail goes to
threads 0..V-2 of CTA 0.  The sizes below cover the empty vector, every tail length, one and a few CTAs, a grid exactly
at the cap ("cap") and a grid at the cap where every thread runs several trips and the tail is nonempty ("trips").

Tolerances.  u is the unit roundoff of T (2^-53 / 2^-24).  A sum of m rounded terms may be off by
LAM·sqrt(m)·u·sum(|terms|), the probabilistic bound of Higham & Mary (SIAM J. Sci. Comput. 41(5), 2019), violated with
probability below 2m·exp(-LAM²/2).  The reductions are two-stage: each thread accumulates its m_t terms in T with fma,
then the per-thread values are summed in double (block sums, then the CTA partials in CTA order); the double stage adds
at most LAM·sqrt(#threads)·2^-53·sum(|terms|).  Integer data in [-8, 8] keeps every partial sum exact in both stages
(per thread well below 2^24), so there the device must give the exact sum bit for bit.
"""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.vectors import handles
from oracle import krylov_oracle as ko
from test_gpu_paths import LAM, SPMV, profiled, unit

SEED = 20260923
f64, f32 = np.float64, np.float32
DTYPES = [f64, f32]
BT, CTAS_PER_SM, UNROLL = 256, 4, 8          # threads per CTA, CTA cap per SM, grid_for(n, 8)
VEC = {f64: 2, f32: 4}
MAX_CHAIN = 512                               # B2K_MAX_CHAIN
SIZES = [0, 1, 2, 3, 4, 5, 7, 255, 256, 257, "cap", "trips"]

_FMA_C = r"""
#include <math.h>
#include <stddef.h>
void vfma_f64(size_t n, const double* a, const double* b, const double* c, double* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fma(a[i], b[i], c[i]);
}
void vfma_f32(size_t n, const float* a, const float* b, const float* c, float* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fmaf(a[i], b[i], c[i]);
}
"""


@pytest.fixture(scope="module")
def fma(tmp_path_factory):
    """fma(a, b, c, T): the correctly rounded a·b + c elementwise in T (arguments broadcast, cast to T first)"""
    d = tmp_path_factory.mktemp("vfma")
    src, so = d / "vfma.c", str(d / "libvfma.so")
    src.write_text(_FMA_C)
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, str(src), "-lm"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)

    def f(a, b, c, dt):
        a, b, c = (np.ascontiguousarray(t, dtype=dt) for t in np.broadcast_arrays(
            np.asarray(a, dtype=dt), np.asarray(b, dtype=dt), np.asarray(c, dtype=dt)))
        out = np.empty(a.shape, dtype=dt)
        fn = lib.vfma_f64 if dt == f64 else lib.vfma_f32
        fn(C.c_size_t(out.size), C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), C.c_void_p(c.ctypes.data),
           C.c_void_p(out.ctypes.data))
        return out
    return f


_NSM = []


def num_sms():
    if not _NSM:
        import torch
        _NSM.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _NSM[0]


def cap_ctas():
    return CTAS_PER_SM * num_sms()


def size_of(name):
    """'cap': grid_for(n, 8) exactly at 4·SMs CTAs, tail empty.  'trips': at the cap with 5x the elements (f64: 20
    vectors = 5 trips per thread, f32: 10 vectors = 2-3 trips), odd, n % 4 == 1: a tail in both types."""
    if name == "cap":
        return UNROLL * BT * cap_ctas()
    if name == "trips":
        return 5 * UNROLL * BT * cap_ctas() + 12345
    return name


def grid_for(n, per_thread=UNROLL):
    return max(1, min(-(-n // (BT * per_thread)), cap_ctas()))


def per_thread_terms(n, dt):
    """most terms one thread of a grid_for(n, 8) reduction accumulates: its grid-strided vectors, plus one tail
    element for thread 0 (the trip length does not change which vectors a thread visits)"""
    threads = grid_for(n) * BT
    return -(-(n // VEC[dt]) // threads) * VEC[dt] + 1


@pytest.fixture(scope="module")
def ctxs():
    """one context per (type, length), reused by the tests of the module; length 0 is a space of a small context"""
    made = {}

    def get(dt, n):
        key = (np.dtype(dt).name, n)
        if key not in made:
            if n == 0:
                c = kk.B200Context(8, 4, dtype=dt)
                made[key] = (c, c.add_space(0, 16))
            else:
                made[key] = (kk.B200Context(n, 16, dtype=dt), 0)
        return made[key]
    yield get
    for c, _ in made.values():
        c.close()


def rand(rng, n, dt, scale=1.0):
    return (scale * rng.standard_normal(n)).astype(dt)


def ids(xs):
    return [str(x) for x in xs]


# ------------------------------------------------------------------------------------------ 1. elementwise ---------

@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_fill_and_splitmix(dt, size, ctxs):
    n = size_of(size)
    ctx, spc = ctxs(dt, n)
    v = ctx.splitmix(SEED, spc)
    assert np.array_equal(v.to_host(), ko.splitmix_vector(SEED, n).astype(dt))
    w = ctx.full(0.1, spc)
    assert np.array_equal(w.to_host(), np.full(n, dt(0.1)))


def elementwise_case(dt, size, ctxs):
    """(n, context, space, x, y, z): three random vectors of T at one of SIZES"""
    n = size_of(size)
    ctx, spc = ctxs(dt, n)
    rng = np.random.default_rng(n + 7)
    return n, ctx, spc, rand(rng, n, dt), rand(rng, n, dt), rand(rng, n, dt)


@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_scale_axpby_axpy2_bitwise(dt, size, ctxs, fma):
    """scale, the three axpby modes and axpy2 against their rounding contracts; an empty vector launches nothing"""
    n, ctx, spc, xh, yh, zh = elementwise_case(dt, size, ctxs)
    x, z = ctx.from_host(xh, spc), ctx.from_host(zh, spc)
    al, be = 0.7071, -1.37
    a, b = dt(al), dt(be)
    l0 = ctx.launches
    # scale!!
    assert np.array_equal(x.scale(al).to_host(), a * xh)
    # beta = 0: y holds NaN and +-Inf and is never read
    bad = np.full(n, np.nan, dtype=dt)
    bad[1::3], bad[2::3] = np.inf, -np.inf
    y = ctx.from_host(bad, spc)
    out = y.add_(x, al, 0.0).to_host()
    assert np.array_equal(out, a * xh) and not np.isnan(out).any()
    # beta = 1 and general beta
    y = ctx.from_host(yh, spc)
    assert np.array_equal(y.add_(x, al, 1.0).to_host(), fma(a, xh, yh, dt))
    y = ctx.from_host(yh, spc)
    assert np.array_equal(y.add_(x, al, be).to_host(), fma(a, xh, b * yh, dt))
    # axpy2 = add!!(add!!(y, x1, a1), x2, a2)
    a1, a2 = 0.3, -2.9
    y = ctx.from_host(yh, spc)
    ctx.check(ctx.lib.b2k_vec_axpy2(ctx.h, y.handle, x.handle, a1, z.handle, a2))
    assert np.array_equal(y.to_host(), fma(dt(a2), zh, fma(dt(a1), xh, yh, dt), dt))
    if n == 0:
        assert ctx.launches == l0            # an empty vector launches nothing


@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_aliased_axpby_equals_the_call_on_a_copy(dt, size, ctxs, fma):
    """add!!(y, y, α, β) in all three modes: the bits of add!!(y, copy(y), α, β), not those of rn((α + β)·y)"""
    n, ctx, spc, xh, yh, zh = elementwise_case(dt, size, ctxs)
    al = 0.7071
    a = dt(al)
    for beta in (0.0, 1.0, -1.37):
        lit = {0.0: a * yh, 1.0: fma(a, yh, yh, dt)}.get(beta, fma(a, yh, dt(beta) * yh, dt))
        y, w = ctx.from_host(yh, spc), ctx.from_host(yh, spc)
        assert np.array_equal(y.add_(w, al, beta).to_host(), lit)
        y = ctx.from_host(yh, spc)
        assert np.array_equal(y.add_(y, al, beta).to_host(), lit), f"add!!(y, y, {al}, {beta})"


@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_givens_rounds_like_add(dt, size, ctxs, fma):
    """rmul!(b, Givens(c, s)) = (add(q1, q2, -s, c), add!!(q2, q1, s, c)): against the restatement and against those
    two B200Vec calls on copies of the vectors; q1 == q2 is refused"""
    n, ctx, spc, xh, yh, zh = elementwise_case(dt, size, ctxs)
    c, s = math.cos(0.3), math.sin(0.3)
    ct, st = dt(c), dt(s)
    q1, q2 = ctx.from_host(xh, spc), ctx.from_host(yh, spc)
    ctx.check(ctx.lib.b2k_basis_givens(ctx.h, q1.handle, q2.handle, c, s))
    g1, g2 = fma(-st, yh, ct * xh, dt), fma(st, xh, ct * yh, dt)
    assert np.array_equal(q1.to_host(), g1), "Givens q1' != fma(-s, q2, rn(c*q1))"
    assert np.array_equal(q2.to_host(), g2), "Givens q2' != fma(s, q1, rn(c*q2))"
    p1, p2 = ctx.from_host(xh, spc), ctx.from_host(yh, spc)
    v1 = p1.add(p2, -s, c)
    v2 = p2.copy().add_(p1, s, c)
    assert np.array_equal(v1.to_host(), g1) and np.array_equal(v2.to_host(), g2)
    with pytest.raises(ValueError):
        ctx.check(ctx.lib.b2k_basis_givens(ctx.h, q1.handle, q1.handle, c, s))


@pytest.mark.parametrize("k", [1, 255, 256, 257, 513])
@pytest.mark.parametrize("beta", [0.0, 1.0, 0.7])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_rank1update_bitwise(dt, beta, k, fma):
    """rank1update!(b, y, x, α, β): column i <- β·col + T(α·x_i)·y, the coefficient formed in double; 256 columns per
    launch, so k = 257 and 513 run the later chunks"""
    n = 1031
    rng = np.random.default_rng(k)
    ctx = kk.B200Context(n, k + 4, dtype=dt)
    B = rng.standard_normal((k, n)).astype(dt)
    vecs = ctx.empty_range(k)
    for j, v in enumerate(vecs):
        v.upload(B[j])
    yh = rand(rng, n, dt)
    xs = rng.standard_normal(k)
    al = 0.37
    kk.rank1update_(kk.OrthonormalBasis(vecs), ctx.from_host(yh), xs, al, beta)
    for j, v in enumerate(vecs):
        cf = dt(al * xs[j])
        want = {0.0: cf * yh, 1.0: fma(cf, yh, B[j], dt)}.get(beta, fma(cf, yh, dt(beta) * B[j], dt))
        assert np.array_equal(v.to_host(), want), f"column {j}"
    ctx.close()


@pytest.mark.parametrize("k", [1, 7, 257])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_householder_is_a_rank1_update_of_its_work_vector(dt, k, fma):
    """b2k_basis_householder(cols, v, β, work): work = Σ v_i col_i, then col_i <- fma(T(-β·v_i), work, col_i).
    β = 0 returns before touching anything."""
    n = 1031
    rng = np.random.default_rng(k + 1)
    ctx = kk.B200Context(n, k + 4, dtype=dt)
    B = rng.standard_normal((k, n)).astype(dt)
    vecs = ctx.empty_range(k)
    for j, v in enumerate(vecs):
        v.upload(B[j])
    vv = rng.standard_normal(k)
    vv[0] = 1.0
    hs = handles(vecs)
    work = ctx.from_host(np.full(n, 5.0))
    ctx.check(ctx.lib.b2k_basis_householder(ctx.h, hs, k, vv.ctypes.data_as(C.POINTER(C.c_double)), 0.0, work.handle))
    assert all(np.array_equal(v.to_host(), B[j]) for j, v in enumerate(vecs))
    assert np.array_equal(work.to_host(), np.full(n, dt(5.0)))
    beta = 2.0 / (vv @ vv)
    ctx.check(ctx.lib.b2k_basis_householder(ctx.h, hs, k, vv.ctypes.data_as(C.POINTER(C.c_double)), beta,
                                            work.handle))
    W = work.to_host()
    # the work vector is the unprojection sum_i v_i col_i: k products per row in T
    B64 = B.astype(f64)
    ref = vv @ B64
    assert np.all(np.abs(W - ref) <= 2 * LAM * math.sqrt(k + 1) * unit(dt) * (np.abs(vv) @ np.abs(B64)) + 1e-300)
    for j, v in enumerate(vecs):
        assert np.array_equal(v.to_host(), fma(dt(-beta * vv[j]), W, B[j], dt)), f"column {j}"
    ctx.close()


# ------------------------------------------------------------------------------------------ 2. reductions ----------

@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_inner_and_norm_exact_on_integers(dt, size, ctxs):
    """integers in [-8, 8]: every partial sum is an integer far below 2^24 per thread and 2^53 overall, so inner and
    norm² are the exact sums"""
    n = size_of(size)
    ctx, spc = ctxs(dt, n)
    rng = np.random.default_rng(n + 3)
    xi, yi = rng.integers(-8, 9, n), rng.integers(-8, 9, n)
    x, y = ctx.from_host(xi.astype(dt), spc), ctx.from_host(yi.astype(dt), spc)
    assert x.inner(y) == float(np.dot(xi, yi))
    assert x.norm() == math.sqrt(float(np.dot(xi, xi)))
    if n == 0:
        assert x.inner(y) == 0.0 and x.norm() == 0.0


@pytest.mark.parametrize("size", SIZES, ids=ids(SIZES))
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_inner_is_symmetric_and_deterministic(dt, size, ctxs):
    """the products of <x, y> and <y, x> are the same fmas in the same order: equal bits; norm(x) = sqrt(inner(x, x));
    a repeated call (ticketed two-stage sum, no atomics on values) gives the same bits"""
    n = size_of(size)
    ctx, spc = ctxs(dt, n)
    rng = np.random.default_rng(n + 5)
    x, y = ctx.from_host(rand(rng, n, dt), spc), ctx.from_host(rand(rng, n, dt), spc)
    s = x.inner(y)
    assert s == y.inner(x) and s == x.inner(y)
    assert x.norm() == math.sqrt(x.inner(x)) and x.norm() == x.norm()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_reductions_within_the_two_stage_bound(dt, ctxs):
    """random data at the multi-trip size: |device - exact| <= (LAM sqrt(m_t) u + LAM sqrt(threads) 2^-53) sum|x_i y_i|
    with m_t the terms of the busiest thread"""
    n = size_of("trips")
    ctx, spc = ctxs(dt, n)
    rng = np.random.default_rng(11)
    xh, yh = rand(rng, n, dt), rand(rng, n, dt)
    x, y = ctx.from_host(xh, spc), ctx.from_host(yh, spc)
    x64, y64 = xh.astype(f64), yh.astype(f64)
    mt, thr = per_thread_terms(n, dt), grid_for(n) * BT
    assert mt >= (8 if dt == f64 else 16)      # several trips per thread
    rel = LAM * math.sqrt(mt) * unit(dt) + LAM * math.sqrt(thr) * 2.0 ** -53
    prods = x64 * y64                            # exact: products of floats fit a double, and of doubles err by u
    exact = math.fsum(prods)
    assert abs(x.inner(y) - exact) <= rel * float(np.abs(prods).sum()) * (1 + 4 * unit(f64))
    sq = math.fsum(x64 * x64)
    assert abs(x.norm() ** 2 - sq) <= 2 * rel * sq


# ------------------------------------------------------------------------------------------ 3. orthogonalize!! -----

def literal_orthogonalize(v, q, tag, eta, dt):
    """orthonormal.jl:458-489 through B200Vec calls: (s, ||v||, passes); v is updated in place"""
    if tag == L.MGS2B:
        tag = L.MGS2
    if tag in (L.CGS, L.MGS):
        s = q.inner(v)
        v.add_(q, -s)
        return s, v.norm(), 1
    if tag in (L.CGS2, L.MGS2):
        s = q.inner(v)
        v.add_(q, -s)
        s2 = q.inner(v)
        v.add_(q, -s2)
        return s + s2, v.norm(), 2
    eps = float(np.finfo(dt).eps)
    nold = v.norm()
    s = q.inner(v)
    v.add_(q, -s)
    nnew = v.norm()
    passes = 1
    while eps < nnew < eta * nold:
        nold = nnew
        s2 = q.inner(v)
        v.add_(q, -s2)
        s += s2
        nnew = v.norm()
        passes += 1
    return s, nnew, passes


TAGS = [L.CGS, L.MGS, L.CGS2, L.MGS2, L.CGSIR, L.MGSIR, L.MGS2B]
IR = (L.CGSIR, L.MGSIR)


@pytest.mark.parametrize("case", ["random", "near", "equal"])
@pytest.mark.parametrize("tag", TAGS, ids=["CGS", "MGS", "CGS2", "MGS2", "CGSIR", "MGSIR", "MGS2B"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_vec_orthogonalize_equals_the_literal_sequence(dt, tag, case):
    """b2k_vec_orthogonalize against inner / add!! / norm called in the reference's order: v, s and the norm bit for
    bit.  The IR loop (eta = 0.75) takes
      random: 1 pass (v is nearly orthogonal to q already, ||v'|| ~ ||v||);
      near:   v = q + d·w, |w| = 1 (d = 1e-9 in f64; 1e-4 in f32, where 1e-9 would sit at the rounding level of q):
              ||v'|| ~ d after pass 1, < eta ||v||, > eps: a second pass, after which ||v''|| ~ ||v'||: 2 passes;
      equal:  v = q with four entries 1/2 (<q, q> = 1 exactly): v' = 0 exactly, the eps exit after 1 pass.
    The pass count is read from the launches: one norm, then (inner, update, norm) per pass."""
    n = 4099
    eta = 0.75
    rng = np.random.default_rng(tag + 13)
    if case == "equal":
        qh = np.zeros(n)
        qh[[0, 255, 256, n - 1]] = 0.5
        vh = qh.copy()
    else:
        qh = rng.standard_normal(n)
        qh /= np.linalg.norm(qh)
        w = rng.standard_normal(n)
        vh = rng.standard_normal(n) if case == "random" else qh + (1e-9 if dt == f64 else 1e-4) * w / np.linalg.norm(w)
    ctx = kk.B200Context(n, 8, dtype=dt)
    q = ctx.from_host(qh)
    v, vl = ctx.from_host(vh), ctx.from_host(vh)
    s, nrm = C.c_double(), C.c_double()
    l0 = ctx.launches
    ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, v.handle, q.handle, tag, eta, C.byref(s), C.byref(nrm)))
    launches = ctx.launches - l0
    sl, nl, passes = literal_orthogonalize(vl, q, tag, eta, dt)
    assert np.array_equal(v.to_host(), vl.to_host())
    assert s.value == sl and nrm.value == nl, (s.value, sl, nrm.value, nl)
    if tag in IR:
        want = {"random": 1, "near": 2, "equal": 1}[case]
        assert passes == want and launches == 1 + 3 * passes, (passes, launches)
        if case == "equal":
            assert nl == 0.0
    else:
        assert launches == (3 if tag in (L.CGS, L.MGS) else 5), launches
    ctx.close()


def test_vec_orthogonalize_refusals():
    ctx = kk.B200Context(100, 6)
    other = ctx.add_space(50, 2)
    q, v, w = ctx.from_host(np.ones(100)), ctx.from_host(np.arange(100.0)), ctx.from_host(np.ones(50), other)
    s, nrm = C.c_double(), C.c_double()
    with pytest.raises(ValueError, match="v == q"):
        ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, q.handle, q.handle, L.CGS, 0.7, C.byref(s), C.byref(nrm)))
    with pytest.raises(ValueError, match="unknown orthogonalizer"):
        ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, v.handle, q.handle, 7, 0.7, C.byref(s), C.byref(nrm)))
    with pytest.raises(L.DimensionMismatch):
        ctx.check(ctx.lib.b2k_vec_orthogonalize(ctx.h, w.handle, q.handle, L.CGS, 0.7, C.byref(s), C.byref(nrm)))
    assert np.array_equal(v.to_host(), np.arange(100.0))     # a refused call leaves v alone
    ctx.close()


# ------------------------------------------------------------------------------------------ 4. CG ------------------

NX, NY = 61, 67                                  # n = 4087: n % 4 == 3, two CTAs, two trips of 2 vectors per thread
SHIFTS = [(0.0, 1.0), (0.3, 1.5)]


def cg_setup(dt, nx=NX, ny=NY, coeffs=(4.0, -1.0, -1.0, -1.0, -1.0, 0.0, 0.0)):
    n = nx * ny
    ctx = kk.B200Context(n, 16, dtype=dt)
    op = kk.B200CSR.from_scipy(ctx, ko.stencil_matrix(nx, ny, 1, coeffs))
    return ctx, op, n


def cg_step(ctx, op, vs, a0, a1, beta, rho):
    pq, nr = C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_cg_step(ctx.h, op.h, *(v.handle for v in vs), a0, a1, beta, rho, C.byref(pq), C.byref(nr)))
    return pq.value, nr.value


def dot_bound(dt, a, b):
    """|computed - exact| of an n-term sum of products in T"""
    return LAM * math.sqrt(a.size) * unit(dt) * float(np.abs(a.astype(f64) * b.astype(f64)).sum())


@pytest.mark.parametrize("shift", SHIFTS, ids=["plain", "shifted"])
@pytest.mark.parametrize("beta", [0.0, 1.0, 0.6])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_cg_step_bitwise(dt, beta, shift, fma):
    """one b2k_cg_step from a prepared (x, r, p, q): p' = rn(r + rn(β p)) (β = 0: p overwritten, NaN ignored),
    q' = apply(p'), α = T(ρ/<p',q'>), x' = fma(α, p', x), r' = fma(-α, q', r); <p',q'> and ||r'|| within the bound"""
    a0, a1 = shift
    ctx, op, n = cg_setup(dt)
    rng = np.random.default_rng(int(beta * 10) + 2)
    xh, rh, ph = rand(rng, n, dt), rand(rng, n, dt), rand(rng, n, dt)
    if beta == 0.0:
        ph[::5] = np.nan
    rho = float(np.dot(rh.astype(f64), rh.astype(f64)))
    x, r, p, q = (ctx.from_host(a) for a in (xh, rh, ph, np.zeros(n)))
    pq, nr = cg_step(ctx, op, (x, r, p, q), a0, a1, beta, rho)
    pn = rh if beta == 0.0 else rh + dt(beta) * ph
    assert np.array_equal(p.to_host(), pn)
    qn = kk.apply(op, ctx.from_host(pn), a0, a1).to_host()
    assert np.array_equal(q.to_host(), qn)
    assert abs(pq - math.fsum(pn.astype(f64) * qn.astype(f64))) <= dot_bound(dt, pn, qn)
    al = dt(rho / pq)
    assert np.array_equal(x.to_host(), fma(al, pn, xh, dt))
    rn = fma(-al, qn, rh, dt)
    assert np.array_equal(r.to_host(), rn)
    assert abs(nr ** 2 - math.fsum(rn.astype(f64) ** 2)) <= 2 * dot_bound(dt, rn, rn)
    ctx.close()


def cg_stepwise(ctx, op, vs, a0, a1, beta, rho, k):
    """k b2k_cg_step calls with the scalar recurrence of cg.jl:74-77 on the host; the per-step records and the
    snapshots of (x, r, p, q) after every step"""
    recs, snaps = [], []
    for _ in range(k):
        pq, nr = cg_step(ctx, op, vs, a0, a1, beta, rho)
        recs.append((pq, nr))
        snaps.append([v.to_host() for v in vs])
        rho_new = nr * nr
        beta, rho = rho_new / rho, rho_new
    return recs, snaps


def cg_chain(ctx, op, vs, a0, a1, beta, rho, tol, nsteps):
    m = max(1, min(nsteps, MAX_CHAIN))
    pqs, nrs, done = (C.c_double * m)(), (C.c_double * m)(), C.c_int32()
    ctx.check(ctx.lib.b2k_cg_chain(ctx.h, op.h, *(v.handle for v in vs), a0, a1, beta, rho, tol, nsteps, pqs, nrs,
                                   C.byref(done)))
    return [(pqs[i], nrs[i]) for i in range(done.value)], done.value


def cg_state(ctx, n, dt, seed):
    """a state after a first iteration: x, r, p random, q scratch; beta, rho as the host would pass them"""
    rng = np.random.default_rng(seed)
    hs = [rand(rng, n, dt) for _ in range(3)] + [np.zeros(n, dt)]
    rr = float(np.dot(hs[1].astype(f64), hs[1].astype(f64)))
    return hs, 0.8, rr


@pytest.mark.parametrize("shift", SHIFTS, ids=["plain", "shifted"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_cg_chain_equals_steps_and_stops_mid_batch(dt, shift):
    """b2k_cg_chain against b2k_cg_step calls: the same records and vectors bit for bit.  A tol between the k-th ||r||
    (a new minimum) and all earlier ones stops the chain after k + 1 iterations, leaving the vectors of step k + 1:
    the launches behind the flag did nothing."""
    a0, a1 = shift
    ctx, op, n = cg_setup(dt)
    hs, beta, rho = cg_state(ctx, n, dt, 4)
    vs = [ctx.from_host(h) for h in hs]
    recs, snaps = cg_stepwise(ctx, op, vs, a0, a1, beta, rho, 32)
    vs = [ctx.from_host(h) for h in hs]
    got, done = cg_chain(ctx, op, vs, a0, a1, beta, rho, 0.0, 32)
    assert done == 32 and got == recs
    assert all(np.array_equal(v.to_host(), h) for v, h in zip(vs, snaps[-1]))
    nrs = [nr for _, nr in recs]
    k = next(i for i in range(10, 31) if nrs[i] < min(nrs[:i]))
    tol = 0.5 * (nrs[k] + min(nrs[:k]))
    vs = [ctx.from_host(h) for h in hs]
    got, done = cg_chain(ctx, op, vs, a0, a1, beta, rho, tol, 32)
    assert done == k + 1 and got == recs[:k + 1]
    assert all(np.array_equal(v.to_host(), h) for v, h in zip(vs, snaps[k]))
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_cg_chain_clamps_to_512_and_refuses(dt):
    """nsteps = 600 runs B2K_MAX_CHAIN = 512 iterations (512 SpMVs), equal to 512 steps.  The 300 x 300 Laplacian
    (condition ~ 3.6e4) is far from converged after 512 iterations, so every record is finite and positive.  nsteps = 0
    is an argument error; a dense operator is not supported."""
    ctx, op, n = cg_setup(dt, 300, 300)
    hs, beta, rho = cg_state(ctx, n, dt, 6)
    vs = [ctx.from_host(h) for h in hs]
    with profiled(ctx) as cnt:
        got, done = cg_chain(ctx, op, vs, 0.0, 1.0, beta, rho, 0.0, 600)
    assert done == MAX_CHAIN and cnt[SPMV] == MAX_CHAIN
    assert all(math.isfinite(pq) and pq > 0 and math.isfinite(nr) and nr > 0 for pq, nr in got)
    assert got[-1][1] > 1e-6 * got[0][1]
    chained = [v.to_host() for v in vs]
    vs = [ctx.from_host(h) for h in hs]
    pq_nr = []
    b, r_ = beta, rho
    for _ in range(MAX_CHAIN):
        pq, nr = cg_step(ctx, op, vs, 0.0, 1.0, b, r_)
        pq_nr.append((pq, nr))
        b, r_ = nr * nr / r_, nr * nr
    assert pq_nr == got
    assert all(np.array_equal(v.to_host(), h) for v, h in zip(vs, chained))
    pqs, nrs, d = (C.c_double * 1)(), (C.c_double * 1)(), C.c_int32()
    with pytest.raises(ValueError):
        ctx.check(ctx.lib.b2k_cg_chain(ctx.h, op.h, *(v.handle for v in vs), 0.0, 1.0, beta, rho, 0.0, 0, pqs, nrs,
                                       C.byref(d)))
    ctx.close()
    m = 64
    ctx = kk.B200Context(m, 8, dtype=dt)
    sv = ctx.add_space(m, 4, sharded=False)
    dop = kk.B200Dense.from_host(ctx, np.eye(m) * 2.0, sv)
    vs = [ctx.from_host(np.ones(m)) for _ in range(4)]
    with pytest.raises(L.B200Error, match="not supported"):
        ctx.check(ctx.lib.b2k_cg_chain(ctx.h, dop.h, *(v.handle for v in vs), 0.0, 1.0, 0.5, 1.0, 0.0, 4, pqs, nrs,
                                       C.byref(d)))
    ctx.close()


# ------------------------------------------------------------------------------------------ 5. BiCGStab ------------

NONSYM = (4.0, -1.3, -0.7, -1.1, -0.9, 0.0, 0.0)
BICG_SHIFTS = [(0.0, 1.0), (0.2, 0.9)]


def bicg_half(ctx, op, rs, r, p, v, s, a0, a1, beta, omega, rho, first):
    sg, ns = C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_bicgstab_half(ctx.h, op.h, rs.handle, r.handle, p.handle, v.handle, s.handle, a0, a1, beta,
                                        omega, rho, int(first), C.byref(sg), C.byref(ns)))
    return sg.value, ns.value


def bicg_full(ctx, op, x, r, rs, p, s, t, a0, a1, alpha):
    om, nr, rn = C.c_double(), C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_bicgstab_full(ctx.h, op.h, x.handle, r.handle, rs.handle, p.handle, s.handle, t.handle,
                                        a0, a1, alpha, C.byref(om), C.byref(nr), C.byref(rn)))
    return om.value, nr.value, rn.value


@pytest.mark.parametrize("first", [1, 0])
@pytest.mark.parametrize("shift", BICG_SHIFTS, ids=["plain", "shifted"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_bicgstab_half_and_full_bitwise(dt, shift, first, fma):
    """b2k_bicgstab_half then _full against the restatement with the kernels' scalars:
      p' = r (first) or rn(r + rn(T(β)·fma(-T(ω), v, p))),  v' = apply(p'),  α = T(ρ/σ),  s' = fma(-α, v', r),
      t' = apply(s'),  ω' = T(<t',s'>/<t',t'>),  x' = fma(ω', s', fma(α, p', x)),  r' = fma(-ω', t', s');
    σ, ||s'||, ω', ||r'|| and <r~, r'> within their bounds; and the same vectors as the literal VectorInterface
    sequence of linsolve._bicgstab run with the same scalars"""
    a0, a1 = shift
    ctx, op, n = cg_setup(dt, coeffs=NONSYM)
    rng = np.random.default_rng(first + 21)
    rsh, rh, ph, vh, xh = (rand(rng, n, dt) for _ in range(5))
    beta, omega = 0.9, 0.45
    rho = float(np.dot(rsh.astype(f64), rh.astype(f64)))
    rs, r, p, v, s, x, t = (ctx.from_host(a) for a in (rsh, rh, ph, vh, np.zeros(n), xh, np.zeros(n)))
    sigma, ns = bicg_half(ctx, op, rs, r, p, v, s, a0, a1, beta, omega, rho, first)
    pn = rh if first else rh + dt(beta) * fma(-dt(omega), vh, ph, dt)
    assert np.array_equal(p.to_host(), pn)
    vn = kk.apply(op, ctx.from_host(pn), a0, a1).to_host()
    assert np.array_equal(v.to_host(), vn)
    assert abs(sigma - math.fsum(rsh.astype(f64) * vn.astype(f64))) <= dot_bound(dt, rsh, vn)
    alpha = rho / sigma
    sn = fma(-dt(alpha), vn, rh, dt)
    assert np.array_equal(s.to_host(), sn)
    assert abs(ns ** 2 - math.fsum(sn.astype(f64) ** 2)) <= 2 * dot_bound(dt, sn, sn)
    om, nr, rho_next = bicg_full(ctx, op, x, r, rs, p, s, t, a0, a1, alpha)
    tn = kk.apply(op, ctx.from_host(sn), a0, a1).to_host()
    assert np.array_equal(t.to_host(), tn)
    ts, tt = math.fsum(tn.astype(f64) * sn.astype(f64)), math.fsum(tn.astype(f64) ** 2)
    assert abs(om - ts / tt) <= (dot_bound(dt, tn, sn) / abs(ts) + dot_bound(dt, tn, tn) / tt) * abs(ts / tt) * 1.01
    w = dt(om)
    xn = fma(w, sn, fma(dt(alpha), pn, xh, dt), dt)
    rn = fma(-w, tn, sn, dt)
    assert np.array_equal(x.to_host(), xn)
    assert np.array_equal(r.to_host(), rn)
    assert abs(nr ** 2 - math.fsum(rn.astype(f64) ** 2)) <= 2 * dot_bound(dt, rn, rn)
    assert abs(rho_next - math.fsum(rsh.astype(f64) * rn.astype(f64))) <= dot_bound(dt, rsh, rn)
    # the literal sequence (USE_FUSED_BICGSTAB = False) with the same scalars, vector for vector
    r, x = ctx.from_host(rh), ctx.from_host(xh)
    if first:
        p = r.copy()
    else:
        p = ctx.from_host(ph).add_(ctx.from_host(vh), -omega)
        p = p.add_(r, 1.0, beta)
    v = kk.apply(op, p, a0, a1)
    s = ctx.zeros().scale_(1.0, r).add_(v, -alpha)
    xhalf = ctx.zeros().scale_(1.0, x).add_(p, alpha)
    t = kk.apply(op, s, a0, a1)
    x = x.scale_(1.0, xhalf).add_(s, om)
    r = r.scale_(1.0, s).add_(t, -om)
    for name, got, want in (("p", p, pn), ("v", v, vn), ("s", s, sn), ("t", t, tn), ("x", x, xn), ("r", r, rn)):
        assert np.array_equal(got.to_host(), want), name
    ctx.close()


def bicg_start(ctx, op, n, dt, a0, a1, seed):
    """vectors (x, r, rs, p, v, s, t) and scalars (rho, rho_old, alpha, omega) after a first iteration"""
    rng = np.random.default_rng(seed)
    bh = rng.random(n).astype(dt)
    x, r, rs = ctx.zeros(), ctx.from_host(bh), ctx.from_host(bh)
    p, v, s, t = ctx.zeros(), ctx.zeros(), ctx.zeros(), ctx.zeros()
    rho = rs.inner(r)
    sg, _ = bicg_half(ctx, op, rs, r, p, v, s, a0, a1, 0.0, 1.0, rho, 1)
    alpha = rho / sg
    om, _, rho_next = bicg_full(ctx, op, x, r, rs, p, s, t, a0, a1, alpha)
    return [w.to_host() for w in (x, r, rs, p, v, s, t)], (rho_next, rho, alpha, om)


def bicg_stepwise(ctx, op, vs, a0, a1, scal, k, tol=0.0, snap=True):
    """k iterations as b2k_bicgstab_half / _full calls with bicgstab.jl's scalar recurrences on the host.  Returns the
    8-double records of the chain and the vectors after each record (stop code 1: after the half step)."""
    x, r, rs, p, v, s, t = vs
    rho, rho_old, alpha, omega = scal
    recs, snaps = [], []
    for _ in range(k):
        beta = (rho / rho_old) * (alpha / omega)
        sg, ns = bicg_half(ctx, op, rs, r, p, v, s, a0, a1, beta, omega, rho, 0)
        alpha = rho / sg
        rec = [rho, sg, alpha, ns, 0.0, 0.0, 0.0, 0.0]
        if ns < tol:
            rec[7] = 1.0
        else:
            omega, nr, rho_next = bicg_full(ctx, op, x, r, rs, p, s, t, a0, a1, alpha)
            rec[4:7] = [omega, nr, rho_next]
            if nr < tol:
                rec[7] = 2.0
            rho_old, rho = rho, rho_next
        recs.append(rec)
        if snap:
            snaps.append([w.to_host() for w in vs])
        if rec[7]:
            break
    return recs, snaps


def bicg_chain(ctx, op, vs, a0, a1, scal, tol, nsteps):
    m = max(1, min(nsteps, MAX_CHAIN - 1))
    rec, done = np.zeros((m, 8)), C.c_int32()
    ctx.check(ctx.lib.b2k_bicgstab_chain(ctx.h, op.h, *(w.handle for w in vs), a0, a1, *scal, tol, nsteps,
                                         rec.ctypes.data_as(C.POINTER(C.c_double)), C.byref(done)))
    return rec[:done.value].tolist(), done.value


@pytest.mark.parametrize("shift", BICG_SHIFTS, ids=["plain", "shifted"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_bicgstab_chain_records_and_both_stops(dt, shift):
    """b2k_bicgstab_chain against half / full stepping: the 8-double records and all seven vectors bit for bit, for
    a run without a stop and for a tol that first undercuts ||s|| (stop code 1: x and r as the half step left them,
    the full step never ran) and one that first undercuts ||r|| (stop code 2).  tol sits halfway between a new minimum
    of the sequence ||s_1||, ||r_1||, ||s_2||, ... and the smallest value before it."""
    a0, a1 = shift
    ctx, op, n = cg_setup(dt, coeffs=NONSYM)
    hs, scal = bicg_start(ctx, op, n, dt, a0, a1, 8)
    K = 60
    vs = [ctx.from_host(h) for h in hs]
    recs, snaps = bicg_stepwise(ctx, op, vs, a0, a1, scal, K)
    vs = [ctx.from_host(h) for h in hs]
    got, done = bicg_chain(ctx, op, vs, a0, a1, scal, 0.0, K)
    assert done == K and got == recs
    assert all(np.array_equal(w.to_host(), h) for w, h in zip(vs, snaps[-1]))
    seq = [x for rec in recs for x in (rec[3], rec[5])]
    for code in (1, 2):
        j = next((j for j in range(4, len(seq)) if j % 2 == code - 1 and seq[j] < min(seq[:j])), None)
        assert j is not None, f"no new minimum of {'||s||' if code == 1 else '||r||'} in {K} iterations"
        tol = 0.5 * (seq[j] + min(seq[:j]))
        vs = [ctx.from_host(h) for h in hs]
        want, wsnaps = bicg_stepwise(ctx, op, vs, a0, a1, scal, K, tol)
        assert len(want) == j // 2 + 1 and want[-1][7] == code
        vs = [ctx.from_host(h) for h in hs]
        got, done = bicg_chain(ctx, op, vs, a0, a1, scal, tol, K)
        assert done == j // 2 + 1 and got == want
        assert all(np.array_equal(w.to_host(), h) for w, h in zip(vs, wsnaps[-1]))
        if code == 1:      # x and r are those of the previous full step
            assert np.array_equal(vs[0].to_host(), snaps[j // 2 - 1][0])
            assert np.array_equal(vs[1].to_host(), snaps[j // 2 - 1][1])
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_bicgstab_chain_clamps_to_511(dt):
    """nsteps = 600 runs B2K_MAX_CHAIN - 1 = 511 iterations (two SpMVs each), equal to 511 half / full steps.  On the
    500 x 500 nonsymmetric stencil (condition ~ 1e5) 511 iterations stay far from convergence: every record finite,
    no stop code."""
    ctx, op, n = cg_setup(dt, 500, 500, NONSYM)
    hs, scal = bicg_start(ctx, op, n, dt, 0.0, 1.0, 9)
    vs = [ctx.from_host(h) for h in hs]
    with profiled(ctx) as cnt:
        got, done = bicg_chain(ctx, op, vs, 0.0, 1.0, scal, 0.0, 600)
    assert done == MAX_CHAIN - 1 and cnt[SPMV] == 2 * (MAX_CHAIN - 1)
    assert np.isfinite(got).all() and not any(rec[7] for rec in got)
    assert got[-1][5] > 1e-6 * got[0][5]
    chained = [w.to_host() for w in vs]
    vs = [ctx.from_host(h) for h in hs]
    want, _ = bicg_stepwise(ctx, op, vs, 0.0, 1.0, scal, MAX_CHAIN - 1, snap=False)
    assert got == want
    assert all(np.array_equal(w.to_host(), h) for w, h in zip(vs, chained))
    ctx.close()
