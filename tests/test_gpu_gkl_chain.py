"""GPU tests of the device-chained GKL step, b2k_gkl_expand_many, in Float64 and Float32.

1. One chained step equals, bit for bit, a numpy restatement of its documented order (include/b200krylov.h, basis.cu):
     v~ = fma(-beta, v_{k-1}, A' (r * T(1/beta)))        the A' SpMV's epilogue (spmv_restate.csr_rows)
     alpha = sqrt of the fused norm of v~                 CGS2: the SpMV's CTA-ordered sum (spmv_restate.dot)
                                                          MGS2B: v~ -= V V' v~ first, alpha from the sweep's finaliser
     u = rn(r * T(1/beta)),  r' = fma(-alpha, u, A (v~ * T(1/alpha)))
     r'' = one classical pass of r' over [U, u], beta = sqrt(||r''||^2)    (tsk_restate.cgs)
     v = rn(v~ * T(1/alpha))                              the flush launch
   on every instance of the GK epilogue: k_spmv_pipe's variants (2, 4) and (3, 3) in both types, and k_spmv_compact's
   <double, float, int16>, <double, float, int32>, <double, double, int16> and <float, float, int16> under both
   variants (whose grids are 4 and 3 CTAs per SM).  b2k_debug_csr_format says which compact instance each of A and
   A' takes.  Shapes: a tall matrix whose transpose has rows longer than one tile (1536 nonzeros: the long-row path),
   a wide one, both with empty rows and columns; odd small ones; and one with at least 2.5 tiles per CTA on both
   sides, a long row on one and a run of more than 1024 empty rows (SPP_RMAX) on the other.
2. A batch of N steps equals N calls of one step bit for bit: alpha, beta and every U, V and r column (CGS2, MGS2B).
3. A stop in the middle of a batch (beta <= tol on a rank-3 matrix): steps_done, the columns and the released
   handles are those of stepping, and the launches behind the stop do nothing.  A +Inf in A stops the first step
   on its non-finite alpha, with beta reported as NaN.
4. Refused calls write nothing.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

import spmv_restate as R
import tsk_restate as TR
from test_gpu_csr_compact import INTS, banded

f64, f32 = np.float64, np.float32


KERNELS = {"pipe24": (0, 1), "pipe33": (0, 0), "compact1": (1, 1), "compact0": (1, 0)}   # (compact copy, variant)
F32V, I16, RP16 = 1, 2, 4                                  # b2k_debug_csr_format bits
INSTANCES = {"dfi16": RP16 | I16 | F32V, "dfi32": RP16 | F32V, "ddi16": RP16 | I16, "ffi16": RP16 | I16}
SP_NNZ = 1536


@contextlib.contextmanager
def kernel(name):
    """pipe24 / pipe33: the plain TMA kernel in variant 1 / 0 (compact copies off); compact1 / compact0: the compact
    copy where the operator has one, in variant 1 / 0"""
    lib = L.load()
    compact, variant = KERNELS[name]
    lib.b2k_debug_set_csr_compact(compact)
    lib.b2k_debug_set_spmv_variant(variant)
    try:
        yield
    finally:
        lib.b2k_debug_set_csr_compact(1)
        lib.b2k_debug_set_spmv_variant(1)


def compact_format(M, dt):
    """b2k_debug_csr_format as build_compact decides it: Float32 values (Float64 only) when every value round-trips
    through float and none is NaN, 16-bit column offsets when every tile of <= SP_NNZ nonzeros keeps col - its first
    row within int16, 16-bit row pointers with either"""
    rb = R.tiles(M.indptr)
    vals = np.asarray(M.data, dtype=dt)
    f32v = dt == f64 and not np.isnan(vals).any() and np.array_equal(vals.astype(np.float32).astype(f64), vals)
    i16 = True
    for b in range(len(rb) - 1):
        p0, p1 = M.indptr[rb[b]], M.indptr[rb[b + 1]]
        if p1 - p0 <= SP_NNZ and p1 > p0:
            o = M.indices[p0:p1].astype(np.int64) - rb[b]
            i16 = i16 and o.min() >= -32768 and o.max() <= 32767
    if M.nnz == 0 or not (f32v or i16):
        return 0
    return RP16 | (I16 if i16 else 0) | (F32V if f32v else 0)


def instance_name(fmt, dt):
    if not fmt:
        return None
    return {f64: {RP16 | I16 | F32V: "dfi16", RP16 | F32V: "dfi32", RP16 | I16: "ddi16"}, f32: {RP16 | I16: "ffi16"}}[dt][fmt]


def launch():
    out = (C.c_int32 * 4)()
    assert L.load().b2k_debug_spmv_launch(out) == L.OK
    return tuple(out)


def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def pairs(m, n, nnz, rng, values):
    A = sp.coo_matrix((values(nnz), (rng.integers(0, m, nnz), rng.integers(0, n, nnz))), shape=(m, n)).tocsr()
    A.sum_duplicates()
    return A


def matrix(kind, seed, ints=False):
    """tall: 24000 x 40, ~2400 nonzeros per column (A' rows take the long-row path); wide: 3000 x 9000.  Both with a
    few empty rows and columns.  7x5, 257x255: odd small shapes.  banded: test_gpu_csr_compact's banded matrix whose
    column offsets reach 32768 above a tile's first row (Float32 values, 32-bit offsets).  ints: integer values in
    [-8, 8] (exact in Float32)."""
    rng = np.random.default_rng(seed)
    values = (lambda k: rng.integers(-8, 9, k).astype(f64)) if ints else rng.standard_normal
    if kind == "banded":
        return banded(100_000, (32768, 32768), values=INTS)
    m, n, nnz = {"tall": (24000, 40, 96000), "wide": (3000, 9000, 60000), "7x5": (7, 5, 20),
                 "257x255": (257, 255, 3000)}[kind]
    A = pairs(m, n, nnz, rng, values)
    keep_r = np.ones(m)
    keep_r[rng.integers(0, m, 5 if m > 100 else 1)] = 0
    keep_c = np.ones(n)
    keep_c[rng.integers(0, n, 3 if n > 100 else 1)] = 0
    A = (sp.diags(keep_r) @ A @ sp.diags(keep_c)).tocsr()
    A.eliminate_zeros()
    A.sort_indices()
    return A


def many_tiles(ns, seed, ints=True):
    """square, with at least 2.5 tiles per CTA of the largest grid (4 CTAs per SM) on both sides: row 3 of A holds
    3000 nonzeros (a tile of its own), columns [5000, 7100) are empty, so A' has a run of 2100 empty rows (a tile of
    more than 1024 rows)"""
    rng = np.random.default_rng(seed)
    nnz = int(3.0 * 4 * ns * SP_NNZ)
    n = nnz // 6
    rows, cols = rng.integers(0, n, nnz), rng.integers(0, n, nnz)
    cols = np.where((cols >= 5000) & (cols < 7100), cols + 2100, cols)
    rows = np.r_[rows, np.full(3000, 3)]
    cols = np.r_[cols, rng.choice(np.r_[np.arange(0, 5000), np.arange(7100, n)], 3000, replace=False)]
    vals = rng.integers(-8, 9, len(rows)).astype(f64) if ints else rng.standard_normal(len(rows))
    vals[vals == 0] = 1.0
    A = sp.coo_matrix((vals, (rows, cols)), shape=(n, n)).tocsr()
    A.sum_duplicates()
    A.eliminate_zeros()
    A.sort_indices()
    return A


class Chain:
    """A, A' on the device with a start state: orthonormal U (m x k), V (n x k), a residual r"""

    def __init__(self, A, dt, k, seed=3):
        self.A, self.dt, self.k = A, dt, k
        self.At = A.T.tocsr()
        self.At.sort_indices()
        m, n = A.shape
        self.ctx = kk.B200Context(m, k + 40, dtype=dt)
        self.sv = self.ctx.add_space(n, k + 40, sharded=False)
        self.op = kk.B200CSR.from_scipy(self.ctx, A).with_spaces(self.sv, 0)
        self.opt = self.op.transpose()
        rng = np.random.default_rng(seed)
        self.U0 = np.linalg.qr(rng.standard_normal((m, k)))[0].astype(dt)
        self.V0 = np.linalg.qr(rng.standard_normal((n, k)))[0].astype(dt)
        self.r0 = rng.standard_normal(m).astype(dt)
        self.beta0 = float(np.linalg.norm(self.r0.astype(f64)))

    def start(self):
        U = [self.ctx.from_host(self.U0[:, j]) for j in range(self.k)]
        V = [self.ctx.from_host(self.V0[:, j], self.sv) for j in range(self.k)]
        return U, self.ctx.from_host(self.r0), V

    def call(self, U, r, V, nsteps, beta, tol, alg):
        """(status, alphas, betas, d, U, r, V) after one b2k_gkl_expand_many call"""
        k = len(U)
        uc = (L.c_vec * (k + nsteps + 1))(*[u.handle for u in U], r.handle)
        vc = (L.c_vec * (k + nsteps))(*[v.handle for v in V])
        al, be = (C.c_double * nsteps)(), (C.c_double * nsteps)()
        done, rout = C.c_int32(), L.c_vec()
        st = self.ctx.lib.b2k_gkl_expand_many(self.ctx.h, self.op.h, self.opt.h, uc, vc, k, nsteps, beta, tol, alg,
                                              al, be, C.byref(done), C.byref(rout))
        d = done.value
        if d > 0:
            r.disown()
            U = U + [kk.B200Vec(self.ctx, uc[k + i]) for i in range(d)]
            V = V + [kk.B200Vec(self.ctx, vc[k + i]) for i in range(d)]
            r = kk.B200Vec(self.ctx, rout.value)
        return st, list(al[:d]), list(be[:d]), d, U, r, V

    def close(self):
        self.opt.free()
        self.op.free()
        self.ctx.close()


def grid_of(op_host, variant):
    """the TMA SpMV grid: min(tiles, per_sm SMs), per_sm 4 in variant 1 (the default) and 3 in variant 0, for the pipe
    and the compact kernel alike"""
    nblk = len(R.tiles(op_host.indptr)) - 1
    return min(nblk, (4 if variant == 1 else 3) * nsm())


def restate_step(fma, dt, A, U, r, V, beta, alg, ns, variant=1):
    """one chained step from the host state (U: m x k, r, V: n x k) -> (alpha, beta, u, v, r'')"""
    At = A.T.tocsr()
    At.sort_indices()
    csr = lambda M: (M.indptr, M.indices, M.data.astype(dt))
    # A' SpMV with the GKL epilogue
    s = R.csr_rows(*csr(At), r, dt, 1.0 / beta, "pipe")
    vt = fma(-dt(beta), V[:, -1], s, dt)
    if alg == L.CGS2:
        gid, rank = R.csr_threads(R.tiles(At.indptr), grid_of(At, variant))
        n2 = R.dot(fma, dt, vt, vt, gid, rank, grid_of(At, variant), "pipe")
    else:
        _, vt, n2 = TR.cgs(V, vt, 1, ns, fma)
    alpha = float(np.sqrt(n2))
    # A SpMV with the GKL epilogue
    s2 = R.csr_rows(*csr(A), vt, dt, 1.0 / alpha, "pipe")
    u = (r * dt(1.0 / beta)).astype(dt)
    rp = fma(-dt(alpha), u, s2, dt)
    _, rpp, b2 = TR.cgs(np.column_stack([U, u]), rp, 1, ns, fma)
    v = (vt * dt(1.0 / alpha)).astype(dt)
    return alpha, float(np.sqrt(b2)), u, v, rpp


def step_cases():
    """(kernel, dt, shape, integer values, the instance A's SpMV must take: pipe or a compact one)"""
    out = []
    for kname in ("pipe24", "pipe33"):
        for dt in (f64, f32):
            for shape in ("tall", "wide", "7x5", "257x255"):
                out.append((kname, dt, shape, False, "pipe"))
    for kname in ("compact1", "compact0"):
        out += [(kname, f64, "tall", False, "ddi16"), (kname, f64, "wide", False, "ddi16"),
                (kname, f32, "tall", False, "ffi16"), (kname, f32, "wide", False, "ffi16"),
                (kname, f64, "tall", True, "dfi16"), (kname, f64, "wide", True, "dfi16"),
                (kname, f64, "banded", True, "dfi32"), (kname, f64, "7x5", False, "ddi16"),
                (kname, f32, "257x255", False, "ffi16")]
    return out


def case_id(c):
    kname, dt, shape, ints, inst = c
    return f"{kname}-{inst if inst != 'pipe' else ('f64' if dt == f64 else 'f32')}-{shape}{'-ints' if ints else ''}"


STEP_CASES = step_cases()


def check_kernels(ch, kname, inst):
    """the formats of A and A' (host prediction = device), and the kernel and instance of the last SpMV, A's"""
    lib = L.load()
    dt = ch.dt
    fa, ft = compact_format(ch.A, dt), compact_format(ch.At, dt)
    assert lib.b2k_debug_csr_format(ch.op.h) == fa and lib.b2k_debug_csr_format(ch.opt.h) == ft
    compact, variant = KERNELS[kname]
    rec = launch()
    if compact and fa:
        assert rec[0] == 3 and instance_name(fa, dt) == inst, (rec, fa, inst)
        assert rec[1] == ((1 if (dt == f32 or fa & F32V) else 0) | (2 if fa & I16 else 0))
    else:
        assert rec[0] == 2 and rec[1] == variant and inst == "pipe", (rec, inst)
    assert rec[2] == grid_of(ch.A, variant)


def one_step(fma, A, dt, kname, alg, k, inst):
    ch = Chain(A, dt, k=k)
    try:
        U, r, V = ch.start()
        with kernel(kname):
            st, al, be, d, U, r, V = ch.call(U, r, V, 1, ch.beta0, 0.0, alg)
            check_kernels(ch, kname, inst)
        assert st == L.OK and d == 1
        a, b, u, v, rr = restate_step(fma, dt, A.astype(dt), ch.U0, ch.r0, ch.V0, ch.beta0, alg, nsm(),
                                      KERNELS[kname][1])
        assert same(np.float64(al[0]), np.float64(a)), (al[0], a)
        assert same(np.float64(be[0]), np.float64(b)), (be[0], b)
        assert same(U[-1].to_host(), u)
        assert same(V[-1].to_host(), v)
        assert same(r.to_host(), rr)
    finally:
        ch.close()


@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
@pytest.mark.parametrize("case", STEP_CASES, ids=[case_id(c) for c in STEP_CASES])
def test_one_step_against_restatement(fma, case, alg):
    kname, dt, shape, ints, inst = case
    A = matrix(shape, seed=5, ints=ints)
    one_step(fma, A, dt, kname, alg, 1 if shape in ("7x5", "257x255") else 3, inst)


MANY = [("pipe24", f64, "dfi32"), ("pipe33", f32, "pipe"), ("compact1", f64, "dfi32"), ("compact0", f64, "dfi32")]


@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
@pytest.mark.parametrize("kname,dt,inst", MANY, ids=[f"{k}-{'f64' if d == f64 else 'f32'}" for k, d, _ in MANY])
def test_one_step_many_tiles_per_cta(fma, kname, dt, inst, alg):
    """every CTA walks 2.5 tiles or more on both sides, through a long row and a tile of more than 1024 rows"""
    A = many_tiles(nsm(), seed=8)
    At = A.T.tocsr()
    grid = 4 * nsm()
    for M in (A, At):
        rb = R.tiles(M.indptr)
        assert len(rb) - 1 >= 2.5 * grid
    assert np.diff(A.indptr).max() > SP_NNZ
    assert np.diff(R.tiles(At.indptr)).max() > 1024
    if kname.startswith("pipe"):
        inst = "pipe"
    one_step(fma, A, dt, kname, alg, 3, inst)


BATCH_CASES = [(kname, dt, shape, False) for kname in KERNELS for dt in (f64, f32) for shape in ("tall", "wide")] + \
    [(kname, f64, shape, True) for kname in ("compact1", "compact0") for shape in ("tall", "banded")]


@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
@pytest.mark.parametrize("kname,dt,shape,ints", BATCH_CASES,
                         ids=[f"{k}-{'f64' if d == f64 else 'f32'}-{s}{'-ints' if i else ''}" for k, d, s, i in BATCH_CASES])
def test_batch_equals_single_steps(kname, dt, shape, ints, alg):
    A = matrix(shape, seed=6, ints=ints)
    N = 7
    ch = Chain(A, dt, k=2)
    try:
        with kernel(kname):
            U1, r1, V1 = ch.start()
            st, al1, be1, d1, U1, r1, V1 = ch.call(U1, r1, V1, N, ch.beta0, 0.0, alg)
            assert st == L.OK and d1 == N
            check_kernels(ch, kname, instance_name(compact_format(A, dt), dt) if KERNELS[kname][0] and
                          compact_format(A, dt) else "pipe")
            U2, r2, V2 = ch.start()
            al2, be2, beta = [], [], ch.beta0
            for _ in range(N):
                st, a, b, d, U2, r2, V2 = ch.call(U2, r2, V2, 1, beta, 0.0, alg)
                assert st == L.OK and d == 1
                al2 += a
                be2 += b
                beta = b[0]
        assert same(np.array(al1), np.array(al2)) and same(np.array(be1), np.array(be2))
        for x, y in zip(U1 + V1 + [r1], U2 + V2 + [r2]):
            assert same(x.to_host(), y.to_host())
    finally:
        ch.close()


def same_nan(a, b):
    """bit for bit, NaNs by position"""
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return a.dtype == b.dtype and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
def test_non_finite_alpha_stops_the_batch(dt, alg):
    """+Inf in one value of A: the first step's v~ and so its alpha are not finite.  nsteps = 4 returns one step, its
    alpha non-finite and its beta NaN, status OK; the input columns are untouched, the column bookkeeping holds
    exactly the one new U and V column and the residual, and the new V column is that of a call of nsteps = 1"""
    A = matrix("wide", seed=5).astype(f64)
    A.data[A.data.size // 2] = np.inf
    lib = L.load()
    got = []
    for nsteps in (4, 1):
        ch = Chain(A, dt, k=2)
        try:
            U, r, V = ch.start()
            before = [x.to_host() for x in U + V]
            used = lib.b2k_debug_used_columns(ch.ctx.h, 0), lib.b2k_debug_used_columns(ch.ctx.h, ch.sv)
            st, al, be, d, U, r, V = ch.call(U, r, V, nsteps, ch.beta0, 0.0, alg)
            assert st == L.OK and d == 1, (st, d)
            assert not np.isfinite(al[0]) and np.isnan(be[0]), (al, be)
            assert all(same(a, x.to_host()) for a, x in zip(before, U[:2] + V[:2]))
            assert lib.b2k_debug_used_columns(ch.ctx.h, 0) == used[0] + 1
            assert lib.b2k_debug_used_columns(ch.ctx.h, ch.sv) == used[1] + 1
            got.append((al, V[-1].to_host()))
        finally:
            ch.close()
    (a4, v4), (a1, v1) = got
    assert same(np.array(a4), np.array(a1)) and same_nan(v4, v1)


@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
def test_stop_inside_a_batch(alg):
    rng = np.random.default_rng(9)
    m, n = 5000, 700
    A = sp.csr_matrix(rng.standard_normal((m, 3)) @ rng.standard_normal((3, n)))
    ch = Chain(A, f64, k=1)
    # the state after GKL's initialize: u1 = x / |x|, v1 = A'u1 / alpha, r = A v1 - alpha u1
    u1 = rng.standard_normal(m)
    u1 /= np.linalg.norm(u1)
    v1 = A.T @ u1
    a1 = np.linalg.norm(v1)
    v1 /= a1
    ch.U0, ch.V0, ch.r0 = u1[:, None], v1[:, None], A @ v1 - a1 * u1
    ch.beta0 = float(np.linalg.norm(ch.r0))
    lib = L.load()
    try:
        tol = 1e-8
        U1, r1, V1 = ch.start()
        used = lib.b2k_debug_used_columns(ch.ctx.h, 0), lib.b2k_debug_used_columns(ch.ctx.h, ch.sv)
        launches = ch.ctx.launches
        st, al1, be1, d1, U1, r1, V1 = ch.call(U1, r1, V1, 12, ch.beta0, tol, alg)
        batch_launches = ch.ctx.launches - launches
        assert st == L.OK and 1 <= d1 < 12 and be1[-1] <= tol and all(b > tol for b in be1[:-1])
        # the columns in use: the d new U and V columns, the new residual in place of the old one
        assert lib.b2k_debug_used_columns(ch.ctx.h, 0) == used[0] + d1
        assert lib.b2k_debug_used_columns(ch.ctx.h, ch.sv) == used[1] + d1
        U2, r2, V2 = ch.start()
        al2, be2, beta = [], [], ch.beta0
        while True:
            st, a, b, d, U2, r2, V2 = ch.call(U2, r2, V2, 1, beta, tol, alg)
            al2 += a
            be2 += b
            beta = b[0]
            if beta <= tol:
                break
        assert same(np.array(al1), np.array(al2)) and same(np.array(be1), np.array(be2))
        for x, y in zip(U1 + V1 + [r1], U2 + V2 + [r2]):
            assert same(x.to_host(), y.to_host())
        # every launch of the batch was enqueued (seed, 3 or 4 per step, flush); the skipped ones changed nothing,
        # which the equality with stepping shows
        assert batch_launches == 2 + 12 * (4 if alg == L.MGS2B else 3)
    finally:
        ch.close()


def test_refusals_write_nothing():
    A = matrix("wide", seed=2)
    ch = Chain(A, f64, k=2)
    lib = L.load()
    try:
        U, r, V = ch.start()
        dense = kk.B200Dense.from_host(ch.ctx, np.ones((A.shape[0], A.shape[1])), ch.sv)
        cases = [
            (ch.op, ch.opt, L.MGS2, U, V, 3, L.ENOTSUP),          # an orthogonalizer that is not chained
            (ch.op, ch.op, L.CGS2, U, V, 3, L.EDIM),              # At is not A's shape transposed
            (ch.op, ch.opt, L.CGS2, U, U, 3, L.EDIM),             # V from the wrong space
            (ch.op, ch.opt, L.CGS2, U, V, 95, L.ENOTSUP),         # more columns than the panel ring holds
            (dense, ch.opt, L.CGS2, U, V, 3, L.ENOTSUP),          # a dense operator
        ]
        for A_, At_, alg, Uc, Vc, nsteps, code in cases:
            k = len(Uc)
            uc = (L.c_vec * (k + nsteps + 1))(*[u.handle for u in Uc], r.handle)
            vc = (L.c_vec * (k + nsteps))(*[v.handle for v in Vc])
            bu, bv = list(uc), list(vc)
            al, be = (C.c_double * nsteps)(*([-3.0] * nsteps)), (C.c_double * nsteps)(*([-3.0] * nsteps))
            done, rout = C.c_int32(-7), L.c_vec(-7)
            used = lib.b2k_debug_used_columns(ch.ctx.h, 0), lib.b2k_debug_used_columns(ch.ctx.h, ch.sv)
            before = [x.to_host() for x in U + V + [r]]
            st = ch.ctx.lib.b2k_gkl_expand_many(ch.ctx.h, A_.h, At_.h, uc, vc, k, nsteps, ch.beta0, 0.0, alg, al,
                                                be, C.byref(done), C.byref(rout))
            assert st == code, (st, code)
            assert list(uc) == bu and list(vc) == bv and done.value == -7 and rout.value == -7
            assert list(al) == [-3.0] * nsteps and list(be) == [-3.0] * nsteps
            assert (lib.b2k_debug_used_columns(ch.ctx.h, 0), lib.b2k_debug_used_columns(ch.ctx.h, ch.sv)) == used
            assert all(same(a, x.to_host()) for a, x in zip(before, U + V + [r]))
        dense.free()
    finally:
        ch.close()
