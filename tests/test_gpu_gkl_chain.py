"""GPU tests of the device-chained GKL step, b2k_gkl_expand_many, in Float64 and Float32.

1. One chained step equals, bit for bit, a numpy restatement of its documented order (include/b200krylov.h, basis.cu):
     v~ = fma(-beta, v_{k-1}, A' (r * T(1/beta)))        the A' SpMV's epilogue (spmv_restate.csr_rows)
     alpha = sqrt of the fused norm of v~                 CGS2: the SpMV's CTA-ordered sum (spmv_restate.dot)
                                                          MGS2B: v~ -= V V' v~ first, alpha from the sweep's finaliser
     u = rn(r * T(1/beta)),  r' = fma(-alpha, u, A (v~ * T(1/alpha)))
     r'' = one classical pass of r' over [U, u], beta = sqrt(||r''||^2)    (tsk_restate.cgs)
     v = rn(v~ * T(1/alpha))                              the flush launch
   on the plain (pipe) and the compact kernels, on a tall matrix whose transpose has rows longer than one tile (1536
   nonzeros: the long-row path) and on a wide one, both with empty rows and columns.
2. A batch of N steps equals N calls of one step bit for bit: alpha, beta and every U, V and r column (CGS2, MGS2B).
3. A stop in the middle of a batch (beta <= tol on a rank-3 matrix): steps_done, the columns and the released
   handles are those of stepping, and the launches behind the stop do nothing.
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

f64, f32 = np.float64, np.float32


@contextlib.contextmanager
def kernel(name):
    """pipe: the plain TMA kernel (compact copies off); compact: the compact copy where the operator has one"""
    lib = L.load()
    lib.b2k_debug_set_csr_compact(1 if name == "compact" else 0)
    try:
        yield
    finally:
        lib.b2k_debug_set_csr_compact(1)


def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def matrix(kind, seed):
    """tall: 24000 x 40, ~2400 nonzeros per column (A' rows take the long-row path); wide: 3000 x 9000.  Both with a
    few empty rows and columns."""
    rng = np.random.default_rng(seed)
    m, n, nnz = (24000, 40, 96000) if kind == "tall" else (3000, 9000, 60000)
    A = sp.coo_matrix((rng.standard_normal(nnz), (rng.integers(0, m, nnz), rng.integers(0, n, nnz))), shape=(m, n))
    A = A.tocsr()
    A.sum_duplicates()
    keep_r = np.ones(m)
    keep_r[rng.integers(0, m, 5)] = 0
    keep_c = np.ones(n)
    keep_c[rng.integers(0, n, 3)] = 0
    A = (sp.diags(keep_r) @ A @ sp.diags(keep_c)).tocsr()
    A.eliminate_zeros()
    A.sort_indices()
    return A


class Chain:
    """A, A' on the device with a start state: orthonormal U (m x k), V (n x k), a residual r"""

    def __init__(self, A, dt, k, seed=3):
        self.A, self.dt, self.k = A, dt, k
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


def grid_of(op_host):
    nblk = len(R.tiles(op_host.indptr)) - 1
    return min(nblk, 4 * nsm())           # the default SpMV variant: 4 CTAs per SM


def restate_step(fma, dt, A, U, r, V, beta, alg, ns):
    """one chained step from the host state (U: m x k, r, V: n x k) -> (alpha, beta, u, v, r'')"""
    At = A.T.tocsr()
    At.sort_indices()
    csr = lambda M: (M.indptr, M.indices, M.data.astype(dt))
    # A' SpMV with the GKL epilogue
    s = R.csr_rows(*csr(At), r, dt, 1.0 / beta, "pipe")
    vt = fma(-dt(beta), V[:, -1], s, dt)
    if alg == L.CGS2:
        gid, rank = R.csr_threads(R.tiles(At.indptr), grid_of(At))
        n2 = R.dot(fma, dt, vt, vt, gid, rank, grid_of(At), "pipe")
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


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("kname", ["pipe", "compact"])
@pytest.mark.parametrize("shape", ["tall", "wide"])
@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
def test_one_step_against_restatement(fma, dt, kname, shape, alg):
    A = matrix(shape, seed=5)
    ch = Chain(A, dt, k=3)
    try:
        U, r, V = ch.start()
        with kernel(kname):
            st, al, be, d, U, r, V = ch.call(U, r, V, 1, ch.beta0, 0.0, alg)
        assert st == L.OK and d == 1
        a, b, u, v, rr = restate_step(fma, dt, A.astype(dt), ch.U0, ch.r0, ch.V0, ch.beta0, alg, nsm())
        assert same(np.float64(al[0]), np.float64(a)), (al[0], a)
        assert same(np.float64(be[0]), np.float64(b)), (be[0], b)
        assert same(U[-1].to_host(), u)
        assert same(V[-1].to_host(), v)
        assert same(r.to_host(), rr)
    finally:
        ch.close()


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("alg", [L.CGS2, L.MGS2B], ids=["cgs2", "mgs2b"])
@pytest.mark.parametrize("shape", ["tall", "wide"])
def test_batch_equals_single_steps(dt, alg, shape):
    A = matrix(shape, seed=6)
    N = 7
    ch = Chain(A, dt, k=2)
    try:
        U1, r1, V1 = ch.start()
        st, al1, be1, d1, U1, r1, V1 = ch.call(U1, r1, V1, N, ch.beta0, 0.0, alg)
        assert st == L.OK and d1 == N
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
