"""GPU tests of b2k_lsmr_chain against the fma-order restatement of tests/lsmr_restate.py: one chained iteration,
bit for bit — every vector, the ring, the record and the state — in Float64 and Float32, with and without lambda,
without reorthogonalisation and with a ring of 5 under MGS, MGS2 and CGS2; the beta and alpha sums against the
restated CTA-ordered sums; the breakdown stop codes 2 (beta <= tol) and 3 (alpha <= tol) and the non-finite stop
(code 4) on the device.

The shapes take the four streaming kernels through their edges on each side: k_lsmr_m on m, k_lsmr_n and
k_lsmr_flush_n on n (grid_for(len, 4), trips of 2 slots), k_lsmr_alpha on n (grid_for(n, 8), trips of 4 slots):
lengths 1, V ± 1, 255, 257, a grid exactly at the 4·SMs cap, and a capped grid with three or more trips per thread,
a partly live second slot in the last trip and a tail."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

import lsmr_restate as LR

f64, f32 = np.float64, np.float32


def nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def plain_kernel():
    """the plain TMA SpMV kernel (the compact copy off), the one spmv_restate's "pipe" rows restate"""
    lib = L.load()
    lib.b2k_debug_set_csr_compact(0)
    try:
        yield
    finally:
        lib.b2k_debug_set_csr_compact(1)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def rect(m, n, seed, nnz=None):
    """m x n: about 1% of the entries (or `nnz` of them) plus the leading diagonal; index pairs drawn directly
    (scipy.sparse.random permutes all m n positions)"""
    rng = np.random.default_rng(seed)
    k = max(1, int(0.01 * m * n)) if nnz is None else nnz
    R = sp.coo_matrix((rng.uniform(0.0, 1.0, k), (rng.integers(0, m, k), rng.integers(0, n, k))), shape=(m, n))
    A = (R.tocsr() + sp.eye(m, n)).tocsr()
    A.sum_duplicates()
    A.sort_indices()
    return A


def edge_shape(name, dt, ns):
    """(m, n, nnz, the edges it puts on each side): tiny and odd pairs; a tall matrix at k_lsmr_m's cap and trips
    (A' rows of thousands of nonzeros: the long-row path); a wide one whose n reaches trips for both grid_for(n, 4)
    and grid_for(n, 8), its A rows longer than 1536"""
    if name == "tall_cap":
        m = LR.edge_size("cap", dt, 4, 2, ns)
        LR.check_edge("cap", m, dt, 4, 2, ns)
        return m, 300, 4 * m
    if name == "tall_trips":
        m = LR.edge_size("trips", dt, 4, 2, ns)
        LR.check_edge("trips", m, dt, 4, 2, ns)
        return m, 300, 4 * m
    if name == "wide_trips":
        n = LR.edge_size("trips", dt, 8, 4, ns)
        LR.check_edge("trips", n, dt, 8, 4, ns)
        LR.check_edge("trips", n, dt, 4, 2, ns)
        return 256, n, 256 * 2000
    m, n = {"1x1": (1, 1), "7x5": (7, 5), "255x257": (255, 257), "257x255": (257, 255)}[name]
    return m, n, None


EDGE_SHAPES = ["1x1", "7x5", "255x257", "257x255", "tall_cap", "tall_trips", "wide_trips"]


class Setup:
    def __init__(self, A, dt, K, seed=5):
        self.A, self.dt, self.K, self.R = A, dt, K, max(K, 1)
        m, n = A.shape
        self.ctx = kk.B200Context(m, 16, dtype=dt)
        self.sv = self.ctx.add_space(n, self.R + 12, sharded=False)
        self.op = kk.B200CSR.from_scipy(self.ctx, A.astype(dt)).with_spaces(self.sv, 0)
        self.opt = self.op.transpose()
        rng = np.random.default_rng(seed)
        self.host = {k: rng.standard_normal(n).astype(dt) for k in ("x", "h", "hbar")}
        self.host.update({k: rng.standard_normal(m).astype(dt) for k in ("r", "Ah", "Ahbar", "u")})
        Q = np.linalg.qr(rng.standard_normal((n, self.R)))[0].astype(dt)
        self.ring = [Q[:, j].copy() for j in range(self.R)]

    def upload(self, host=None, ring=None):
        host, ring = host or self.host, ring or self.ring
        c = self.ctx
        self.d = {k: c.from_host(v, self.sv if k in ("x", "h", "hbar") else 0) for k, v in host.items()}
        self.d["av"] = c.zeros()
        self.dring = [c.from_host(q, self.sv) for q in ring]
        self.dspare = c.zeros(self.sv)

    def call(self, st, tol, iter0, nsteps, alg):
        rec, done = np.zeros((nsteps, 16)), C.c_int32(-1)
        sin, sout = (C.c_double * 10)(*st), (C.c_double * 10)()
        rh = (L.c_vec * self.R)(*[q.handle for q in self.dring])
        d = self.d
        s = self.ctx.lib.b2k_lsmr_chain(self.ctx.h, self.op.h, self.opt.h, d["x"].handle, d["h"].handle,
                                        d["hbar"].handle, d["r"].handle, d["Ah"].handle, d["Ahbar"].handle,
                                        d["u"].handle, d["av"].handle, rh, self.K, self.dspare.handle, alg, iter0,
                                        sin, tol, nsteps, rec.ctypes.data_as(C.POINTER(C.c_double)), sout,
                                        C.byref(done))
        return s, rec[:max(done.value, 0)], list(sout)

    def close(self):
        self.opt.free()
        self.op.free()
        self.ctx.close()


STATE = [1.3, 0.7, 0.9, 1.1, 1.4, 0.8, 0.6, 0.35, 0.5]


def one_iteration(fma, A, dt, lam, K, alg):
    s = Setup(A, dt, K)
    try:
        k = 8                                        # the ring is full: the sweep covers all 5 slots, v_8 in slot 2
        st = STATE + [lam]
        s.upload()
        with plain_kernel():
            status, rec, sout = s.call(st, 0.0, k - 1, 1, alg)
        assert status == L.OK and len(rec) == 1
        At = A.T.tocsr()
        At.sort_indices()
        out, ring, spare, a_sum, b_sum, st2, rrec = LR.iteration(fma, dt, A.astype(dt), At.astype(dt), st, s.host,
                                                                 s.ring, K, alg, 0.0, nsm(), k, alpha_dev=rec[0, 0],
                                                                 beta_dev=rec[0, 1])
        # the CTA-ordered sums
        assert same(f64(rec[0, 1]), f64(b_sum)), (rec[0, 1], b_sum)
        assert same(f64(rec[0, 0]), f64(a_sum)), (rec[0, 0], a_sum)
        # the recurrence and its record
        assert same(rec[0, :14], np.array(rrec[:14])), (rec[0], rrec)
        assert same(np.array(sout), np.array(st2))
        # every vector and the ring
        for key in ("x", "h", "hbar", "r", "Ah", "Ahbar", "u"):
            assert same(s.d[key].to_host(), out[key]), key
        for j in range(s.R):
            assert same(s.dring[j].to_host(), ring[j]), j
    finally:
        s.close()


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("lam", [0.0, 0.3])
@pytest.mark.parametrize("K,alg", [(1, L.MGS), (5, L.MGS), (5, L.MGS2), (5, L.CGS2)], ids=["k1", "mgs", "mgs2", "cgs2"])
def test_one_iteration_bit_for_bit(fma, dt, lam, K, alg):
    one_iteration(fma, rect(3000, 800, 4), dt, lam, K, alg)


EDGE_RINGS = {"k1": (1, L.MGS), "mgs": (5, L.MGS), "cgs2": (5, L.CGS2)}
EDGE_CASES = [(shape, ring) for shape in EDGE_SHAPES for ring in EDGE_RINGS
              if shape != "1x1" or ring == "k1"]                      # a ring of 5 needs n >= 5


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("shape,ring", EDGE_CASES, ids=[f"{s}-{r}" for s, r in EDGE_CASES])
def test_one_iteration_bit_for_bit_at_the_edges(fma, shape, ring, dt):
    K, alg = EDGE_RINGS[ring]
    m, n, nnz = edge_shape(shape, dt, nsm())
    one_iteration(fma, rect(m, n, 4, nnz), dt, 0.3, K, alg)


def breakdown_problem(kind, m=400, n=120, seed=7):
    """three distinct singular values; b in the range (the u side runs out: beta <= tol), or with a part orthogonal
    to it (the v side runs out: alpha <= tol).  b is large, so |zetabar| is still above tol when that happens."""
    rng = np.random.default_rng(seed)
    U, _ = np.linalg.qr(rng.standard_normal((m, n)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = sp.csr_matrix(U @ np.diag(np.repeat([3.0, 2.0, 1.0], n // 3)) @ V.T)
    A.sort_indices()
    b = A @ rng.standard_normal(n)
    if kind == "alpha":
        w = rng.standard_normal(m)
        b = b + (w - U @ (U.T @ w))
    return A, 1e6 * b


@pytest.mark.parametrize("shape", [(400, 120), (401, 123)], ids=["400x120", "401x123"])
@pytest.mark.parametrize("kind,code", [("beta", 2), ("alpha", 3)])
@pytest.mark.parametrize("K,alg", [(1, L.MGS), (4, L.MGS), (4, L.CGS2)], ids=["k1", "mgs", "cgs2"])
def test_breakdown_stop_codes(kind, code, K, alg, shape):
    A, b = breakdown_problem(kind, *shape)
    s = Setup(A, f64, K)
    try:
        beta = float(np.linalg.norm(b))
        u = b / beta
        v = (A.T @ b) / beta
        alpha = float(np.linalg.norm(v))
        v = v / alpha
        n, m = A.shape[1], A.shape[0]
        host = {"x": np.zeros(n), "h": v.copy(), "hbar": np.zeros(n), "r": b.copy(), "Ah": np.zeros(m),
                "Ahbar": np.zeros(m), "u": u}
        ring = [v] + [np.zeros(n) for _ in range(s.R - 1)]
        s.upload(host, ring)
        status, rec, sout = s.call([alpha, beta, alpha, 1.0, 1.0, 1.0, 0.0, 0.0, alpha * beta, 0.0], 1e-8, 0, 20,
                                   alg)
        assert status == L.OK
        assert rec[-1, 7] == code and len(rec) < 20
        assert rec[-1, 6] > 1e-8                     # not converged: the driver continues with the literal loop
        assert rec[-1, 8] == (0.0 if code == 2 else 1.0)
        if code == 3:                                # v stays unnormalised in the spare column, the ring untouched
            assert np.linalg.norm(s.dspare.to_host()) <= 1e-8
    finally:
        s.close()


def bits_nan(a):
    """the bytes of a with every NaN replaced by one canonical NaN (NaN payloads are not part of the contract)"""
    a = np.array(a)
    a[np.isnan(a)] = np.nan
    return a.tobytes()


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("K,alg", [(1, L.MGS), (5, L.CGS2)], ids=["k1", "cgs2"])
def test_non_finite_stop_code_4(fma, dt, K, alg):
    """rho_old rho-bar_old underflows to 0 in the seeded state, so g is infinite while alpha, beta and zeta-bar stay
    finite and non-zero: code 4, the record and every vector as restated (NaN by position), and nsteps = 3 leaves
    everything as nsteps = 1 does"""
    A = rect(257, 255, 4)
    st = [1.3, 0.7, 0.9, 1e-200, 1e-200, 0.8, 0.6, 0.35, 0.5, 0.3]
    k = 8
    At = A.T.tocsr()
    At.sort_indices()
    results = []
    for nsteps in (3, 1):
        s = Setup(A, dt, K)
        try:
            s.upload()
            with plain_kernel():
                status, rec, sout = s.call(st, 0.0, k - 1, nsteps, alg)
            assert status == L.OK and len(rec) == 1
            results.append((rec, sout, {key: s.d[key].to_host() for key in s.d if key != "av"},
                            [q.to_host() for q in s.dring], s.dspare.to_host()))
        finally:
            s.close()
    out, ring, spare, a_sum, b_sum, st2, rrec = LR.iteration(fma, dt, A.astype(dt), At.astype(dt), st, s.host,
                                                             s.ring, K, alg, 0.0, nsm(), k)
    rec, sout, vecs, dring, dspare = results[0]
    assert rec[0, 7] == 4.0 and rrec[7] == 4.0 and np.isinf(rec[0, 12])
    assert all(np.isfinite(rec[0, i]) and rec[0, i] != 0.0 for i in (0, 1, 6))
    assert bits_nan(rec[0, :14]) == bits_nan(np.array(rrec[:14]))
    assert bits_nan(sout) == bits_nan(np.array(st2, dtype=f64))
    for key in ("x", "h", "hbar", "r", "Ah", "Ahbar", "u"):
        assert bits_nan(vecs[key]) == bits_nan(out[key]), key
    for j in range(s.R):
        assert bits_nan(dring[j]) == bits_nan(ring[j]), j
    # the launches behind the stop did nothing
    r1, s1, v1, q1, sp1 = results[1]
    assert bits_nan(rec) == bits_nan(r1) and bits_nan(sout) == bits_nan(s1)
    for key in vecs:
        assert bits_nan(vecs[key]) == bits_nan(v1[key]), key
    assert all(bits_nan(a) == bits_nan(b) for a, b in zip(dring, q1)) and bits_nan(dspare) == bits_nan(sp1)
