"""GPU parity of the C-ABI primitives (called through the ctypes binding) against plain
numpy float64 restatements of the same reference ops (VectorInterface / orthonormal.jl)."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
import test_gpu_transform as T
from test_gpu_transform import expected_kernel

SEED = 20260923
UR_KERNEL = {1: T.K_UR218, 2: T.K_UR236, 3: T.K_UR418}


def splitmix_host(seed, n, offset=0):
    i = (np.arange(n, dtype=np.uint64) + np.uint64(offset) + np.uint64(seed))
    with np.errstate(over="ignore"):
        z = i + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def laplace2d(nx, ny, coeffs=(4.0, -1.0, -1.0, -1.0, -1.0)):
    c, w, e, s, n = coeffs
    ex = sp.diags([w * np.ones(nx - 1), e * np.ones(nx - 1)], [-1, 1], shape=(nx, nx))
    ey = sp.diags([s * np.ones(ny - 1), n * np.ones(ny - 1)], [-1, 1], shape=(ny, ny))
    A = sp.kron(sp.identity(ny), ex) + sp.kron(ey, sp.identity(nx)) + c * sp.identity(nx * ny)
    return A.tocsr()


@pytest.mark.parametrize("dtype,n", [(np.float64, 1000), (np.float64, 70001), (np.float32, 4099),
                                     (np.float64, 1), (np.float64, 255), (np.float64, 257)])
def test_blas1(dtype, n):
    ctx = kk.B200Context(n, 8, dtype=dtype)
    rng = np.random.default_rng(1)
    xh = rng.standard_normal(n).astype(dtype)
    yh = rng.standard_normal(n).astype(dtype)
    x, y = ctx.from_host(xh), ctx.from_host(yh)
    tol = 1e-13 if dtype == np.float64 else 2e-5
    assert np.array_equal(x.to_host(), xh)
    ref = float(np.dot(xh.astype(np.float64), yh.astype(np.float64)))
    assert abs(x.inner(y) - ref) <= tol * np.linalg.norm(xh) * np.linalg.norm(yh)
    assert abs(x.norm() - np.linalg.norm(xh.astype(np.float64))) <= tol * np.linalg.norm(xh)
    y.add_(x, 0.5, -2.0)
    yh = (-2.0 * yh + 0.5 * xh).astype(dtype)
    np.testing.assert_allclose(y.to_host(), yh, rtol=4 * tol, atol=4 * tol)
    y.add_(x, 3.0)
    yh = yh + dtype(3.0) * xh
    np.testing.assert_allclose(y.to_host(), yh, rtol=4 * tol, atol=4 * tol)
    y.add_(x, 2.0, 0.0)          # beta = 0: hard overwrite
    np.testing.assert_allclose(y.to_host(), 2 * xh, rtol=tol)
    z = x.scale(0.25)
    np.testing.assert_array_equal(z.to_host(), (dtype(0.25) * xh))
    x.scale_(-3.0)
    np.testing.assert_array_equal(x.to_host(), (dtype(-3.0) * xh))
    w = x.zerovector()
    assert not w.to_host().any()
    # deterministic: same bits when repeated
    assert x.inner(z) == x.inner(z)
    ctx.close()


def test_splitmix_matches_host():
    n = 5000
    ctx = kk.B200Context(n, 4)
    v = ctx.splitmix(SEED)
    np.testing.assert_array_equal(v.to_host(), splitmix_host(SEED, n))
    ctx.close()


@pytest.fixture(params=[(1, 1), (1, 0), (0, 1)], ids=["pipe-2x4", "pipe-3x3", "stream"])
def spmv_kernel(request):
    """the TMA-pipelined SpMV in its two stage/occupancy variants and the plain streaming kernel"""
    lib = L.load()
    lib.b2k_debug_set_spmv_pipe(request.param[0])
    lib.b2k_debug_set_spmv_variant(request.param[1])
    yield request.param[0]
    lib.b2k_debug_set_spmv_pipe(1)
    lib.b2k_debug_set_spmv_variant(1)


@pytest.mark.parametrize("nx,ny", [(100, 100), (125, 80), (1, 7), (2048, 3), (37, 1), (1000, 700)])
def test_spmv_stencil_and_csr(nx, ny, spmv_kernel):
    n = nx * ny
    A = laplace2d(nx, ny)
    ctx = kk.B200Context(n, 8)
    op_s = kk.B200CSR.stencil(ctx, nx, ny)
    op_c = kk.B200CSR.from_scipy(ctx, A)
    # the device-assembled stencil is the same CSR matrix
    As = op_s.to_scipy()
    assert As.shape[0] == n and op_s.nnz == A.nnz
    assert abs(As[:, :n] - A).max() == 0
    xh = splitmix_host(SEED, n)
    x = ctx.from_host(xh)
    ref = A @ xh
    for op in (op_s, op_c):
        y = kk.apply(op, x)
        np.testing.assert_allclose(y.to_host(), ref, rtol=1e-14, atol=1e-14)
        # fused <v, A x>
        v = ctx.from_host(np.cos(np.arange(n)))
        y2 = ctx.empty()
        d = op.apply_dot_into(y2, x, v)
        np.testing.assert_array_equal(y2.to_host(), y.to_host())
        assert abs(d - np.dot(np.cos(np.arange(n)), ref)) <= 1e-12 * max(1.0, np.linalg.norm(ref)) * np.sqrt(n)
        # shifted apply: a1*A x + a0*x
        ysh = kk.apply(op, x, 0.3, -1.5)
        np.testing.assert_allclose(ysh.to_host(), -1.5 * ref + 0.3 * xh, rtol=1e-13, atol=1e-13)
    ctx.close()


def test_spmv_irregular_rows_and_csc(spmv_kernel):
    rng = np.random.default_rng(5)
    n = 3000
    A = sp.random(n, n, density=0.002, random_state=7, format="lil")
    A[17, :] = rng.standard_normal(n)          # one long row (> 2048 nnz)
    A[100:140, :] = 0                            # empty rows
    A[2000:, :] = 0                              # a long run of empty rows (> rowptr staging)
    A[2500, 3] = 1.5
    A = A.tocsr()
    A.sort_indices()
    ctx = kk.B200Context(n, 6)
    xh = rng.standard_normal(n)
    x = ctx.from_host(xh)
    op = kk.B200CSR.from_scipy(ctx, A)
    np.testing.assert_allclose(kk.apply(op, x).to_host(), A @ xh, rtol=1e-12, atol=1e-12)
    Ac = A.tocsc()
    Ac.sort_indices()
    op2 = kk.B200CSR.from_julia_csc(ctx, n, n, Ac.indptr + 1, Ac.indices + 1, Ac.data)
    np.testing.assert_allclose(kk.apply(op2, x).to_host(), A @ xh, rtol=1e-12, atol=1e-12)
    ctx.close()


def _basis(ctx, n, k, rng, contiguous=True):
    Q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    if contiguous:
        vecs = ctx.empty_range(k)
    else:
        vecs = [ctx.empty() for _ in range(2 * k)][::2]
    for j, v in enumerate(vecs):
        v.upload(Q[:, j])
    return Q, kk.OrthonormalBasis(vecs)


@pytest.mark.parametrize("n,k", [(1000, 5), (70001, 30), (256, 8), (513, 61), (100, 1), (5000, 9),
                                 (20000, 130)])
def test_project_unproject(n, k):
    rng = np.random.default_rng(n + k)
    ctx = kk.B200Context(n, 2 * k + 6)
    Q, b = _basis(ctx, n, k, rng, contiguous=(k % 2 == 0))
    xh = rng.standard_normal(n)
    x = ctx.from_host(xh)
    y = np.zeros(k)
    kk.project_(y, b, x)
    np.testing.assert_allclose(y, Q.T @ xh, rtol=1e-12, atol=1e-12)
    y2 = np.ones(k)
    kk.project_(y2, b, x, 2.0, -0.5)
    np.testing.assert_allclose(y2, -0.5 + 2.0 * (Q.T @ xh), rtol=1e-12, atol=1e-12)
    c = rng.standard_normal(k)
    z = ctx.from_host(xh)
    kk.unproject_(z, b, c, -1.0, 1.0)
    np.testing.assert_allclose(z.to_host(), xh - Q @ c, rtol=1e-12, atol=1e-12)
    kk.unproject_(z, b, c, 0.7, 0.0)
    np.testing.assert_allclose(z.to_host(), 0.7 * (Q @ c), rtol=1e-12, atol=1e-12)
    kk.unproject_(z, b, c, 1.0, 2.5, )
    np.testing.assert_allclose(z.to_host(), 2.5 * 0.7 * (Q @ c) + Q @ c, rtol=1e-12, atol=1e-12)
    # range r: subset of columns
    if k >= 3:
        r = [0, 2]
        yr = np.zeros(2)
        kk.project_(yr, b, x, 1.0, 0.0, r)
        np.testing.assert_allclose(yr, Q[:, r].T @ xh, rtol=1e-12, atol=1e-12)
    lc = b * c
    np.testing.assert_allclose(lc.to_host(), Q @ c, rtol=1e-12, atol=1e-12)
    ctx.close()


ALGS = [kk.cgs, kk.mgs, kk.cgs2, kk.mgs2, kk.ClassicalGramSchmidtIR(eta=0.75), kk.ModifiedGramSchmidtIR(eta=0.75)]


@pytest.mark.parametrize("alg", ALGS, ids=lambda a: type(a).__name__)
@pytest.mark.parametrize("n,k", [(2000, 7), (70001, 30), (300, 61)])
@pytest.mark.parametrize("coop", [1, 0])
def test_orthogonalize(alg, n, k, coop):
    """test/linalg.jl:4-25 invariants: x reproduces the removed components, result is
    orthogonal to the basis, norm identity."""
    L.load().b2k_debug_set_coop(coop)
    rng = np.random.default_rng(3 * n + k)
    ctx = kk.B200Context(n, k + 6)
    Q, b = _basis(ctx, n, k, rng)
    vh = rng.standard_normal(n)
    v = ctx.from_host(vh)
    v, x = kk.orthogonalize_(v, b, alg)
    nrm = kk.orthogonalize_.last_norm
    out = v.to_host()
    tol = 1e-12 if alg.tag not in (L.CGS, L.MGS) else 1e-10
    np.testing.assert_allclose(x, Q.T @ vh, rtol=tol, atol=tol)
    assert np.abs(Q.T @ out).max() < tol * np.linalg.norm(vh)
    np.testing.assert_allclose(out, vh - Q @ (Q.T @ vh), rtol=tol, atol=tol * np.linalg.norm(vh))
    assert abs(nrm - np.linalg.norm(out)) < 1e-12 * np.linalg.norm(vh)
    assert abs(np.hypot(np.linalg.norm(x), nrm) - np.linalg.norm(vh)) < 1e-11 * np.linalg.norm(vh)
    L.load().b2k_debug_set_coop(1)
    ctx.close()


def test_cgs2_coop_equals_split_bitwise():
    n, k = 50001, 48
    rng = np.random.default_rng(0)
    ctx = kk.B200Context(n, k + 6)
    Q, b = _basis(ctx, n, k, rng)
    vh = rng.standard_normal(n)
    res = []
    for coop in (1, 0):
        L.load().b2k_debug_set_coop(coop)
        v = ctx.from_host(vh)
        v, x = kk.orthogonalize_(v, b, kk.cgs2)
        res.append((v.to_host(), x.copy(), kk.orthogonalize_.last_norm))
        v.free()
    L.load().b2k_debug_set_coop(1)
    assert np.array_equal(res[0][0], res[1][0])
    assert np.array_equal(res[0][1], res[1][1])
    assert res[0][2] == res[1][2]
    ctx.close()


def test_orthogonalize_single_vector():
    n = 12345
    rng = np.random.default_rng(9)
    ctx = kk.B200Context(n, 6)
    qh = rng.standard_normal(n)
    qh /= np.linalg.norm(qh)
    vh = rng.standard_normal(n)
    q = ctx.from_host(qh)
    for alg in ALGS:
        v = ctx.from_host(vh)
        v, s = kk.orthogonalize_(v, q, alg)
        assert abs(s - qh @ vh) < 1e-12
        assert abs(qh @ v.to_host()) < 1e-12
        v.free()
    ctx.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n,m,keep", [(70001, 30, 18), (5000, 60, 36), (300, 61, 61), (1000, 3, 1),
                                      (512, 30, 18), (100003, 90, 75),
                                      # wider than the resident ring (96 f64 / 192 f32 columns): staged-tile kernel
                                      (20011, 100, 64), (3000, 130, 130), (777, 256, 40), (5000, 200, 199)])
def test_basistransform(n, m, keep, dtype):
    rng = np.random.default_rng(n)
    ctx = kk.B200Context(n, m + 4, dtype=dtype)
    Q, _ = np.linalg.qr(rng.standard_normal((n, m)))
    Q = Q.astype(dtype)
    vecs = ctx.empty_range(m)
    for j, v in enumerate(vecs):
        v.upload(Q[:, j])
    b = kk.OrthonormalBasis(vecs)
    U, _ = np.linalg.qr(rng.standard_normal((m, m)))
    kk.basistransform_(b, U[:, :keep])
    assert L.load().b2k_debug_transform_kernel() == expected_kernel(dtype, m, keep)
    ref = Q.astype(np.float64) @ U[:, :keep]
    tol = 1e-12 if dtype == np.float64 else 2e-6
    for j in range(keep):
        np.testing.assert_allclose(b[j].to_host(), ref[:, j], rtol=tol, atol=tol)
    for j in range(keep, m):        # untouched
        np.testing.assert_array_equal(b[j].to_host(), Q[:, j])
    ctx.close()


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("n,m,keep", [(70001, 60, 36), (5000, 30, 18), (257, 61, 35), (100003, 96, 36), (999, 5, 1)])
def test_basistransform_constant_bank_variants(n, m, keep, mode):
    """k_transform_ur (DFMA with U in the kernel-parameter constant bank; thread <-> 2x18, 2x36, 4x18 register
    tiles) against the dense product; sums in increasing i with fma, so the three layouts agree bit for bit."""
    lib = L.load()
    rng = np.random.default_rng(n + m)
    Q, _ = np.linalg.qr(rng.standard_normal((n, m)))
    U, _ = np.linalg.qr(rng.standard_normal((m, m)))
    ref = Q @ U[:, :keep]
    outs = []
    try:
        for md in (mode, 1):
            lib.b2k_debug_set_transform(md)
            ctx = kk.B200Context(n, m + 4)
            vecs = ctx.empty_range(m)
            for j, v in enumerate(vecs):
                v.upload(Q[:, j])
            b = kk.OrthonormalBasis(vecs)
            kk.basistransform_(b, U[:, :keep])
            assert lib.b2k_debug_transform_kernel() == expected_kernel(np.float64, m, keep, md) == UR_KERNEL[md]
            out = np.column_stack([b[j].to_host() for j in range(m)])
            np.testing.assert_allclose(out[:, :keep], ref, rtol=1e-12, atol=1e-12)
            np.testing.assert_array_equal(out[:, keep:], Q[:, keep:])
            outs.append(out)
            ctx.close()
    finally:
        lib.b2k_debug_set_transform(0)
    np.testing.assert_array_equal(outs[0], outs[1])


@pytest.mark.parametrize("n,m,keep", [(70001, 60, 36), (5000, 30, 18), (257, 61, 35), (100003, 96, 36), (999, 5, 1),
                                      (4096, 40, 25), (3001, 59, 31), (777, 36, 36),
                                      # the hybrid at its limit (m <= 92); DMMA at its limit (m·ceil8(keep) = 3680)
                                      (100003, 92, 36), (20011, 92, 40)])
@pytest.mark.parametrize("mode", [4, 5, 6, 7], ids=["dmma+dfma", "dfma8x9", "dmma", "dfma8x9-512"])
def test_basistransform_hybrid_dmma_dfma(n, m, keep, mode):
    """k_transform_hyb (output columns [0, 24) on the FP64 tensor pipe, [24, 36) as register-blocked DFMA, in the same
    warps) and k_transform_f89 (DFMA only, thread <-> 8 rows x 9 outputs) against the dense product, ragged tiles and
    chunk tails included.  At m = 96 neither the hybrid (m·40·8 > 29 440 bytes) nor DMMA (96·40 > 3680) fits: modes 4
    and 6 fall back to k_transform.  keep = 40 is past every keep <= 36 kernel: all four modes run DMMA."""
    lib = L.load()
    rng = np.random.default_rng(7 * n + m)
    Q, _ = np.linalg.qr(rng.standard_normal((n, m)))
    U, _ = np.linalg.qr(rng.standard_normal((m, m)))
    ref = Q @ U[:, :keep]
    lib.b2k_debug_set_transform(mode)
    try:
        ctx = kk.B200Context(n, m + 4)
        vecs = ctx.empty_range(m)
        for j, v in enumerate(vecs):
            v.upload(Q[:, j])
        b = kk.OrthonormalBasis(vecs)
        kk.basistransform_(b, U[:, :keep])
        kid = lib.b2k_debug_transform_kernel()
        assert kid == expected_kernel(np.float64, m, keep, mode)
        if m == 96 and mode in (4, 6):
            assert kid == T.K_F64_SMEM
        elif keep == 40:
            assert kid == T.K_DMMA
        else:
            assert kid == {4: T.K_HYB, 5: T.K_F89, 6: T.K_DMMA, 7: T.K_F89W}[mode]
        out = np.column_stack([b[j].to_host() for j in range(m)])
        np.testing.assert_allclose(out[:, :keep], ref, rtol=1e-12, atol=1e-12)
        np.testing.assert_array_equal(out[:, keep:], Q[:, keep:])
        ctx.close()
    finally:
        lib.b2k_debug_set_transform(0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_givens_householder_rank1(dtype):
    """test/linalg.jl:27-44: Givens / Householder on a basis equal the dense result."""
    n, k = 4001, 10
    rng = np.random.default_rng(2)
    ctx = kk.B200Context(n, k + 6, dtype=dtype)
    Q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    Q = Q.astype(dtype).astype(np.float64)
    vecs = ctx.empty_range(k)
    for j, v in enumerate(vecs):
        v.upload(Q[:, j])
    b = kk.OrthonormalBasis(vecs)
    f32 = dtype == np.float32
    c, s = np.cos(0.3), np.sin(0.3)
    kk.rmul_givens_(b, 2, 5, c, s)
    Q2 = Q.copy()
    Q2[:, 2], Q2[:, 5] = c * Q[:, 2] - s * Q[:, 5], s * Q[:, 2] + c * Q[:, 5]
    for j in range(k):
        np.testing.assert_allclose(b[j].to_host(), Q2[:, j], rtol=1e-14 if not f32 else 1e-6, atol=1e-15 if not f32 else 1e-7)
    # Householder on columns r
    r = [1, 2, 3, 4, 7]
    vv = rng.standard_normal(len(r))
    vv[0] = 1.0
    beta = 2.0 / (vv @ vv)
    kk.rmul_householder_(b, beta, vv, r)
    Q3 = Q2.copy()
    w = Q2[:, r] @ vv
    Q3[:, r] -= beta * np.outer(w, vv)
    for j in range(k):
        np.testing.assert_allclose(b[j].to_host(), Q3[:, j], rtol=1e-13 if not f32 else 1e-5, atol=1e-14 if not f32 else 1e-6)
    # rank-1 update with beta != 1
    y = ctx.from_host(rng.standard_normal(n))
    xh = rng.standard_normal(k)
    kk.rank1update_(b, y, xh, 0.5, 2.0)
    Q4 = 2.0 * Q3 + 0.5 * np.outer(y.to_host(), xh)
    for j in range(k):
        np.testing.assert_allclose(b[j].to_host(), Q4[:, j], rtol=1e-13 if not f32 else 1e-5, atol=1e-14 if not f32 else 1e-5)
    ctx.close()


def test_dense_gemv_f32():
    m, n = 20011, 300
    ctx = kk.B200Context(m, 8, dtype=np.float32)
    sv = ctx.add_space(n, 8, sharded=False)
    rng = np.random.default_rng(4)
    A = (rng.random((m, n)) - 0.5).astype(np.float32)
    op = kk.B200Dense.from_host(ctx, A, sv)
    xh = rng.standard_normal(n).astype(np.float32)
    uh = rng.standard_normal(m).astype(np.float32)
    x = ctx.from_host(xh, sv)
    u = ctx.from_host(uh)
    y = kk.apply_normal(op, x)
    ref = A.astype(np.float64) @ xh.astype(np.float64)
    np.testing.assert_allclose(y.to_host(), ref, rtol=2e-5, atol=2e-5 * np.abs(ref).max())
    z = kk.apply_adjoint(op, u)
    ref2 = A.astype(np.float64).T @ uh.astype(np.float64)
    np.testing.assert_allclose(z.to_host(), ref2, rtol=2e-5, atol=2e-5 * np.abs(ref2).max())
    ctx.close()


def test_errors_map_to_exceptions():
    ctx = kk.B200Context(100, 4)
    ctx2_space = ctx.add_space(50, 4)
    a, b2 = ctx.zeros(), ctx.zeros(ctx2_space)
    with pytest.raises(kk.DimensionMismatch):
        a.inner(b2)
    with pytest.raises(kk.B200Error):
        [ctx.empty() for _ in range(10)]
    ctx.close()


@pytest.mark.parametrize("alg", ALGS, ids=lambda a: type(a).__name__)
@pytest.mark.parametrize("n,k", [(100003, 30), (2_000_128, 12)])
def test_orthogonalize_float32_multi_tile(alg, n, k):
    """Float32 path of the fused / pipelined Gram-Schmidt kernels with many row tiles per CTA
    (config 4's vector length), against a float64 numpy restatement."""
    rng = np.random.default_rng(n + k)
    ctx = kk.B200Context(n, k + 6, dtype=np.float32)
    Q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    Q = Q.astype(np.float32)
    vecs = ctx.empty_range(k)
    for j, v in enumerate(vecs):
        v.upload(Q[:, j])
    b = kk.OrthonormalBasis(vecs)
    vh = rng.standard_normal(n).astype(np.float32)
    v = ctx.from_host(vh)
    v, x = kk.orthogonalize_(v, b, alg)
    nrm = kk.orthogonalize_.last_norm
    out = v.to_host().astype(np.float64)
    Q64, v64 = Q.astype(np.float64), vh.astype(np.float64)
    scale = np.linalg.norm(v64)
    tol = 3e-6 if alg.tag not in (L.CGS, L.MGS) else 3e-5
    np.testing.assert_allclose(x, Q64.T @ v64, atol=tol * scale)
    assert np.abs(Q64.T @ out).max() < tol * scale
    assert abs(nrm - np.linalg.norm(out)) < 1e-5 * scale
    assert np.isfinite(out).all()
    ctx.close()


def test_block_multi_rhs_kernels():
    """block.cu: block_inner / block_axpy as multi-right-hand-side launches (incl. > 48 basis columns = several
    passes and > 8 block columns), SpMM bit-identical to single applies, BCGS2 against a basis, CholeskyQR2
    equal to the MGS factor and refusing a rank-deficient block."""
    import ctypes as C
    from krylovkit_jl_b200.factorizations import blocklanczos as blz
    from krylovkit_jl_b200.orthonormal import OrthonormalBasis
    rng = np.random.default_rng(5)
    n = 70_001                                           # ragged last tile
    ctx = kk.B200Context(n, 140)
    Xh = rng.standard_normal((n, 60))
    Yh = rng.standard_normal((n, 11))
    X = [ctx.from_host(Xh[:, j]) for j in range(60)]
    Y = [ctx.from_host(Yh[:, j]) for j in range(11)]
    M = blz.block_inner(kk.Block(X), kk.Block(Y))
    np.testing.assert_allclose(M, Xh.T @ Yh, rtol=1e-12, atol=1e-9)
    C_ = rng.standard_normal((60, 11))
    blz.block_axpy_(kk.Block(Y), X, C_)
    Yn = Yh - Xh @ C_
    np.testing.assert_allclose(np.column_stack([y.to_host() for y in Y]), Yn, rtol=1e-12, atol=1e-10)
    # SpMM == loop of SpMVs, bit for bit
    nx, ny = 271, 193
    ctx2 = kk.B200Context(nx * ny, 40)
    op = kk.B200CSR.stencil(ctx2, nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0, 0))
    Z = [ctx2.from_host(rng.standard_normal(nx * ny)) for _ in range(5)]
    AZ = blz._apply_block(op, kk.Block(Z))
    for z, az in zip(Z, AZ):
        assert np.array_equal(kk.apply(op, z).to_host(), az.to_host())
    # BCGS2 + CholeskyQR2
    Q, _ = np.linalg.qr(rng.standard_normal((n, 50)))
    V = OrthonormalBasis([ctx.from_host(Q[:, j]) for j in range(50)])
    Rh = rng.standard_normal((n, 4)) + Q[:, :4] * 100.0
    Rb = kk.Block([ctx.from_host(Rh[:, i]) for i in range(4)])
    H, G = blz.block_orthogonalize_fast_(Rb, V)
    Ro = np.column_stack([r.to_host() for r in Rb])
    assert np.abs(Q.T @ Ro).max() < 1e-12 * np.abs(Rh).max() * 50
    np.testing.assert_allclose(H, Q.T @ Rh, rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(G, Ro.T @ Ro, rtol=1e-12)
    np.testing.assert_allclose(Ro, Rh - Q @ (Q.T @ Rh), atol=1e-9)
    Rfac, ok = blz.block_cholqr_(Rb, 1e-12, G)
    assert ok
    Qo = np.column_stack([r.to_host() for r in Rb])
    np.testing.assert_allclose(Qo.T @ Qo, np.eye(4), atol=1e-13)
    np.testing.assert_allclose(Qo @ Rfac, Ro, rtol=1e-12, atol=1e-12)
    assert np.allclose(np.tril(Rfac, -1), 0) and np.all(np.diag(Rfac) > 0)
    Rm = np.linalg.qr(Ro)[1]
    np.testing.assert_allclose(Rfac, Rm * np.sign(np.diag(Rm))[:, None], rtol=1e-10, atol=1e-10)
    # rank-deficient block: refused, untouched
    D = [ctx.from_host(Rh[:, 0]), ctx.from_host(Rh[:, 1]), ctx.from_host(2.0 * Rh[:, 0] - Rh[:, 1])]
    before = [d.to_host() for d in D]
    _, ok = blz.block_cholqr_(kk.Block(D), 1e-12)
    assert not ok
    for d, b in zip(D, before):
        assert np.array_equal(d.to_host(), b)
    ctx.close()
    ctx2.close()


@pytest.mark.parametrize("grid,coeffs", [((97, 61, 1), (4.0, -1.0, -1.0, -1.0, -1.0, 0.0, 0.0)),
                                          ((64, 50, 1), (4.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0)),
                                          ((23, 17, 13), (6.0, -1.0, -1.1, -0.9, -1.0, -1.2, -0.8))])
def test_matrix_free_stencil_equals_assembled_operator(grid, coeffs):
    """b2k_op_create_stencil_free evaluates the stencil from the vector (no stored matrix): apply, shifted apply and
    the fused dot are bit-identical to the assembled CSR operator; the device-chained Lanczos steps run on it too."""
    from krylovkit_jl_b200.factorizations import lanczos as lz
    nx, ny, nz = grid
    n = nx * ny * nz
    rng = np.random.default_rng(8)
    ctx = kk.B200Context(n, 48)
    A = kk.B200CSR.stencil(ctx, nx, ny, nz, coeffs)
    F = kk.B200CSR.stencil_free(ctx, nx, ny, nz, coeffs)
    assert F.n_rows == n               # (the real library reports nnz == 0: nothing is stored)
    x = ctx.from_host(rng.standard_normal(n))
    v = ctx.from_host(rng.standard_normal(n))
    assert np.array_equal(kk.apply(F, x).to_host(), kk.apply(A, x).to_host())
    assert np.array_equal(kk.apply(F, x, 0.3, 1.7).to_host(), kk.apply(A, x, 0.3, 1.7).to_host())
    ya, yf = ctx.empty(), ctx.empty()
    da, df = A.apply_dot_into(ya, x, v), F.apply_dot_into(yf, x, v)
    assert np.array_equal(ya.to_host(), yf.to_host())
    assert abs(da - df) <= 1e-13 * abs(da)            # same products, other partition of the final sum
    res = []
    for op in (A, F):
        it = lz.LanczosIterator(op, ctx.from_host(np.random.default_rng(3).random(n)), kk.cgs2)
        f = lz.initialize(it)
        lz.expand_many_(it, f, 20, 0.0)
        res.append((np.array(f.alphas), np.array(f.betas)))
        del f, it
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=1e-13)
    np.testing.assert_allclose(res[0][1], res[1][1], rtol=1e-12)
    ctx.close()
