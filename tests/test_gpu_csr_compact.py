"""The compact CSR stream (k_spmv_compact: Float32 values, 16-bit column offsets, 16-bit row pointers) against the
plain k_spmv_pipe on the same operator, bit for bit: y, the fused dot, the shifted apply and the chained Lanczos batch.
b2k_debug_csr_format says which parts of each operator compressed, b2k_debug_spmv_kernel which kernel ran."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.factorizations import lanczos as lz
from oracle import krylov_oracle as ko

F32V, I16, RP16 = 1, 2, 4          # b2k_debug_csr_format bits
K_PIPE, K_COMPACT = 2, 3           # b2k_debug_spmv_kernel ids
SP_NNZ = 1536
SEED = 20261016


def run_both(fn, expect_compact):
    """fn() with the compact kernel allowed, then with B2K_CSR_COMPACT=0's plain kernel; checks which kernel ran"""
    lib = L.load()
    out = []
    try:
        for on in (1, 0):
            lib.b2k_debug_set_csr_compact(on)
            out.append(fn())
            assert lib.b2k_debug_spmv_kernel() == (K_COMPACT if on and expect_compact else K_PIPE)
    finally:
        lib.b2k_debug_set_csr_compact(1)
    return out


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def check_op(ctx, op, fmt, A=None):
    """apply, fused dot and shifted apply of op, compact vs plain; A (scipy) for a loose sanity check"""
    lib = L.load()
    assert lib.b2k_debug_csr_format(op.h) == fmt
    n = op.n_rows
    dt = ctx.np_dtype
    xh = ko.splitmix_vector(SEED, n, dtype=dt)
    x = ctx.from_host(xh)
    v = ctx.from_host(np.cos(np.arange(n)).astype(dt))

    def fn():
        y = kk.apply(op, x).to_host()
        y2 = ctx.empty()
        d = op.apply_dot_into(y2, x, v)
        ysh = kk.apply(op, x, 0.3, -1.5).to_host()
        return y, y2.to_host(), np.float64(d), ysh

    c, p = run_both(fn, fmt != 0)
    for a, b in zip(c, p):
        assert same_bits(a, b)
    if A is not None:
        ref = A.astype(np.float64) @ xh.astype(np.float64)
        fin = np.isfinite(ref)
        tol = 1e-12 if dt == np.float64 else 1e-4
        np.testing.assert_allclose(c[0][fin], ref[fin], rtol=tol, atol=tol * np.abs(A).sum(axis=1).A1.max())


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("grid", [(300, 200, 1), (40, 30, 20)], ids=["2d", "3d"])
def test_stencils(dtype, grid):
    nx, ny, nz = grid
    ctx = kk.B200Context(nx * ny * nz, 8, dtype=dtype)
    op = kk.B200CSR.stencil(ctx, nx, ny, nz)
    check_op(ctx, op, RP16 | I16 | (F32V if dtype == np.float64 else 0))
    ctx.close()


def banded(n, reach, values):
    """3 nonzeros a row ({r-1, r, r+1}, clipped); the first row of two tiles reaches exactly `reach` below / above the
    tile's first row.  Tiles as finish_csr cuts them: rows [ceil(b T / 3), ...) with T = SP_NNZ - 3 + 1."""
    T = SP_NNZ - 3 + 1
    cols = [[0, 1, 2]] + [[r - 1, r, r + 1] for r in range(1, n - 1)] + [[n - 3, n - 2, n - 1]]
    r0s = [-(-b * T // 3) for b in range(n * 3 // T + 1)]
    lo = next(r for r in r0s if r >= reach[0])
    hi = next(r for r in r0s if r > lo and r + reach[1] < n)
    cols[lo] = [lo - reach[0], lo, lo + 1]
    cols[hi] = [hi - 1, hi, hi + reach[1]]
    rows = np.repeat(np.arange(n), 3)
    A = sp.csr_matrix((values(3 * n), (rows, np.array(cols).ravel())), shape=(n, n))
    A.sort_indices()
    return A


INTS = lambda m: np.random.default_rng(1).integers(-8, 9, m).astype(np.float64)
REALS = lambda m: np.random.default_rng(2).standard_normal(m)
BANDED = [  # (dtype, reach below / above, values, format)
    (np.float64, (32768, 32767), INTS, RP16 | I16 | F32V),
    (np.float64, (32768, 32767), REALS, RP16 | I16),
    (np.float64, (32768, 32768), INTS, RP16 | F32V),
    (np.float64, (32769, 32767), REALS, 0),
    (np.float32, (32768, 32767), REALS, RP16 | I16),
    (np.float32, (32768, 32768), REALS, 0),
]


@pytest.mark.parametrize("dtype,reach,values,fmt", BANDED,
                         ids=[f"{np.dtype(d).name}-{r[0]}-{r[1]}-{v is INTS and 'ints' or 'reals'}" for d, r, v, _ in BANDED])
def test_banded_offset_limits(dtype, reach, values, fmt):
    n = 100_000
    A = banded(n, reach, values)
    ctx = kk.B200Context(n, 8, dtype=dtype)
    op = kk.B200CSR.from_scipy(ctx, A)
    check_op(ctx, op, fmt, A)
    ctx.close()


@pytest.mark.parametrize("special,fmt", [(np.nextafter(np.float64(np.float32(0.1)), 1.0), RP16 | I16),
                                         (-0.0, RP16 | I16 | F32V), (np.inf, RP16 | I16 | F32V),
                                         (np.nan, RP16 | I16)], ids=["1ulp", "negzero", "inf", "nan"])
def test_value_eligibility(special, fmt):
    """the 5-point stencil with one value replaced"""
    nx, ny = 120, 90
    c = [4.0, -1.0, -1.0, -1.0, -1.0]
    ex = sp.diags([c[1] * np.ones(nx - 1), c[2] * np.ones(nx - 1)], [-1, 1], shape=(nx, nx))
    ey = sp.diags([c[3] * np.ones(ny - 1), c[4] * np.ones(ny - 1)], [-1, 1], shape=(ny, ny))
    M = (sp.kron(sp.identity(ny), ex) + sp.kron(ey, sp.identity(nx)) + c[0] * sp.identity(nx * ny)).tocsr()
    M.sort_indices()
    M.data[777] = special
    ctx = kk.B200Context(nx * ny, 8)
    op = kk.B200CSR.from_scipy(ctx, M)
    check_op(ctx, op, fmt)
    ctx.close()


@pytest.mark.parametrize("dtype,values", [(np.float64, "ints"), (np.float64, "reals"), (np.float32, "reals")])
def test_long_rows_empty_rows_wide_tiles(dtype, values):
    rng = np.random.default_rng(5)
    n = 6000
    A = sp.random(n, n, density=0.002, random_state=7, format="lil")
    A[17, :] = 1.0                               # a row longer than SP_NNZ: a tile of its own, plain arrays
    A[100:140, :] = 0                            # empty rows
    A[2000:3500, :] = 0                          # a tile of more than SPP_RMAX = 1024 rows: rowptr read from global
    A[3000, 3] = 1.5
    A = A.tocsr()
    A.sort_indices()
    A.data = (rng.integers(-5, 6, A.nnz).astype(np.float64) if values == "ints" else rng.standard_normal(A.nnz))
    assert np.diff(A.indptr).max() > SP_NNZ
    fmt = RP16 | I16 | (F32V if dtype == np.float64 and values == "ints" else 0)
    ctx = kk.B200Context(n, 8, dtype=dtype)
    op = kk.B200CSR.from_scipy(ctx, A)
    check_op(ctx, op, fmt, A)
    ctx.close()


def test_transpose_gets_the_compact_view():
    nx, ny = 150, 120
    ex = sp.diags([-1.0 * np.ones(nx - 1), -2.0 * np.ones(nx - 1)], [-1, 1], shape=(nx, nx))
    ey = sp.diags([-3.0 * np.ones(ny - 1), -0.5 * np.ones(ny - 1)], [-1, 1], shape=(ny, ny))
    M = (sp.kron(sp.identity(ny), ex) + sp.kron(ey, sp.identity(nx)) + 4.0 * sp.identity(nx * ny)).tocsr()
    ctx = kk.B200Context(nx * ny, 8)
    op = kk.B200CSR.from_scipy(ctx, M)
    check_op(ctx, op.transpose(), RP16 | I16 | F32V, M.T.tocsr())
    ctx.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("orth", [kk.cgs2, kk.mgs2b], ids=["cgs2", "mgs2b"])
def test_chained_lanczos_batch(dtype, orth):
    """b2k_lanczos_expand_many chains SpMVs with the 1/β gather, the vout store and the fused α (mgs2b: the
    dot_sub_vec form): compact and plain give the same bits, and so does the loop of synchronous steps"""
    nx, ny, nsteps = 97, 61, 40
    lib = L.load()

    def batch(chain):
        lib.b2k_debug_set_chain(chain)
        try:
            ctx = kk.B200Context(nx * ny, nsteps + 8, dtype=dtype)
            op = kk.B200CSR.stencil(ctx, nx, ny)
            x0 = ctx.from_host(ko.splitmix_vector(SEED, nx * ny, dtype=dtype))
            it = lz.LanczosIterator(op, x0, orth)
            f = lz.initialize(it)
            assert lz.expand_many_(it, f, nsteps, 0.0) == nsteps
            out = (np.array(f.alphas), np.array(f.betas), np.column_stack([v.to_host() for v in f.V]), f.r.to_host())
            del f, it, x0
            ctx.close()
            return out
        finally:
            lib.b2k_debug_set_chain(1)

    runs = {}
    for chain in (1, 0):
        c, p = run_both(lambda: batch(chain), True)
        for a, b in zip(c, p):
            assert same_bits(a, b)
        runs[chain] = c
    for a, b in zip(runs[1], runs[0]):
        assert same_bits(a, b)
