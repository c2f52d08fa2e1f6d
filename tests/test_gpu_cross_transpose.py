"""GPU tests of the two device primitives a two-sided (BiArnoldi) Krylov method needs: the cross Gram matrix
b2k_basis_cross_inner (G = X'Y of two column lists, one sweep) and the device-side CSR transpose
b2k_op_create_transpose (B200CSR.transpose()).

Rounding contract of b2k_basis_cross_inner (basis.cu), restated on the host by `cross_restate` and compared bit for
bit.  The lists are split into column blocks of at most 64 x 64; for each block, with NO = ceil(pb/4) ceil(qb/4)
entry tiles and RS the largest power of two <= min(32, 256 / NO) row slices, grid = min(ceil(n / 64), #SMs) CTAs,
CTA g owning the 64-row tiles g, g + grid, ...:
  a[g, s][i, j] = fma chain in the vector type T, from 0, over the rows r of CTA g's tiles (ascending) with
                  r % RS == s: a = fma(X[r, i], Y[r, j], a);
  G[i, j]       = sum over g in order (from 0.0, in double) of  sum over s in order (from 0.0) of (double) a[g, s].
The fma of the host restatement is libm's (gcc, -ffp-contract=off), through the `fma` fixture of test_gpu_blas1.

Tolerances.  u is the unit roundoff of T.  At n = 1e7 the result is compared with a float64 reference within
LAM sqrt(m) u sum(|terms|) (Higham & Mary's probabilistic bound, m the longest fma chain) plus the same bound for the
double stages and for the reference itself.  Integer data in [-8, 8] keeps every partial sum exact.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.vectors import handles
from test_gpu_blas1 import fma, num_sms  # noqa: F401  (fma: module fixture)
from test_gpu_paths import LAM, SP_NNZ, unit

SEED = 20261016
f64, f32 = np.float64, np.float32
DTYPES = [f64, f32]
CI_B, CI_R, CROSS = 64, 64, 9          # column block, rows per tile, profile class of the sweep


# ---------------------------------------------------------------- cross Gram ----

def row_slices(pb, qb):
    no = -(-pb // 4) * -(-qb // 4)
    rs = 1
    while rs * 2 <= 32 and rs * 2 * no <= 256:
        rs *= 2
    return rs


def blocks(p, q, p0, q0):
    """the column blocks the library sweeps (those with an entry outside the skip block)"""
    out = []
    for i0 in range(0, p, CI_B):
        for j0 in range(0, q, CI_B):
            pb, qb = min(CI_B, p - i0), min(CI_B, q - j0)
            if not (i0 + pb <= p0 and j0 + qb <= q0):
                out.append((i0, pb, j0, qb))
    return out


def cross_restate(X, Y, p0, q0, fma, dt, nsm):
    """the documented contract, entry by entry; skipped entries are NaN"""
    n, p = X.shape
    q = Y.shape[1]
    G = np.full((p, q), np.nan)
    if n == 0:
        G[:, :] = 0.0
        G[:p0, :q0] = np.nan
        return G
    ntiles = -(-n // CI_R)
    grid = min(ntiles, nsm)
    Xp = np.vstack([X, np.zeros((1, p))]).astype(dt)
    Yp = np.vstack([Y, np.zeros((1, q))]).astype(dt)
    for i0, pb, j0, qb in blocks(p, q, p0, q0):
        rs = row_slices(pb, qb)
        lists = [[t * CI_R + r for t in range(g, ntiles, grid) for r in range(s, CI_R, rs) if t * CI_R + r < n]
                 for g in range(grid) for s in range(rs)]
        m = max(len(li) for li in lists)
        idx = np.full((grid * rs, m), n, dtype=np.int64)
        for k, li in enumerate(lists):
            idx[k, :len(li)] = li
        idx = idx.reshape(grid, rs, m)
        acc = np.zeros((grid, rs, pb, qb), dtype=dt)
        for step in range(m):
            xr = Xp[idx[:, :, step], i0:i0 + pb]
            yr = Yp[idx[:, :, step], j0:j0 + qb]
            acc = fma(xr[..., :, None], yr[..., None, :], acc, dt)
        part = np.zeros((grid, pb, qb))
        for s in range(rs):
            part = part + acc[:, s].astype(f64)
        tot = np.zeros((pb, qb))
        for g in range(grid):
            tot = tot + part[g]
        G[i0:i0 + pb, j0:j0 + qb] = tot
    G[:p0, :q0] = np.nan
    return G


def call_cross(ctx, X, Y, p0=0, q0=0, G=None, ldg=None):
    p, q = len(X), len(Y)
    if G is None:
        G = np.full((ldg or p, q), np.nan, order="F")
    st = ctx.lib.b2k_basis_cross_inner(ctx.h, handles(X), p, handles(Y), q, p0, q0,
                                       G.ctypes.data_as(C.POINTER(C.c_double)), G.shape[0])
    return st, G


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def lists_for(ctx, rng, n, p, q, dt, shared=True, data=None):
    """p + q columns uploaded in a shuffled order; with `shared` the last quarter of Y repeats columns of X"""
    k_sh = (q // 4) if shared and q >= 4 and p >= q // 4 else 0
    cols = ctx.empty_range(p + q - k_sh)
    M = data if data is not None else rng.standard_normal((n, len(cols)))
    for v, c in zip(cols, M.T):
        v.upload(np.ascontiguousarray(c, dtype=dt))
    order = rng.permutation(len(cols))
    X = [cols[i] for i in order[:p]]
    Y = [cols[i] for i in order[p:]] + X[:k_sh]
    Xh = np.column_stack([v.to_host() for v in X]).astype(f64)
    Yh = np.column_stack([v.to_host() for v in Y]).astype(f64)
    return cols, X, Y, Xh, Yh


def size_of(name):
    nsm = num_sms()
    return {"sub": 37, "ragged": 3 * CI_R + 5, "one": nsm * CI_R, "several": 3 * nsm * CI_R + 41}[name]


SHAPES = [(1, 1, 0, 0), (31, 31, 18, 18), (32, 33, 1, 1), (33, 32, 0, 0), (64, 64, 18, 18), (65, 65, 0, 0),
          (65, 31, 64, 31), (31, 65, 1, 1)]


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("size", ["sub", "ragged", "one", "several"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{p}x{q}-skip{p0}x{q0}" for p, q, p0, q0 in SHAPES])
def test_cross_inner_matches_restatement(fma, dt, size, shape):
    p, q, p0, q0 = shape
    n = size_of(size)
    rng = np.random.default_rng([SEED, n, p, q])
    ctx = kk.B200Context(n, p + q + 4, dtype=dt)
    cols, X, Y, Xh, Yh = lists_for(ctx, rng, n, p, q, dt)
    before = ctx.launches
    st, G = call_cross(ctx, X, Y, p0, q0)
    assert st == L.OK
    assert ctx.launches - before == 2 * len(blocks(p, q, p0, q0))
    assert same(G, cross_restate(Xh, Yh, p0, q0, fma, dt, num_sms()))
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("p0", [0, 1, 18])
def test_cross_inner_256_columns(fma, dt, p0):
    """the largest lists: 4 x 4 column blocks, the skip block removes none / part of one / part of one"""
    n, p, q = 300, 256, 256
    rng = np.random.default_rng([SEED, p0])
    ctx = kk.B200Context(n, p + q + 4, dtype=dt)
    cols, X, Y, Xh, Yh = lists_for(ctx, rng, n, p, q, dt)
    st, G = call_cross(ctx, X, Y, p0, p0)
    assert st == L.OK
    assert same(G, cross_restate(Xh, Yh, p0, p0, fma, dt, num_sms()))
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_cross_inner_small_integers_exact(dt):
    n, p, q = 3 * num_sms() * CI_R + 41, 33, 31
    rng = np.random.default_rng(SEED + 1)
    ctx = kk.B200Context(n, p + q + 4, dtype=dt)
    cols, X, Y, Xh, Yh = lists_for(ctx, rng, n, p, q, dt, data=rng.integers(-8, 9, size=(n, p + q)))
    st, G = call_cross(ctx, X, Y)
    assert st == L.OK
    exact = Xh.astype(np.int64).T @ Yh.astype(np.int64)
    assert np.array_equal(G, exact.astype(f64))
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_cross_inner_large_n_bound_and_repeatable(dt):
    """n = 1e7: within the two-stage bound of a float64 reference; a second call gives the same bits"""
    n, p, q = 10_000_000, 16, 16
    ctx = kk.B200Context(n, p + q + 2, dtype=dt)
    X = [ctx.splitmix(1000 + i) for i in range(p)]
    Y = [ctx.splitmix(2000 + j) for j in range(q)]
    c = ctx.full(-0.5)           # centre the uniform [0, 1) entries
    for v in X + Y:
        v.add_(c, 1.0, 1.0)
    Xh = np.column_stack([v.to_host().astype(f64) for v in X])
    Yh = np.column_stack([v.to_host().astype(f64) for v in Y])
    st, G = call_cross(ctx, X, Y)
    assert st == L.OK
    st2, G2 = call_cross(ctx, X, Y)
    assert st2 == L.OK and np.array_equal(G, G2)
    ref = Xh.T @ Yh
    S = np.abs(Xh).T @ np.abs(Yh)
    grid = min(-(-n // CI_R), num_sms())
    chain = -(-(-(-n // CI_R)) // grid) * CI_R      # rows of the longest per-thread chain (RS = 1 bound)
    tol = LAM * (np.sqrt(chain) * unit(dt) + np.sqrt(grid * 32) * 2.0 ** -53 + np.sqrt(n) * 2.0 ** -53) * S
    assert np.all(np.abs(G - ref) <= tol)
    ctx.close()


def test_cross_inner_touches_only_what_it_owns():
    """skip block and columns outside G's p x q are untouched, and so is every column of the slab"""
    n, p, q, p0, q0, ldg = 1000, 20, 12, 7, 5, 24
    rng = np.random.default_rng(SEED + 2)
    ctx = kk.B200Context(n, p + q + 6, dtype=f64)
    cols, X, Y, Xh, Yh = lists_for(ctx, rng, n, p, q, f64)
    extra = ctx.from_host(rng.standard_normal(n))
    slab = [v.to_host() for v in cols + [extra]]
    G = np.full((ldg, q + 1), 7.25, order="F")
    st = ctx.lib.b2k_basis_cross_inner(ctx.h, handles(X), p, handles(Y), q, p0, q0,
                                       G.ctypes.data_as(C.POINTER(C.c_double)), ldg)
    assert st == L.OK
    assert np.all(G[:p0, :q0] == 7.25) and np.all(G[p:, :] == 7.25) and np.all(G[:, q:] == 7.25)
    ref = Xh.T @ Yh
    mask = np.ones((p, q), bool)
    mask[:p0, :q0] = False
    assert np.allclose(G[:p, :q][mask], ref[mask], rtol=1e-12, atol=1e-10)
    assert all(np.array_equal(a, v.to_host()) for a, v in zip(slab, cols + [extra]))
    # everything skipped: no launch, nothing written
    before = ctx.launches
    st, G3 = call_cross(ctx, X, Y, p, q)
    assert st == L.OK and ctx.launches == before and np.all(np.isnan(G3))
    ctx.close()


def test_cross_inner_profile_class_counts_sweeps():
    n = 5000
    ctx = kk.B200Context(n, 150, dtype=f64)
    X = ctx.empty_range(70)
    Y = ctx.empty_range(70)
    for v in X + Y:
        ctx.check(ctx.lib.b2k_vec_fill(ctx.h, v.handle, 1.0))
    ctx.check(ctx.lib.b2k_prof_reset(ctx.h))
    ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 1))
    st, _ = call_cross(ctx, X, Y, 64, 64)          # blocks (0,0) skipped: three sweeps
    ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 0))
    assert st == L.OK
    cnt, byt = C.c_int64(), C.c_double()
    ctx.check(ctx.lib.b2k_prof_read(ctx.h, CROSS, C.byref(cnt), None, C.byref(byt)))
    assert cnt.value == 3
    assert byt.value == 8.0 * n * ((64 + 6) + (6 + 64) + (6 + 6))
    ctx.close()


def test_cross_inner_refusals_write_nothing():
    n = 500
    rng = np.random.default_rng(SEED + 3)
    ctx = kk.B200Context(n, 12, dtype=f64)
    sp1 = ctx.add_space(n + 1, 2)
    cols, X, Y, _, _ = lists_for(ctx, rng, n, 3, 4, f64, shared=False)
    other = ctx.from_host(rng.standard_normal(n + 1), space=sp1)
    slab = [v.to_host() for v in cols]
    G = np.full((8, 8), 3.5, order="F")
    Gp = G.ctypes.data_as(C.POINTER(C.c_double))
    hx, hy = handles(X), handles(Y)
    cases = [
        (L.EINVAL, (hx, 0, hy, 4, 0, 0, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 0, 0, 0, Gp, 8)),
        (L.EINVAL, (hx, 257, hy, 4, 0, 0, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 257, 0, 0, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 4, 4, 0, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 4, 0, 5, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 4, -1, 0, Gp, 8)),
        (L.EINVAL, (hx, 3, hy, 4, 0, 0, Gp, 2)),
        (L.EINVAL, (hx, 3, hy, 4, 0, 0, None, 8)),
        (L.EINVAL, (None, 3, hy, 4, 0, 0, Gp, 8)),
        (L.EDIM, (hx, 3, handles(Y[:3] + [other]), 4, 0, 0, Gp, 8)),
        (L.EDIM, (handles([other] + X[1:]), 3, hy, 4, 0, 0, Gp, 8)),
    ]
    for code, args in cases:
        assert ctx.lib.b2k_basis_cross_inner(ctx.h, *args) == code, args
        assert np.all(G == 3.5)
    assert all(np.array_equal(a, v.to_host()) for a, v in zip(slab, cols))
    ctx.close()


def test_cross_inner_python_wrapper_updates_in_place():
    """kk.cross_inner with skip = the size of an earlier call only fills the new rows and columns"""
    n = 777
    rng = np.random.default_rng(SEED + 4)
    ctx = kk.B200Context(n, 24, dtype=f64)
    W = [ctx.from_host(rng.standard_normal(n)) for _ in range(9)]
    V = [ctx.from_host(rng.standard_normal(n)) for _ in range(9)]
    G = np.zeros((10, 10), order="F")
    kk.cross_inner(W[:5], V[:5], G=G)
    lead = G[:5, :5].copy()
    kk.cross_inner(W, V, skip=(5, 5), G=G)
    full = kk.cross_inner(W, V)
    mask = np.ones((9, 9), bool)
    mask[:5, :5] = False
    assert np.array_equal(G[:5, :5], lead)
    assert np.array_equal(G[:9, :9][mask], full[mask])       # same 9 x 9 block shape: same summation order
    assert np.allclose(lead, full[:5, :5], rtol=1e-13, atol=1e-12)
    assert np.all(G[9, :] == 0) and np.all(G[:, 9] == 0)
    ctx.close()


# ---------------------------------------------------------------- transpose ----

def upload(ctx, A, idx=np.int64, base=0):
    A = A.tocsr()
    A.sort_indices()
    return kk.B200CSR.from_csr_arrays(ctx, A.shape[0], A.shape[1], A.indptr.astype(idx) + base,
                                      A.indices.astype(idx) + base, A.data, index_base=base)


def arrays(op):
    rp = np.empty(op.n_rows + 1, dtype=np.int32)
    ci = np.empty(op.nnz, dtype=np.int32)
    va = np.empty(op.nnz, dtype=op.ctx.np_dtype)
    op.ctx.check(op.ctx.lib.b2k_op_csr_download(op.ctx.h, op.h, rp.ctypes.data, ci.ctypes.data, va.ctypes.data))
    return rp, ci, va


def host_transpose(A, dt):
    T = A.T.tocsr().astype(dt)
    T.sort_indices()
    return T.indptr.astype(np.int32), T.indices.astype(np.int32), T.data


_MATS = {}


def matrices():
    if _MATS:
        return _MATS
    rng = np.random.default_rng(SEED + 5)
    out = _MATS
    out["square"] = sp.random(3000, 3000, density=0.002, random_state=rng, format="csr") + sp.eye(3000)
    out["wide"] = sp.random(700, 2100, density=0.004, random_state=rng, format="csr")
    out["tall"] = sp.random(2100, 700, density=0.004, random_state=rng, format="csr")
    A = sp.random(1500, 1500, density=0.003, random_state=rng, format="lil")
    A[100:140, :] = 0
    A[:, 900:960] = 0
    out["empty-rows-cols"] = A.tocsr()
    out["nnz0"] = sp.csr_matrix((1200, 800))
    L_ = sp.random(4000, 4000, density=0.0005, random_state=rng, format="lil")
    L_[17, :] = rng.standard_normal(4000)               # one row past the long-row SpMV threshold
    L_[:, 5] = rng.standard_normal((4000, 1))           # and one long column: a long row of A'
    out["long-row"] = L_.tocsr()
    for k, M in out.items():
        M = M.tocsr()
        M.eliminate_zeros()
        out[k] = M
    assert out["long-row"][17].nnz > SP_NNZ and out["long-row"][:, 5].nnz > SP_NNZ
    return out


MATS = ["square", "wide", "tall", "empty-rows-cols", "nnz0", "long-row"]


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("idx,base", [(np.int64, 0), (np.int32, 1)], ids=["i64-0", "i32-1"])
@pytest.mark.parametrize("name", MATS)
def test_transpose_arrays_and_spmv(dt, idx, base, name):
    A = matrices()[name]
    m, n = A.shape
    ctx = kk.B200Context(m, 4, dtype=dt)
    sp_n = ctx.add_space(n, 4) if n != m else 0
    op = upload(ctx, A.astype(dt), idx, base)
    t = op.transpose()
    assert (t.n_rows, t.n_cols, t.nnz) == (n, m, A.nnz)
    rp, ci, va = arrays(t)
    hrp, hci, hva = host_transpose(A.astype(dt), dt)
    assert np.array_equal(rp, hrp) and np.array_equal(ci, hci) and np.array_equal(va, hva)
    # SpMV with the device transpose == SpMV with the host-built transpose, bit for bit
    th = upload(ctx, A.T.tocsr().astype(dt))
    rng = np.random.default_rng(SEED + 6)
    x = ctx.from_host(rng.standard_normal(m).astype(dt))
    y1, y2 = ctx.empty(sp_n), ctx.empty(sp_n)
    t.apply_into(y1, x)
    th.apply_into(y2, x)
    assert np.array_equal(y1.to_host(), y2.to_host())
    ctx.close()


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("grid", [(40, 30, 1), (12, 9, 7)], ids=["2d", "3d"])
def test_transpose_of_stencil_is_swapped_stencil(dt, grid):
    c = (4.5, -1.25, -0.75, -1.5, -0.5, -1.125, -0.875)
    sw = (c[0], c[2], c[1], c[4], c[3], c[6], c[5])
    nx, ny, nz = grid
    ctx = kk.B200Context(nx * ny * nz, 4, dtype=dt)
    t = kk.B200CSR.stencil(ctx, nx, ny, nz, c).transpose()
    s = kk.B200CSR.stencil(ctx, nx, ny, nz, sw)
    assert all(np.array_equal(a, b) for a, b in zip(arrays(t), arrays(s)))
    ctx.close()


def test_transpose_refusals_and_spaces():
    ctx = kk.B200Context(600, 4, dtype=f64)
    free = kk.B200CSR.stencil_free(ctx, 30, 20)
    with pytest.raises(L.B200Error, match="matrix-free"):
        free.transpose()
    D = kk.B200Dense.from_host(ctx, np.ones((600, 5)), ctx.add_space(5, 4))
    h = L.c_op()
    assert ctx.lib.b2k_op_create_transpose(ctx.h, C.byref(h), D.h) == L.ENOTSUP
    assert "apply_adjoint" in ctx.lib.b2k_last_error(ctx.h).decode()
    # A' would have 900 rows: no space of that length
    A = sp.random(600, 900, density=0.01, random_state=1, format="csr")
    op = upload(ctx, A)
    with pytest.raises(L.DimensionMismatch):
        op.transpose()
    # explicit spaces are swapped
    s9 = ctx.add_space(900, 4)
    op.with_spaces(s9, 0)
    t = op.transpose()
    assert (t.space_in, t.space_out) == (0, s9)
    ctx.close()
