"""CPU tests of the row-sharded composition (tests/dist_restate.py) that test_gpu_zz_dist_restate.py holds the sharded
kernels to: with one rank it is the single-GPU restatement; on small integers every composed value is exact; and on
the data the GPU test uses, the rank-order fold gives different bits than the reverse fold, than a fold that starts
from d_0 instead of 0.0, than the lane tree coef_colsum forms over three rank sets, and than the unsharded order, so
a kernel or transport that moves a cross-rank sum fails there."""
import numpy as np
import pytest

import dist_restate as D
import spmv_restate as R
import tsk_restate as ts
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

f64, f32 = np.float64, np.float32
BIG = 1e16          # ulp(1e16) = 2


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("kernel", ["stream", "pipe"])
def test_one_rank_is_the_single_gpu_restatement(fma, dt, kernel):
    n = 3000
    rowptr, cols, vals = D.band_csr(n, 40, 40, 1)
    vals = vals.astype(dt)
    rng = np.random.default_rng(2)
    x, v, s = (rng.standard_normal(n).astype(dt) for _ in range(3))
    rb = R.tiles(rowptr)
    grid = len(rb) - 1 if kernel == "stream" else 1
    for kw in (dict(dotv=v), dict(xscale=-0.7, dot_self=True, shifted=True, a0=0.3, a1=-1.25),
               dict(dotv=v, dsub=s, dsc=-0.45)):
        want = R.apply(fma, dt, kernel, grid, x, csr=(rowptr, cols, vals), rowblk=rb, **kw)
        got = D.spmv(fma, dt, kernel, grid, x, 0, n, csr=D.local_csr(rowptr, cols, vals, 0, n), **kw)
        for a, b in zip(got[:2], want[:2]):
            assert np.array_equal(a, b)
        assert (got[2] is None and want[2] is None) or D.fold([got[2]]) == want[2]
    nx, ny = 50, 60
    st = (nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0))
    xs = rng.standard_normal(nx * ny).astype(dt)
    want = R.apply(fma, dt, "stencil", 2, xs, stencil=st, dot_self=True)
    got = D.spmv(fma, dt, "stencil", 2, xs, 0, nx * ny, stencil=st, dot_self=True)
    assert np.array_equal(got[0], want[0]) and got[2] == want[2]


def test_stencil_csr_is_the_assembled_order(fma):
    """the host CSR of the assembled stencil gives the matrix-free stencil's rows, shard by shard"""
    dims, co = (17, 13, 11), (4.0, -1.4, -0.6, -1.2, -0.8, -0.3, -0.7)
    csr = D.stencil_csr(*dims, co, f64)
    n = int(np.prod(dims))
    x = np.random.default_rng(4).standard_normal(n)
    sizes = [3 * 17 * 13, 8 * 17 * 13]
    off = D.offsets(sizes)
    for p, m in enumerate(sizes):
        a = D.spmv(fma, f64, "pipe", 3, x, off[p], m, csr=D.local_csr(*csr, off[p], m))[0]
        b = D.spmv(fma, f64, "stencil", 3, x, off[p], m, stencil=(*dims, co))[0]
        assert np.array_equal(a, b)


@pytest.mark.parametrize("dt", [f64, f32])
def test_integer_data_is_exact(fma, dt):
    """every row, halo entry and rank partial counted once: the composed y and dot are A x and <v, A x>"""
    sizes = [700, 1900, 1100]
    n = sum(sizes)
    rowptr, cols, vals = D.band_csr(n, 57, 9, 3, ints=True)
    A = np.zeros((n, n))
    np.add.at(A, (np.repeat(np.arange(n), np.diff(rowptr)), cols), vals)
    rng = np.random.default_rng(5)
    x, v = rng.integers(-3, 4, n).astype(dt), rng.integers(-3, 4, n).astype(dt)
    off = D.offsets(sizes)
    ys, ds = [], []
    for p, m in enumerate(sizes):
        y, _, d = D.spmv(fma, dt, "pipe", 2, x, off[p], m, csr=D.local_csr(rowptr, cols, vals.astype(dt), off[p], m),
                         dotv=v, shifted=True, a0=2.0, a1=-1.0)
        ys.append(y)
        ds.append(d)
    want = 2.0 * x.astype(f64) - A @ x.astype(f64)
    assert np.array_equal(np.concatenate(ys).astype(f64), want)
    assert D.fold(ds) == v.astype(f64) @ want


def test_lanczos_step_on_integers_is_exact(fma):
    """the composed step on a diagonal operator with integer data: alpha0 = <v, A v>, the coefficients <q_j, x>, the
    update x - sum_j h_j q_j and ||w||^2 all exact"""
    sizes = [600, 1000, 800]
    n = sum(sizes)
    rng = np.random.default_rng(6)
    d = rng.integers(-2, 3, n).astype(f64)
    csr = (np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64), d)
    V = np.zeros((n, 3))
    for j in range(3):                       # disjoint unit-like columns: every h_j an integer
        V[j * 7:(j + 1) * 7 + 1, j] = 1.0
    r = rng.integers(-2, 3, n).astype(f64)
    ws, v, a0, alpha, beta, n2 = D.lanczos_step(fma, f64, sizes, V, r, 1.0, csr, "pipe", [1, 1, 1], 132)
    w = d * r
    assert a0 == r @ w
    x = w - V[:, -1] * 1.0 - a0 * r
    Q = np.column_stack([V, r])
    h = Q.T @ x
    assert alpha == a0 + h[-1]
    x2 = x - Q @ h
    assert np.array_equal(np.concatenate(ws), x2) and n2 == x2 @ x2 and beta == np.sqrt(x2 @ x2)


def test_the_fold_tells_the_orders_apart():
    """three rank partials: the rank-order fold from 0.0 against the reverse fold and against coef_colsum's lane tree
    (lanes 0, 1, 2 hold the sets; xor 2 adds sets 0 and 2 first); two: against a fold that starts from d_0 (signed
    zeros)"""
    d = [1.0, BIG, -BIG]
    assert D.fold(d) == (1.0 + BIG) - BIG == 0.0
    assert D.fold(d[::-1]) == (-BIG + BIG) + 1.0 == 1.0
    d = [BIG, 1.0, -BIG]
    assert D.fold(d) == 0.0
    assert ts.colsum(np.array(d)[:, None])[0] == (BIG - BIG) + 1.0 == 1.0
    d2 = [-0.0, -0.0]
    assert np.signbit(d2[0] + d2[1]) and not np.signbit(D.fold(d2))


@pytest.mark.parametrize("nranks", [2, 3])
@pytest.mark.parametrize("dt", [f64, f32])
def test_the_gpu_data_tells_the_orders_apart(fma, dt, nranks):
    """on the data of the GPU test's fold case the composed dot differs from the single-GPU launch over all rows and,
    at three ranks, from the reverse fold and from the lane tree"""
    sizes, csr, x, v = D.fold_case(dt, nranks)
    off = D.offsets(sizes)
    ds = [D.spmv(fma, dt, "pipe", 2, x, off[p], m, csr=D.local_csr(*csr, off[p], m), dotv=v)[2]
          for p, m in enumerate(sizes)]
    composed = D.fold(ds)
    if nranks == 3:
        assert composed != D.fold(ds[::-1])
        assert composed != ts.colsum(np.array(ds)[:, None])[0]
    _, _, whole = R.apply(fma, dt, "pipe", 2, x, csr=csr, rowblk=R.tiles(csr[0]), dotv=v)
    assert composed != whole
