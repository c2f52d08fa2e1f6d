"""CPU tests of the SpMV restatement (tests/spmv_restate.py) that test_gpu_spmv_fused.py holds the kernels to: each
summation order it restates gives a different double than the order it replaces on a constructed input, so a kernel
that moves a sum fails there; the tile partition follows finish_csr's rules; and on integer data, where every order
gives the exact result, the restated y and dot are A x and <v, A x>."""
import numpy as np
import pytest

import spmv_restate as R
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

f64, f32 = np.float64, np.float32
BIG = 1e16          # ulp(1e16) = 2: 1e16 + 1 rounds back to 1e16


def test_warps_in_order_differ_from_block_sum():
    """pipe / compact add the 8 warp sums in order; stream / stencil butterfly them (block_sum)"""
    v = np.zeros(R.BT)
    v[[0, 32, 64, 96]] = [BIG, 1.0, -BIG, 1.0]          # one nonzero per warp: the warp sums are these
    assert R.cta_reduce(v, "pipe") == ((BIG + 1.0) - BIG) + 1.0 == 1.0
    assert R.cta_reduce(v, "stream") == (BIG - BIG) + (1.0 + 1.0) == 2.0     # lanes 0+2 and 1+3, then 0+1


def test_partials_in_cta_order_differ_from_reversed():
    """the last CTA adds the partials in CTA order, thread t taking t, t + 256, ...; reversed gives another double"""
    part = np.zeros(300)
    part[[157, 171, 215, 252]] = [-BIG, 3.0, BIG, 1.0]
    for kernel in ("pipe", "stream"):
        assert R.last_cta(part, kernel) != R.last_cta(part[::-1], kernel)
    assert R.last_cta(part, "pipe") == 5.0 and R.last_cta(part[::-1], "pipe") == 4.0


@pytest.mark.parametrize("dt", [f64, f32])
def test_stored_column_order_differs_from_sorted(dt):
    """a row is summed in stored order, not by ascending column"""
    big = dt(BIG) if dt == f64 else dt(2.0 ** 25)
    rowptr, cols, vals = np.array([0, 3]), np.array([0, 2, 1]), np.array([big, 1.0, -big], dtype=dt)
    x = np.ones(3, dtype=dt)
    y = R.csr_rows(rowptr, cols, vals, x, dt, None, "pipe")
    order = np.argsort(cols, kind="stable")
    ys = R.csr_rows(rowptr, cols[order], vals[order], x, dt, None, "pipe")
    assert y[0] == (big + dt(1.0)) - big == 0.0
    assert ys[0] == (big - big) + dt(1.0) == 1.0


@pytest.mark.parametrize("dt", [f64, f32])
def test_fma_chain_differs_from_plus_equals(fma, dt):
    """a thread's dot terms go into dacc with fma in T, not dacc += rn(dv sd)"""
    e = dt(2.0 ** -27) if dt == f64 else dt(2.0 ** -12)
    dv = np.array([1.0, 1.0 + e], dtype=dt)
    sd = np.array([-1.0, 1.0 + e], dtype=dt)
    gid, rank = np.array([0, 0]), np.array([0, 1])
    d = R.dot(fma, dt, dv, sd, gid, rank, 1, "pipe")
    assert d == float(2 * e) + float(e) * float(e)                       # the exact dv1 sd1 + dv0 sd0
    plus = (dv[1] * sd[1]) + (dv[0] * sd[0])
    assert d != float(plus) and float(plus) == float(2 * e)


def test_rows_of_a_pipe_thread_are_chained_in_tile_order():
    """CTA b takes tiles b, b + G, ...; consumer t rows r0 + t, r0 + t + 256, ...; a stencil thread t rows t, t + 256 G"""
    rowblk = np.array([0, 600, 700, 1300])                 # 3 tiles on a grid of 2
    gid, rank = R.csr_threads(rowblk, 2)
    assert gid[5] == 5 and gid[261] == 5 and gid[517] == 5 and gid[705] == 5
    assert [rank[5], rank[261], rank[517], rank[705]] == [0, 1, 2, 3]
    assert gid[605] == R.BT + 5 and rank[605] == 0
    gid, rank = R.csr_threads(rowblk, 3)                    # k_spmv_stream: one tile per CTA
    assert gid[705] == 2 * R.BT + 5 and rank[705] == 0 and gid[261] == 5 and rank[261] == 1
    gid, rank = R.stencil_threads(2000, 3)
    assert gid[1000] == 1000 - 768 and rank[1000] == 1


def rowptr_of(lens):
    return np.r_[0, np.cumsum(lens)].astype(np.int64)


def check_partition(rowptr, rb):
    lens = np.diff(rowptr)
    assert rb[0] == 0 and rb[-1] == len(lens) and np.all(np.diff(rb) > 0)
    for a, b in zip(rb[:-1], rb[1:]):
        assert rowptr[b] - rowptr[a] <= R.SP_NNZ or b - a == 1


def test_tiles_maxrow_768_is_the_nnz_balanced_partition():
    rp = rowptr_of([768, 768, 768, 1])                     # T = 769, nnz = 2305: 3 tiles
    rb = R.tiles(rp)
    assert rb.tolist() == [0, 2, 3, 4]                     # lower_bound(rowptr, 0 / 769 / 1538)
    check_partition(rp, rb)
    assert R.tiles(rowptr_of([0] * 5000)).tolist() == [0, 5000]     # nnz = 0: one tile of all rows
    rp = rowptr_of(np.random.default_rng(1).integers(0, 9, 20000))
    rb = R.tiles(rp)
    T = R.SP_NNZ - 8 + 1
    assert len(rb) - 1 == -(-rp[-1] // T) and all(rp[rb[b]] >= b * T > rp[rb[b] - 1] for b in range(1, len(rb) - 1))
    check_partition(rp, rb)


def test_tiles_maxrow_769_is_greedy():
    assert R.tiles(rowptr_of([769, 769, 1])).tolist() == [0, 1, 3]
    # a long row alone, runs of <= 1536 nonzeros, at most 2048 rows
    rp = rowptr_of([10, 1537, 1536, 0] + [0] * 5000 + [769])
    rb = R.tiles(rp)
    assert rb.tolist() == [0, 1, 2, 2 + 2048, 2 + 4096, 5005]
    check_partition(rp, rb)


@pytest.mark.parametrize("kernel", ["stream", "pipe"])
@pytest.mark.parametrize("dt", [f64, f32])
def test_integer_data_gives_the_exact_product_and_dot(fma, kernel, dt):
    """every row, shift and dot term accounted for once: with small integers every order is exact"""
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 6, 4000)
    lens[[10, 2000]] = [2500, 1537]
    rp = rowptr_of(lens)
    cols = rng.integers(0, 4000, rp[-1])
    vals = rng.integers(-3, 4, rp[-1]).astype(dt)
    x, v = rng.integers(-3, 4, 4000).astype(dt), rng.integers(-3, 4, 4000).astype(dt)
    A = np.zeros((4000, 4000))
    np.add.at(A, (np.repeat(np.arange(4000), lens), cols), vals.astype(f64))
    rb = R.tiles(rp)
    grid = len(rb) - 1 if kernel == "stream" else 5
    y, vout, d = R.apply(fma, dt, kernel, grid, x, csr=(rp, cols, vals), rowblk=rb, a0=2.0, a1=-1.0, shifted=True,
                         dotv=v)
    want = 2.0 * x.astype(f64) - A @ x.astype(f64)
    assert np.array_equal(y.astype(f64), want) and d == float(v.astype(f64) @ want)
    nx, ny = 50, 80
    y, vout, d = R.apply(fma, dt, "stencil", 3, x, stencil=(nx, ny, 1, (4, -1, -1, -1, -1, 0, 0)), dot_self=True)
    g = x.astype(f64).reshape(ny, nx)
    p = np.pad(g, 1)
    want = (4 * g - p[1:-1, :-2] - p[1:-1, 2:] - p[:-2, 1:-1] - p[2:, 1:-1]).ravel()
    assert np.array_equal(y.astype(f64), want) and d == float(x.astype(f64) @ want)
