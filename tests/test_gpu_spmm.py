"""GPU tests of apply(A, ::Block), b2k_op_apply_block, against the exact host restatement of tests/spmv_restate.py: every
row of every vector bit for bit (signed zeros by their bits, NaNs by position).

The contract (DESIGN §3.6): Y[i] = A X[i] for the p vectors of a block, bit-identical to p single applies.  A
single-GPU square CSR operator with X and Y in one slab runs k_spmm_pipe, one launch per group of at most 8 vectors
(profile class 7); the tail group of np < 8 vectors pads its column table by repeating entry 0.  Everything else runs
the loop of single applies (profile class 0), vector by vector: p = 1, X and Y in different spaces, a rectangular
operator, the matrix-free stencil, the streaming SpMV selected (b2k_debug_set_spmv_pipe(0)) and B2K_BLOCK_KERNELS=0.
Refused before anything is written: p < 1 (B2K_EINVAL), Y[j] aliasing X[i] (B2K_EINVAL), and X or Y spanning two
spaces (B2K_EDIM, from b2k_resolve_cols).  A repeated Y handle is written in vector order, so the later vector wins, as
in the loop.

k_spmm_pipe's rows are k_spmv_pipe's: R.csr_rows(..., xscale=None, kernel="pipe") on finish_csr's tiles (R.tiles).  A
row of a tile of at most 1536 nonzeros is its rounded products summed from (T)0 in CSR order; a longer row, alone in
its tile, is the strided double sums of consumer threads 0..255, each warp's butterfly, then red[0 .. 7] added in order
from 0.0 by thread 0, rounded to T once: exactly k_spmv_pipe's long row.  The streaming SpMV sums a long row's warp
sums by block_sum instead (R.cta_reduce(..., "stream")), so against stream applies the long rows are held to their own
restatements; the block path never stands in for the stream kernel, as b2k_debug_set_spmv_pipe(0) sends it to the loop.

The many-tiles matrix gives every CTA of the grid G = min(nblk, 3 SMs) at least three tiles (CTA c takes tiles c,
c + G, c + 2G, ...), so the two-stage ring wraps and flips its phase; a long tile sits between two short ones of one
CTA (release without a read stage), a tile of more than 1024 rows (row pointers read from global memory) between two
staged ones, and two long tiles follow each other; the last tile is ragged.
"""
import contextlib
import os

import numpy as np
import pytest

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.factorizations import blocklanczos as bl
from krylovkit_jl_b200.vectors import handles
from test_gpu_blas1 import num_sms
from test_gpu_paths import SPMM, SPMV, edge_matrix, profiled
from test_gpu_spmv_fused import COMPACT, COMPACT_INST, PIPE, STREAM, device_tiles, kernel, launch, same

import spmv_restate as R

gpu = pytest.mark.gpu
f64, f32 = np.float64, np.float32
DTS = [f64, f32]
DIDS = ["f64", "f32"]
SM_H100 = 132                  # the H100 SXM's SM count, for the CPU checks of the many-tiles layout
NCOLS = 56                     # slab columns of a shared context: 24 X, 24 Y and room to spare
SENTINEL = 7.5                 # what a Y column holds before a call
COEFFS = (4.0, -1.4, -0.6, -1.2, -0.8, -0.3, -0.7)
TALL = 1300                    # rows of a 1536-nonzero tile that reads its row pointers from global memory (> 1024)
# CTA c of the many-tiles matrix meets these tiles in this order
PROBES = {7: ("short", "long", "short"), 11: ("short", "tall", "short"), 13: ("long", "long", "tall")}


# ------------------------------------------------------------------ matrices (host) ----

def short_tile(rng, cap):
    """row lengths 1..11 of exactly `cap` nonzeros (the last row takes the rest, maybe 0)"""
    d = rng.integers(1, 12, 2 * cap)
    c = np.cumsum(d)
    m = int(np.searchsorted(c, cap, side="right"))
    return list(d[:m]) + [cap - (int(c[m - 1]) if m else 0)]


def many_tiles(sms, far=False, seed=5):
    """(rowptr, cols, vals, kinds, rowblk) of a greedy-partitioned matrix of 3 G + 5 tiles, G = 3 sms: short tiles of
    exactly 1536 nonzeros whose first row is never empty (so each ends where it was built), long rows (1537 .. 3999)
    and tall tiles (TALL rows, 1536 nonzeros) where PROBES puts them, a ragged last tile of 700.  Columns near the
    diagonal (16-bit tile offsets) or, far=True, anywhere; standard normal values."""
    G = 3 * sms
    kinds = ["short"] * (3 * G + 5)
    for c, ks in PROBES.items():
        for j, k in enumerate(ks):
            kinds[c + j * G] = k
    kinds[-1] = "ragged"
    rng = np.random.default_rng(seed)
    lens, rowblk = [], [0]
    for k in kinds:
        if k == "long":
            lens.append(int(rng.integers(R.SP_NNZ + 1, 4000)))
        elif k == "tall":
            t = np.ones(TALL, np.int64)
            t[rng.choice(TALL, R.SP_NNZ - TALL, replace=False)] = 2
            lens.extend(t.tolist())
        else:
            lens.extend(short_tile(rng, R.SP_NNZ if k == "short" else 700))
        rowblk.append(len(lens))
    lens = np.array(lens, np.int64)
    n, rowptr = len(lens), np.r_[0, np.cumsum(lens)]
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, n, rowptr[-1]) if far else np.clip(rows + rng.integers(-400, 401, rowptr[-1]), 0, n - 1)
    return rowptr, cols, rng.standard_normal(rowptr[-1]), kinds, np.array(rowblk, np.int64)


def regular(maxrow, n=20000):
    """nnz-balanced partition at maxrow 768, greedy at 769"""
    rng = np.random.default_rng(maxrow)
    lens = rng.integers(0, 12, n)
    lens[[5, 9000]] = maxrow
    rowptr = np.r_[0, np.cumsum(lens)]
    return rowptr, rng.integers(0, n, rowptr[-1]), rng.standard_normal(rowptr[-1])


def tiny(n=200):
    rng = np.random.default_rng(n)
    lens = rng.integers(0, 9, n)
    rowptr = np.r_[0, np.cumsum(lens)]
    return rowptr, rng.integers(0, n, rowptr[-1]), rng.standard_normal(rowptr[-1])


def edge_arrays():
    A = edge_matrix()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64), A.data.copy()


def specials():
    """rows of 0..8 nonzeros around three long rows (1600, 2000, 1537 at rows 3, 10, 17)"""
    n = 6000
    rng = np.random.default_rng(77)
    lens = rng.integers(0, 9, n)
    lens[[3, 10, 17]] = [1600, 2000, 1537]
    rowptr = np.r_[0, np.cumsum(lens)]
    return rowptr, rng.integers(0, n, rowptr[-1]), rng.standard_normal(rowptr[-1])


def f32_exact(vals):
    return vals.astype(f32).astype(f64)


def long_refs(host, x, dt, kernel_name):
    """{row: y_row} of the rows of more than 1536 nonzeros as `kernel_name` sums them"""
    rowptr, cols, vals = host
    out = {}
    with np.errstate(all="ignore"):
        for r in np.flatnonzero(np.diff(rowptr) > R.SP_NNZ):
            a, b = rowptr[r], rowptr[r + 1]
            prod = vals[a:b] * np.asarray(x, dt)[cols[a:b]]
            out[int(r)] = dt(R.cta_reduce(R.strided_sums(prod.astype(f64)), kernel_name))
    return out


def diff_rows(got, want):
    ng, nw = np.isnan(got), np.isnan(want)
    eq = (ng & nw) | (~ng & ~nw & (got.view(np.uint8).reshape(len(got), -1) ==
                                   want.view(np.uint8).reshape(len(want), -1)).all(axis=1))
    return np.flatnonzero(~eq)


def check(got, want, what):
    if not same(got, want):
        bad = diff_rows(np.asarray(got), np.asarray(want))
        raise AssertionError(f"{what}: {bad.size} rows differ, e.g. rows {bad[:8]}: got {got[bad[:4]]}, "
                             f"want {want[bad[:4]]}")


# ------------------------------------------------------------------ device set-ups ----

class Setup:
    """one square CSR operator in a context of NCOLS columns, with a pool of X vectors and their restated A X"""

    def __init__(self, rowptr, cols, vals, dt, fmt=None, pool=24, seed=3):
        n = len(rowptr) - 1
        self.dt, self.n = dt, n
        self.host = (np.asarray(rowptr, np.int64), np.asarray(cols, np.int64), np.asarray(vals).astype(dt))
        self.ctx = kk.B200Context(n, NCOLS, dtype=dt)
        self.op = kk.B200CSR.from_csr_arrays(self.ctx, n, n, *self.host)
        self.rowblk = R.tiles(rowptr)
        assert np.array_equal(device_tiles(self.op), self.rowblk)
        if fmt is not None:
            assert L.load().b2k_debug_csr_format(self.op.h) == fmt
        rng = np.random.default_rng(seed)
        self.xh = []
        for _ in range(pool):
            x = rng.standard_normal(n).astype(dt)
            x[rng.integers(0, n, n // 50)] = -0.0
            self.xh.append(x)
        self.X = [self.ctx.from_host(x) for x in self.xh]
        self._ref = {}

    def ref(self, i):
        if i not in self._ref:
            self._ref[i] = R.csr_rows(*self.host, self.xh[i], self.dt, None, "pipe")
        return self._ref[i]

    def fresh(self, p, space=0):
        Y = [self.ctx.empty(space) for _ in range(p)]
        for y in Y:
            y.upload(np.full(len(y), SENTINEL, self.dt))
        return Y


def block(ctx, op, X, Y, p=None):
    return ctx.lib.b2k_op_apply_block(ctx.h, op.h, handles(X), handles(Y), len(X) if p is None else p)


F32V_I16, F32V_ONLY, I16_ONLY = 4 | 1 | 2, 4 | 1, 4 | 2       # b2k_debug_csr_format of the compact instances


def make_setup(name, dt):
    if name.startswith("many"):
        far = name == "many-dfi32"
        rowptr, cols, vals, _, _ = many_tiles(num_sms(), far=far)
        if name != "many":
            vals = f32_exact(vals)
        fmt = {"many": I16_ONLY, "many-dfi16": F32V_I16, "many-dfi32": F32V_ONLY}[name]
        return Setup(rowptr, cols, vals, dt, fmt if dt == f64 else I16_ONLY)
    if name.startswith("edge"):
        rowptr, cols, vals = edge_arrays()
        if name == "edge-dfi16":
            vals = f32_exact(vals)
        return Setup(rowptr, cols, vals, dt, (F32V_I16 if name == "edge-dfi16" else I16_ONLY) if dt == f64
                     else I16_ONLY)
    raise KeyError(name)


@pytest.fixture(scope="module")
def setups():
    made = {}

    def get(name, dt):
        key = (name, np.dtype(dt).name)
        if key not in made:
            made[key] = make_setup(name, dt)
        return made[key]

    yield get
    for s in made.values():
        s.ctx.close()


def run_and_check(s, idx, Y=None):
    """SpMM of the pool vectors idx into Y (fresh if None) against the restatement; returns Y"""
    p = len(idx)
    X = [s.X[i] for i in idx]
    Y = s.fresh(p) if Y is None else Y
    with profiled(s.ctx) as cnt:
        s.ctx.check(block(s.ctx, s.op, X, Y))
    assert cnt[SPMM] == -(-p // 8) and cnt[SPMV] == 0, cnt
    for j, i in enumerate(idx):
        check(Y[j].to_host(), s.ref(i), f"vector {j} of {p}")
    return Y


def free(vs):
    for v in vs:
        v.free()


# ------------------------------------------------------------------ CPU: the restatement and the layout ----

def test_many_tiles_layout_gives_every_cta_three_tiles_or_more():
    """for an H100's 132 SMs: 3 G + 5 tiles on G = 396 CTAs, the probes where PROBES says, a ragged last tile, and
    finish_csr's greedy partition (as restated) cuts the tiles where the builder did"""
    rowptr, cols, vals, kinds, rowblk = many_tiles(SM_H100)
    G, nblk = 3 * SM_H100, len(rowblk) - 1
    assert np.array_equal(R.tiles(rowptr), rowblk)
    assert nblk >= 3 * G + 1 and min(nblk, 3 * SM_H100) == G
    per_cta = np.bincount(np.arange(nblk) % G, minlength=G)
    assert per_cta.min() >= 3 and per_cta.max() == 4
    tnnz, trows = np.diff(rowptr[rowblk]), np.diff(rowblk)
    kind = np.where(tnnz > R.SP_NNZ, "long", np.where(trows > 1024, "tall", "short"))
    for c, ks in PROBES.items():
        assert tuple(kind[c::G][:3]) == ks, (c, kind[c::G])
    assert tnnz[-1] < R.SP_NNZ and np.all(tnnz[kind != "long"] <= R.SP_NNZ)
    assert np.all(trows[kind == "long"] == 1) and np.all(trows <= R.SP_ROWS)
    assert 1_700_000 < rowptr[-1] < 2_000_000
    assert np.abs(cols - np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr)))[
        np.repeat(kind != "long", tnnz)].max() <= 400


@pytest.mark.parametrize("dt", DTS, ids=DIDS)
def test_restated_rows_are_exact_on_small_integers(dt):
    """with small integers every order is exact: the restated rows of the many-tiles matrix (long rows included) and
    of the edge matrix are A x"""
    import scipy.sparse as sp
    rng = np.random.default_rng(2)
    for rowptr, cols, _ in (many_tiles(SM_H100)[:3], edge_arrays()):
        n = len(rowptr) - 1
        vals = rng.integers(-3, 4, rowptr[-1]).astype(dt)
        x = rng.integers(-3, 4, n).astype(dt)
        A = sp.csr_matrix((vals.astype(f64), cols, rowptr), shape=(n, n))
        y = R.csr_rows(rowptr, cols, vals, x, dt, None, "pipe")
        assert y.dtype == dt and np.array_equal(y.astype(f64), A @ x.astype(f64))


def test_long_rows_in_warp_order_are_not_block_sum():
    """the long-row restatement the SpMM is held to (warps in order) and the streaming kernel's (block_sum) give
    different doubles on a constructed row, so a test that names one cannot pass with the other"""
    big = 1e16
    prod = np.zeros(2000)
    prod[[0, 32, 64, 96]] = [big, 1.0, -big, 1.0]     # one term in each of the first four warps' lanes 0
    rowptr, cols = np.array([0, 2000]), np.arange(2000)
    got = R.csr_rows(rowptr, cols, prod, np.ones(2000), f64, None, "pipe")[0]
    assert got == 1.0 and long_refs((rowptr, cols, prod), np.ones(2000), f64, "stream")[0] == 2.0


# ------------------------------------------------------------------ 1. group sizes ----

GROUPS = [2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 24]


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
@pytest.mark.parametrize("p", GROUPS)
def test_group_sizes_on_many_tiles_per_cta(setups, p, dt):
    """every group width 1..8 (tails of 1 at p = 9, 17), both parities of the last product buffer, 1 to 3 launches"""
    s = setups("many", dt)
    free(run_and_check(s, list(range(p))))


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
def test_many_tiles_layout_on_the_device(setups, dt):
    """the device's tiles and grid give the layout the docstring claims"""
    s = setups("many", dt)
    G, nblk = min(len(s.rowblk) - 1, 3 * num_sms()), len(s.rowblk) - 1
    assert nblk >= 3 * G + 1
    rowptr = s.host[0]
    tnnz, trows = np.diff(rowptr[s.rowblk]), np.diff(s.rowblk)
    kind = np.where(tnnz > R.SP_NNZ, "long", np.where(trows > 1024, "tall", "short"))
    for c, ks in PROBES.items():
        assert tuple(kind[c::G][:3]) == ks
    assert tnnz[-1] < R.SP_NNZ


# ------------------------------------------------------------------ 2. matrices ----

def matrix_arrays(name):
    if name == "edge":
        return edge_arrays()
    if name in ("maxrow768", "maxrow769"):
        return regular(int(name[-3:]))
    if name == "tiny":
        return tiny()
    if name == "empty":
        return np.zeros(3001, np.int64), np.zeros(0, np.int64), np.zeros(0)
    raise KeyError(name)


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
@pytest.mark.parametrize("name", ["edge", "maxrow768", "maxrow769", "tiny", "empty"])
def test_matrices(name, dt):
    """rows of 1536 / 1537 / 3000 and empty runs past a tile's rows; both finish_csr rules; one tile; no nonzeros"""
    rowptr, cols, vals = matrix_arrays(name)
    s = Setup(rowptr, cols, vals, dt, pool=9)
    nblk = len(s.rowblk) - 1
    lens = np.diff(rowptr)
    if name == "maxrow768":
        assert lens.max() == 768 and nblk == -(-rowptr[-1] // (R.SP_NNZ - 768 + 1))
    if name == "maxrow769":
        assert lens.max() == 769 and np.all(np.diff(rowptr[s.rowblk]) <= R.SP_NNZ)
    if name == "tiny":
        assert s.n < 256 and nblk == 1
    if name == "empty":
        assert nblk == 1 and s.n > 2048
        for x in s.X[:3]:                                   # non-finite operands change nothing
            x.upload(np.full(s.n, np.nan, dt))
    Y = run_and_check(s, list(range(9)))
    if name == "empty":
        for y in Y:
            assert same(y.to_host(), np.zeros(s.n, dt))     # +0, not the sentinel, not -0
    s.ctx.close()


# ------------------------------------------------------------------ 3. values ----

@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
def test_special_values(dt):
    """Inf in A against 0 in x and 0 in A against Inf in x (NaN), NaN in x, rows of -0 products (+0: the sums start at
    +0), Float64 values that are not exact in Float32, Float32 products in the subnormal range (the build does not flush
    them) — in short and in long rows"""
    rowptr, cols, vals = specials()
    n = len(rowptr) - 1
    lens = np.diff(rowptr)
    rows = np.repeat(np.arange(n), lens)
    rng = np.random.default_rng(8)
    xs = [rng.standard_normal(n) for _ in range(5)]
    # X0: A has +Inf / -Inf in column ca (the long row 10 among others), x0[ca] = 0
    counts = np.bincount(cols, minlength=n)
    ca = cols[rowptr[10]:rowptr[11]][np.argmax(counts[cols[rowptr[10]:rowptr[11]]])]     # in many rows
    vals[cols == ca] = np.where(rng.random(int((cols == ca).sum())) < 0.5, np.inf, -np.inf)
    xs[0][ca] = 0.0
    # X1: A has 0 in column cb (the long row 17 among others), x1[cb] = -Inf
    counts[ca] = -1
    cb = cols[rowptr[17]:rowptr[18]][np.argmax(counts[cols[rowptr[17]:rowptr[18]]])]
    vals[cols == cb] = 0.0
    xs[1][cb] = -np.inf
    # X2: NaN in x
    xs[2][cols[rowptr[3] + 1]] = np.nan
    xs[2][cols[rowptr[500]]] = np.nan
    # X3: rows 3 (long) and 40..60 hold products of -0 only: A's zeros signed against x3, x3 nonzero finite there
    zrows = np.r_[3, 40:61]
    zm = np.isin(rows, zrows)
    xs[3][cols[zm]] = np.where(xs[3][cols[zm]] == 0, 1.0, xs[3][cols[zm]])
    # X4: tiny x (2^-70) against tiny A in rows 17 (long) and 100..400: 2^-140-ish products, subnormal in Float32
    xs[4] = xs[4] * 2.0 ** -70
    tm = np.isin(rows, np.r_[17, 100:401])
    vals[tm] *= 2.0 ** -70
    vals = vals.astype(dt)
    vals[zm] = np.where(np.asarray(xs[3], dt)[cols[zm]] > 0, -0.0, 0.0).astype(dt)
    s = Setup(rowptr, cols, vals, dt, pool=5)
    for i, x in enumerate(xs):
        s.xh[i] = np.asarray(x, dt)
        s.X[i].upload(s.xh[i])
    with np.errstate(all="ignore"):
        p4 = vals * s.xh[4][cols]
        p3 = vals * s.xh[3][cols]
    if dt == f32:                                           # the products really are subnormal
        sub = (p4 != 0) & (np.abs(p4) < np.finfo(f32).tiny)
        assert sub[tm].sum() > 1000 and sub[rowptr[17]:rowptr[18]].sum() > 1000
    else:
        assert np.any(vals.astype(f32).astype(f64) != vals)
    assert np.all(np.signbit(p3[zm]) & (p3[zm] == 0))
    Y = run_and_check(s, list(range(5)))
    y = [v.to_host() for v in Y]
    assert np.isnan(y[0][10]) and np.isnan(y[1][17]) and np.isnan(y[2][3])
    assert np.isnan(y[0]).sum() > 3 and np.isnan(y[1]).sum() > 3
    assert np.all((y[3][zrows] == 0) & ~np.signbit(y[3][zrows]))
    if dt == f32:
        assert np.any((y[4] != 0) & (np.abs(y[4]) < np.finfo(f32).tiny))
    s.ctx.close()


# ------------------------------------------------------------------ 4. column layouts ----

LAYOUTS = ["contiguous", "interleaved", "reversed", "y_first", "scattered"]


def layout(name, p, ncols):
    """(X columns, Y columns) in one slab of ncols columns"""
    a, b = list(range(p)), list(range(p, 2 * p))
    if name == "contiguous":
        return a, b
    if name == "interleaved":
        return list(range(0, 2 * p, 2)), list(range(1, 2 * p, 2))
    if name == "reversed":
        return a[::-1], b[::-1]
    if name == "y_first":
        return b, a
    perm = np.random.default_rng(p).permutation(ncols)[:2 * p].tolist()
    return perm[:p], perm[p:]


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
@pytest.mark.parametrize("name", LAYOUTS)
def test_column_layouts(name, dt):
    """X and Y anywhere in one slab: Y right, every other column (X included) untouched, a second call the same bits"""
    rowptr, cols, vals = edge_arrays()
    n, p, ncols = len(rowptr) - 1, 9, 23
    ctx = kk.B200Context(n, ncols, dtype=dt)
    op = kk.B200CSR.from_csr_arrays(ctx, n, n, rowptr, cols, vals.astype(dt))
    V = [ctx.empty() for _ in range(ncols)]
    assert [v.handle & 0xFFFFF for v in V] == list(range(ncols))
    rng = np.random.default_rng(ncols)
    data = [rng.standard_normal(n).astype(dt) for _ in range(ncols)]
    for v, d in zip(V, data):
        v.upload(d)
    xc, yc = layout(name, p, ncols)
    X, Y = [V[c] for c in xc], [V[c] for c in yc]
    host = (rowptr, cols, vals.astype(dt))
    want = [R.csr_rows(*host, data[c], dt, None, "pipe") for c in xc]
    for call in range(2):
        with profiled(ctx) as cnt:
            ctx.check(block(ctx, op, X, Y))
        assert cnt[SPMM] == 2 and cnt[SPMV] == 0
        for c in range(ncols):
            got = V[c].to_host()
            if c in yc:
                check(got, want[yc.index(c)], f"call {call}: Y column {c}")
            else:
                check(got, data[c], f"call {call}: column {c} is not in Y")
    ctx.close()


# ------------------------------------------------------------------ 5. same bits as single applies ----

SINGLE = [("edge", f64, "c_ddi16"), ("edge", f32, "c_ffi16"), ("edge-dfi16", f64, "c_dfi16"),
          ("many", f64, "c_ddi16"), ("many", f32, "c_ffi16"), ("many-dfi16", f64, "c_dfi16"),
          ("many-dfi32", f64, "c_dfi32")]


@gpu
@pytest.mark.parametrize("name,dt,inst", SINGLE, ids=[f"{m}-{np.dtype(d).name}" for m, d, _ in SINGLE])
def test_same_bits_as_single_applies(setups, name, dt, inst):
    """SpMM of 10 vectors against 10 applies under k_spmv_stream, k_spmv_pipe (both variants) and the compact instance
    the matrix takes.  Stream's long rows (block_sum) are held to their own restatement, SpMM's to k_spmv_pipe's."""
    s = setups(name, dt)
    p = 10
    idx = list(range(p))
    Y = run_and_check(s, idx)
    yh = [y.to_host() for y in Y]
    lens = np.diff(s.host[0])
    short = lens <= R.SP_NNZ
    assert (~short).sum() >= 2
    Z = s.fresh(p)
    for kname in ("stream", "pipe24", "pipe33", "compact"):
        with kernel(kname):
            for i in idx:
                s.op.apply_into(Z[i], s.X[i])
                rec = launch()
                want_k = {"stream": STREAM, "compact": COMPACT}.get(kname, PIPE)
                assert rec[0] == want_k, (kname, rec)
                if kname == "compact":
                    assert rec[1] == COMPACT_INST[inst]
        for i in idx:
            z = Z[i].to_host()
            if kname != "stream":
                check(z, yh[i], f"{kname}: vector {i}")
                continue
            check(z[short], yh[i][short], f"stream, rows of <= 1536 nonzeros: vector {i}")
            for r, v in long_refs(s.host, s.xh[i], dt, "stream").items():
                assert same(z[r], v), (r, z[r], v)
    free(Y + Z)


# ------------------------------------------------------------------ 6. fallbacks ----

@contextlib.contextmanager
def block_kernels(on):
    """B2K_BLOCK_KERNELS for the contexts created inside.  b2k_block_init copies the variable into a process-wide flag
    at every context creation, but only when it is set: the exit sets it back to 1 and creates a context before
    restoring the environment."""
    saved = os.environ.get("B2K_BLOCK_KERNELS")
    os.environ["B2K_BLOCK_KERNELS"] = "1" if on else "0"
    try:
        yield
    finally:
        os.environ["B2K_BLOCK_KERNELS"] = "1"
        kk.B200Context(8, 2).close()
        if saved is None:
            del os.environ["B2K_BLOCK_KERNELS"]
        else:
            os.environ["B2K_BLOCK_KERNELS"] = saved


@contextlib.contextmanager
def spmv_pipe_off():
    lib = L.load()
    lib.b2k_debug_set_spmv_pipe(0)
    try:
        yield
    finally:
        lib.b2k_debug_set_spmv_pipe(1)


FALLBACKS = ["p1", "two_spaces", "rectangular", "stencil", "spmv_pipe_off", "block_kernels_off"]


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallback_to_single_applies(case, dt):
    """each case runs p single applies and no SpMM, and gives the restated rows"""
    rng = np.random.default_rng(31)
    p, kname, xspace, yspace = 3, "pipe", 0, 0
    env = block_kernels(False) if case == "block_kernels_off" else contextlib.nullcontext()
    with env:
        if case == "stencil":
            dims = (41, 23, 7)
            n = m = int(np.prod(dims))
            ctx = kk.B200Context(n, 12, dtype=dt)
            op = kk.B200CSR.stencil_free(ctx, *dims, coeffs=COEFFS)
        else:
            rowptr, cols, vals = edge_arrays()
            m = len(rowptr) - 1
            n = m + 777 if case == "rectangular" else m
            if case == "rectangular":
                cols = cols + rng.integers(0, 778, len(cols))          # columns past m
            ctx = kk.B200Context(m, 12, dtype=dt)
            if case in ("rectangular", "two_spaces"):
                xspace = ctx.add_space(n, 8)
            op = kk.B200CSR.from_csr_arrays(ctx, m, n, rowptr, cols, vals.astype(dt))
            host = (rowptr, cols, vals.astype(dt))
        if case == "p1":
            p = 1
        if case == "spmv_pipe_off":
            kname = "stream"
        xh = [rng.standard_normal(n).astype(dt) for _ in range(p)]
        X = [ctx.from_host(x, xspace) for x in xh]
        Y = [ctx.from_host(np.full(m, SENTINEL, dt), yspace) for _ in range(p)]
        with spmv_pipe_off() if case == "spmv_pipe_off" else contextlib.nullcontext():
            with profiled(ctx) as cnt:
                ctx.check(block(ctx, op, X, Y))
        assert cnt[SPMV] == p and cnt[SPMM] == 0, cnt
        for i in range(p):
            if case == "stencil":
                want = R.stencil_rows(*dims, COEFFS, xh[i], dt, None)
            else:
                want = R.csr_rows(*host, xh[i], dt, None, kname)
            check(Y[i].to_host(), want, f"{case}: vector {i}")
        ctx.close()


# ------------------------------------------------------------------ 7. refusals and odd inputs ----

@gpu
def test_refusals_write_nothing():
    """p = 0, Y aliasing X, X or Y spanning two spaces: refused, nothing launched, no column changed"""
    rowptr, cols, vals = edge_arrays()
    n, p = len(rowptr) - 1, 4
    ctx = kk.B200Context(n, 16)
    sp1 = ctx.add_space(n, 4)
    op = kk.B200CSR.from_csr_arrays(ctx, n, n, rowptr, cols, vals)
    rng = np.random.default_rng(4)
    X = [ctx.from_host(rng.standard_normal(n)) for _ in range(p)]
    Y = [ctx.from_host(np.full(n, SENTINEL)) for _ in range(p)]
    other = ctx.from_host(rng.standard_normal(n), sp1)
    before = [v.to_host() for v in X + Y + [other]]
    cases = [(X, Y, 0, L.EINVAL), (X, Y, -1, L.EINVAL), (X, [Y[0], X[2], Y[2], Y[3]], p, L.EINVAL),
             (X, [Y[0], Y[1], Y[2], X[0]], p, L.EINVAL), ([X[0], X[1], other, X[3]], Y, p, L.EDIM),
             (X, [Y[0], other, Y[2], Y[3]], p, L.EDIM)]
    for Xc, Yc, pc, code in cases:
        with profiled(ctx) as cnt:
            assert block(ctx, op, Xc, Yc, pc) == code
        assert cnt[SPMM] == 0 and cnt[SPMV] == 0
        for v, b in zip(X + Y + [other], before):
            assert same(v.to_host(), b)
    ctx.close()


@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
def test_repeated_y_the_later_vector_wins(setups, dt):
    """Y[1] = Y[8] (two launches) and Y[3] = Y[4] (one launch): what the loop of applies leaves"""
    s = setups("edge", dt)
    p = 9
    Yd = s.fresh(7)
    Y = [Yd[0], Yd[1], Yd[2], Yd[3], Yd[3], Yd[4], Yd[5], Yd[6], Yd[1]]
    X = s.X[:p]
    with profiled(s.ctx) as cnt:
        s.ctx.check(block(s.ctx, s.op, X, Y))
    assert cnt[SPMM] == 2 and cnt[SPMV] == 0
    got = {y.handle: y.to_host() for y in Yd}
    last = {Y[i].handle: i for i in range(p)}
    for h, i in last.items():
        check(got[h], s.ref(i), f"column of Y[{i}]")
    Z = s.fresh(7)
    W = [Z[0], Z[1], Z[2], Z[3], Z[3], Z[4], Z[5], Z[6], Z[1]]
    for x, w in zip(X, W):
        s.op.apply_into(w, x)
    for y, z in zip(Yd, Z):
        check(z.to_host(), got[y.handle], "the loop of applies")
    free(Yd + Z)


# ------------------------------------------------------------------ 8. the Python wrapper ----

@gpu
@pytest.mark.parametrize("dt", DTS, ids=DIDS)
def test_blocklanczos_apply_block_is_the_c_call(setups, dt):
    s = setups("edge", dt)
    p = 11
    X = s.X[:p]
    with profiled(s.ctx) as cnt:
        B = bl._apply_block(s.op, kk.Block(X))
    assert cnt[SPMM] == 2 and cnt[SPMV] == 0 and len(B) == p
    Y = run_and_check(s, list(range(p)))
    for i in range(p):
        check(B[i].to_host(), Y[i].to_host(), f"vector {i}")
        check(B[i].to_host(), s.ref(i), f"vector {i}")
    free(Y + B.vec)
