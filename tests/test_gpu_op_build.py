"""GPU tests of the kernels that build operator data on the device, bit for bit, in Float64 and Float32.  The iteration
tests check every kernel against the data it is given; these check that data.

A. The device CSR transpose (b2k_op_create_transpose: k_iota, a CUB radix sort of the column keys over bits
   [0, end_bit) with end_bit the smallest e >= 1 with 2^e >= n_cols, k_transpose_gather, k_transpose_rowptr) against
   `transpose_restated`: the nonzeros of A stably sorted by column, so within a column in CSR(A) order, each one's
   row in A its column in A', and row c of A' starting at the first sorted nonzero of column >= c.  The cases put
   n_cols at every end_bit and 8-bit radix-digit edge up to 2^24 + 1 with columns 0 and n_cols - 1 occupied, take
   nnz from 1 to 3.1e7 (CUB's single-tile path up to its multi-pass onesweep path), a column of more than 2^16
   entries from rows spread over the whole matrix, empty leading and trailing rows and columns, one row, and rows
   with unsorted and repeated columns (CSR ingestion keeps them as stored).  The index forms int32 / int64 with base
   0 / 1 rotate over the cases.  For each case A'' is checked too (A itself when its rows are sorted without
   repeats, else the restatement applied twice: every row stably sorted by column), the tiles and compact view of A'
   against those of A' built from the host arrays, and one SpMV with each, bit for bit.
B. The pencil's pattern check (b2k_pencil_create, k_pattern_diff over rowptr then colidx).  Pairs with equal nnz
   whose patterns differ in one colidx entry (index 0, the last index, an index past the first grid-stride sweep of
   4·SMs·256 entries) or only in rowptr (a nonzero moved across a row boundary) must take the composed path (0),
   with w, bx, A x and the dots as spmv_restated, libm's fma and b2k_vec_inner give them.  Pairs of one pattern
   that reach the device by different routes (CSC and CSR ingestion, A'' and A, an assembled stencil and its host
   CSR, a Float32-exact compact value stream and a plain one, two empty matrices) must take the fused path (1), with
   the same vectors and the dots of k_spmv_pipe's order at the pencil's grid.
C. The splitmix dense fill (k_dense_fill_splitmix) against oracle.krylov_oracle.dense_splitmix: column j as A e_j and
   row i as A' e_i (every other term a product with zero, so both are exact), and the padding rows [m, ld) zero
   through b2k_op_apply_normal_gram, whose z = A'(A e_j) is restated by oracle/onepass_restate.py on A padded with
   zero rows.

The CPU tests check the restatements at tiny sizes against per-entry loops, and that the transpose cases would catch
an unstable sort and an end_bit one too small.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.operators import apply_adjoint, apply_normal_gram
from oracle import krylov_oracle as ko
from oracle import onepass_restate as rs
import op_ingest_cases as K
import spmv_restate as R
from test_gpu_blas1 import fma, num_sms  # noqa: F401  (fma: module fixture)
from test_gpu_pencil import SHAPES, device_tiles, random_pattern, shape, spmv_restated, with_values

gpu = pytest.mark.gpu
f64, f32 = np.float64, np.float32
DTS = [pytest.param(f64, id="f64"), pytest.param(f32, id="f32")]
SEED = 20261019


def bits(a):
    a = np.asarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


# ================================================================ A. transpose ====

def end_bit(n_cols):
    """the key bits b2k_op_create_transpose sorts on: the smallest e >= 1 with 2^e >= n_cols"""
    e = 1
    while e < 32 and (1 << e) < n_cols:
        e += 1
    return e


def radix_sort(bits_):
    """a stable sort on the low `bits_` bits of the keys only, as CUB's DeviceRadixSort with end_bit = bits_"""
    return lambda keys: np.argsort(keys & ((1 << bits_) - 1), kind="stable")


def stable_sort(keys):
    """np.argsort(kind="stable") in two 16-bit passes (numpy's radix sort): the same permutation, in O(nnz)"""
    p = np.argsort((keys & 0xFFFF).astype(np.uint16), kind="stable")
    return p[np.argsort((keys[p] >> 16).astype(np.uint16), kind="stable")]


def unstable_sort(keys):
    """a negative control: sorted by key, equal keys in reverse order"""
    return np.lexsort((-np.arange(len(keys)), keys))


def transpose_restated(rowptr, colidx, vals, n_cols, sort=stable_sort):
    """(rowptr, colidx, vals) of A' as b2k_op_create_transpose builds it from CSR(A), with `sort` for the sort"""
    rowptr = np.asarray(rowptr, np.int64)
    colidx = np.asarray(colidx, np.int64)
    perm = sort(colidx)
    rows = np.repeat(np.arange(len(rowptr) - 1, dtype=np.int64), np.diff(rowptr))
    trowptr = np.searchsorted(colidx[perm], np.arange(n_cols + 1), side="left")
    return trowptr.astype(np.int32), rows[perm].astype(np.int32), np.asarray(vals)[perm]


def transpose_loops(rowptr, colidx, vals, n_cols):
    """the same, entry by entry: every nonzero appended to its column's list in CSR order"""
    lists = [[] for _ in range(n_cols)]
    for r in range(len(rowptr) - 1):
        for k in range(rowptr[r], rowptr[r + 1]):
            lists[colidx[k]].append((r, vals[k]))
    trp = np.cumsum([0] + [len(li) for li in lists]).astype(np.int32)
    tci = np.array([r for li in lists for r, _ in li], dtype=np.int32)
    tva = np.array([v for li in lists for _, v in li], dtype=np.asarray(vals).dtype)
    return trp, tci, tva


class Case:
    def __init__(self, name, n_rows, n_cols, rowptr, colidx, sorted_rows):
        self.name, self.n_rows, self.n_cols, self.sorted_rows = name, n_rows, n_cols, sorted_rows
        self.rowptr, self.colidx = np.asarray(rowptr, np.int64), np.asarray(colidx, np.int64)
        self.nnz = len(self.colidx)


def from_pairs(rows, cols, n_rows, n_cols):
    """sorted rows without repeats from (row, col) pairs"""
    key = np.unique(np.asarray(rows, np.int64) * n_cols + np.asarray(cols, np.int64))
    r, c = key // n_cols, key % n_cols
    return np.concatenate(([0], np.cumsum(np.bincount(r, minlength=n_rows)))), c


def scattered(rng, n_rows, n_cols, nnz, rows=None, cols=None):
    """about nnz random entries in rows [r0, r1) and columns [c0, c1), plus (row 0, column 0) and (last row,
    column n_cols - 1) unless the ranges exclude them"""
    r0, r1 = rows or (0, n_rows)
    c0, c1 = cols or (0, n_cols)
    rr = rng.integers(r0, r1, nnz)
    cc = rng.integers(c0, c1, nnz)
    rr[:2], cc[:2] = (r0, r1 - 1), (c0, c1 - 1)
    return from_pairs(rr, cc, n_rows, n_cols)


def gapped(rng, n_rows, n_cols, per_row):
    """per_row sorted distinct columns in each row from random gaps, in O(nnz): row r's columns are running sums of
    gaps in [1, 2 n_cols / (per_row + 1)) from -1, those >= n_cols dropped; column 0 opens row 0, the last row ends at
    column n_cols - 1"""
    total = n_rows * per_row
    g = max(1, 2 * n_cols // (per_row + 1))
    gaps = rng.integers(1, g, total, dtype=np.int64) if g > 1 else np.ones(total, np.int64)
    gaps[0] = 1
    cs = np.cumsum(gaps)
    start = np.repeat(cs[::per_row] - gaps[::per_row], per_row)
    col = cs - start - 1
    row = np.repeat(np.arange(n_rows, dtype=np.int64), per_row)
    keep = col < n_cols
    row, col = row[keep], col[keep]
    last = np.flatnonzero(row == row[-1])
    col[last[-1]] = n_cols - 1
    return np.concatenate(([0], np.cumsum(np.bincount(row, minlength=n_rows)))), col


def unsorted_with_repeats(rng, n_rows, n_cols, nnz):
    """random columns in random order within each row, a tenth of the entries stored twice"""
    rr = np.sort(rng.integers(0, n_rows, nnz))
    cc = rng.integers(0, n_cols, nnz)
    rr[0], cc[0], rr[-1], cc[-1] = 0, 0, n_rows - 1, n_cols - 1
    rep = rng.choice(nnz, nnz // 10, replace=False)
    rr, cc = np.concatenate((rr, rr[rep])), np.concatenate((cc, cc[rep]))
    order = np.argsort(rr, kind="stable")
    rr, cc = rr[order], cc[order]
    return np.concatenate(([0], np.cumsum(np.bincount(rr, minlength=n_rows)))), cc


EDGE_COLS = [1, 2, 255, 256, 257, 511, 512, 513, 65535, 65536, 65537, (1 << 24) - 1, 1 << 24, (1 << 24) + 1]
LONG_COL = 70_001                  # entries of the long column: more than 2^16
CASES = ([f"cols-{n}" for n in EDGE_COLS] + [f"nnz-{k}" for k in (1, 2, 3, 700, 5000, 200_000, 2_000_000)]
         + ["nnz-31M", "long-column", "empty-edges", "one-row", "one-row-one-col", "unsorted-repeats",
            "unsorted-repeats-big"])
FORMS = [(np.int32, 0), (np.int64, 1), (np.int32, 1), (np.int64, 0)]
_CASES = {}


def case(name):
    """the matrix of a case (cached: the big ones are shared by both types)"""
    if name in _CASES:
        return _CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    sorted_rows = True
    if name.startswith("cols-"):
        n_cols = int(name[5:])
        n_rows = 3001
        rp, ci = scattered(rng, n_rows, n_cols, min(20_000, n_rows * n_cols // 2))
    elif name == "nnz-31M":          # 2^21 + 3 rows of 15 columns in 2^24 + 1: four radix passes over 3.1e7 keys
        n_rows, n_cols = (1 << 21) + 3, (1 << 24) + 1
        rp, ci = gapped(rng, n_rows, n_cols, 15)
    elif name.startswith("nnz-"):
        k = int(name[4:])
        n_rows, n_cols = 20_011, 70_001
        if k == 1:                   # the one entry in the last column
            rp, ci = np.concatenate((np.zeros(n_rows, np.int64), [1])), np.array([n_cols - 1])
        else:
            rp, ci = scattered(rng, n_rows, n_cols, k)
    elif name == "long-column":      # column 4099 in 70 001 rows spread over all 2^17 + 7, plus 3 random per row
        n_rows, n_cols = (1 << 17) + 7, 9_001
        rr = np.concatenate((rng.integers(0, n_rows, 3 * n_rows), rng.choice(n_rows, LONG_COL, replace=False),
                             [0, n_rows - 1]))
        cc = np.concatenate((rng.integers(0, n_cols, 3 * n_rows), np.full(LONG_COL, 4099), [0, n_cols - 1]))
        rp, ci = from_pairs(rr, cc, n_rows, n_cols)
    elif name == "empty-edges":      # rows [0, 37) and [4963, 5000), columns [0, 300) and [5700, 6000) empty
        n_rows, n_cols = 5000, 6000
        rp, ci = scattered(rng, n_rows, n_cols, 30_000, rows=(37, 4963), cols=(300, 5700))
    elif name == "one-row":          # one row of 3000 > SP_NNZ nonzeros: 65 537 rows of at most one
        n_rows, n_cols = 1, 65537
        rp, ci = scattered(rng, n_rows, n_cols, 3000)
    elif name == "one-row-one-col":
        n_rows, n_cols = 1, 1
        rp, ci = np.array([0, 1]), np.array([0])
    elif name == "unsorted-repeats":
        n_rows, n_cols, sorted_rows = 4000, 3001, False
        rp, ci = unsorted_with_repeats(rng, n_rows, n_cols, 20_000)
    elif name == "unsorted-repeats-big":
        n_rows, n_cols, sorted_rows = (1 << 16) + 1, (1 << 16) + 1, False
        rp, ci = unsorted_with_repeats(rng, n_rows, n_cols, 1_000_000)
    else:
        raise ValueError(name)
    c = Case(name, n_rows, n_cols, rp, ci, sorted_rows)
    c.vals = rng.standard_normal(c.nnz)
    _CASES[name] = c
    return c


def arrays(op):
    return K.download(op)[1]


def tiles_and_format(op):
    return device_tiles(op), op.ctx.lib.b2k_debug_csr_format(op.h)


def same_arrays(got, want):
    return all(K.same(g, w) for g, w in zip(got, want))


def test_transpose_restatement_matches_loops():
    """tiny matrices: sorted, unsorted with repeats, empty rows and columns, no nonzeros"""
    rng = np.random.default_rng(SEED)
    mats = [scattered(rng, 7, 9, 20) + (7, 9), unsorted_with_repeats(rng, 6, 5, 25) + (6, 5),
            scattered(rng, 9, 11, 15, rows=(2, 7), cols=(3, 8)) + (9, 11), (np.zeros(5, np.int64), [], 4, 3),
            (np.array([0, 1]), np.array([0]), 1, 1)]
    for rp, ci, m, n in mats:
        ci = np.asarray(ci, np.int64)
        va = rng.standard_normal(len(ci))
        want = transpose_loops(rp, ci, va, n)
        assert same_arrays(transpose_restated(rp, ci, va, n), want)
        assert same_arrays(transpose_restated(rp, ci, va, n, radix_sort(end_bit(n))), want)
        assert same_arrays(transpose_restated(rp, ci, va, n, lambda k: np.argsort(k, kind="stable")), want)
        if len(ci) and np.all(np.diff(ci)[np.diff(np.repeat(np.arange(m), np.diff(rp))) == 0] > 0):
            T = sp.csr_matrix((va, ci, rp), shape=(m, n)).T.tocsr()
            T.sort_indices()
            assert same_arrays(want, (T.indptr.astype(np.int32), T.indices.astype(np.int32), T.data))


def test_end_bit_edges():
    assert [end_bit(n) for n in EDGE_COLS] == [1, 1, 8, 8, 9, 9, 9, 10, 16, 16, 17, 24, 24, 25]
    for n in EDGE_COLS:
        assert (n - 1) >> end_bit(n) == 0 and (n < 3 or (n - 1) >> (end_bit(n) - 1) != 0)


@pytest.mark.parametrize("name", [c for c in CASES if c != "nnz-31M"])
def test_transpose_cases_catch_a_bad_sort(name):
    """each case with a column of two or more entries tells the restatement from an unstable sort, and each n_cols
    edge case from 2 up tells it from a radix sort on end_bit - 1 bits (column n_cols - 1 then sorts among the low
    columns); the two-pass sort is np.argsort's stable one"""
    c = case(name)
    want = transpose_restated(c.rowptr, c.colidx, c.vals, c.n_cols)
    if c.nnz <= 2_000_000:
        assert same_arrays(want, transpose_restated(c.rowptr, c.colidx, c.vals, c.n_cols,
                                                     lambda k: np.argsort(k, kind="stable")))
    assert same_arrays(want, transpose_restated(c.rowptr, c.colidx, c.vals, c.n_cols, radix_sort(end_bit(c.n_cols))))
    if np.bincount(c.colidx, minlength=1).max(initial=0) >= 2:
        assert not same_arrays(want, transpose_restated(c.rowptr, c.colidx, c.vals, c.n_cols, unstable_sort))
    if name.startswith("cols-") and c.n_cols >= 2:
        assert not same_arrays(want, transpose_restated(c.rowptr, c.colidx, c.vals, c.n_cols,
                                                        radix_sort(end_bit(c.n_cols) - 1)))


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("name", CASES)
def test_transpose(name, dt):
    c = case(name)
    idx, base = FORMS[CASES.index(name) % len(FORMS)]
    va = c.vals.astype(dt)
    ctx = kk.B200Context(c.n_rows, 4, dtype=dt)
    try:
        sp_n = ctx.add_space(c.n_cols, 4) if c.n_cols != c.n_rows else 0
        A = kk.B200CSR.from_csr_arrays(ctx, c.n_rows, c.n_cols, (c.rowptr + base).astype(idx),
                                       (c.colidx + base).astype(idx), va, index_base=base)
        t = A.transpose()
        assert (t.n_rows, t.n_cols, t.nnz) == (c.n_cols, c.n_rows, c.nnz)
        want = transpose_restated(c.rowptr, c.colidx, va, c.n_cols)
        got = arrays(t)
        for g, w, what in zip(got, want, ("rowptr", "colidx", "vals")):
            assert K.same(g, w), what
        tt = t.transpose()
        if c.sorted_rows:
            assert same_arrays(arrays(tt), (c.rowptr.astype(np.int32), c.colidx.astype(np.int32), va))
            (tb2, fmt2), (tb, fmt) = tiles_and_format(tt), tiles_and_format(A)
            assert np.array_equal(tb2, tb) and fmt2 == fmt
        else:
            assert same_arrays(arrays(tt), transpose_restated(*want, c.n_rows))
        tt.free()
        # A' built from the host arrays: the same tiles, compact view and products
        th = kk.B200CSR.from_csr_arrays(ctx, c.n_cols, c.n_rows, *want)
        (tb_d, fmt_d), (tb_h, fmt_h) = tiles_and_format(t), tiles_and_format(th)
        assert np.array_equal(tb_d, tb_h) and fmt_d == fmt_h
        x = ctx.from_host(np.random.default_rng(c.n_rows).standard_normal(c.n_rows).astype(dt))
        y1, y2 = ctx.empty(sp_n), ctx.empty(sp_n)
        t.apply_into(y1, x)
        th.apply_into(y2, x)
        assert np.array_equal(bits(y1.to_host()), bits(y2.to_host()))
    finally:
        ctx.close()


# ================================================================ B. pencil pattern check ====

def sweep(nsm):
    """entries k_pattern_diff's grid covers in its first grid-stride sweep"""
    return 4 * nsm * 256


def csr(rowptr, colidx, vals, n):
    """a scipy CSR holding exactly these arrays (no sorting, no summing)"""
    return sp.csr_matrix((np.asarray(vals), np.asarray(colidx, np.int32), np.asarray(rowptr, np.int32)), shape=(n, n))


def differ(P, how, nsm):
    """a pattern with P's nnz that differs from P as named: one colidx entry (at index 0, the last index, or the first
    index of k_pattern_diff's second sweep), or rowptr only (the first nonzero of row r moved into row r - 1, for r = 1
    or the middle row)"""
    n = P.shape[0]
    rp, ci = P.indptr.astype(np.int64).copy(), P.indices.astype(np.int64).copy()
    if how.startswith("col-"):
        k = {"col-first": 0, "col-last": P.nnz - 1, "col-far": sweep(nsm)}[how]
        assert k < P.nnz
        ci[k] = (ci[k] + 1) % n
    else:
        r = 1 if how == "row-first" else n // 2 + 1
        assert 1 <= r < n and rp[r] < rp[r + 1]
        rp[r] += 1
    return csr(rp, ci, np.ones(P.nnz), n)


def smallest_pairs():
    """n = 2: equal nnz, patterns that differ in colidx only and in rowptr only"""
    A = csr([0, 1, 2], [0, 1], [1.0, 1.0], 2)
    return {"col": (A, csr([0, 1, 2], [1, 0], [1.0, 1.0], 2)), "row": (A, csr([0, 2, 2], [0, 1], [1.0, 1.0], 2))}


def test_pattern_pairs_differ_only_as_named():
    rng = np.random.default_rng(SEED + 1)
    P = random_pattern(rng, 3000, 5)
    for how in ("col-first", "col-last", "col-far", "row-first", "row-mid"):
        Q = differ(P, how, 2)
        assert Q.nnz == P.nnz and Q.indptr[-1] == P.nnz
        drp, dci = np.flatnonzero(Q.indptr != P.indptr), np.flatnonzero(Q.indices != P.indices)
        if how.startswith("col-"):
            assert len(drp) == 0 and list(dci) == [{"col-first": 0, "col-last": P.nnz - 1, "col-far": 2048}[how]]
        else:
            assert len(dci) == 0 and list(drp) == [1 if how == "row-first" else 1501]
    for A, B in smallest_pairs().values():
        assert A.nnz == B.nnz and not (np.array_equal(A.indptr, B.indptr) and np.array_equal(A.indices, B.indices))


def run_pencil(ctx, dA, dB, A, B, x, vp, fma, dt, path):
    """apply (with and without vprev, with the dot) and rayleigh: the path after each call, and w, bx, ax bit for bit
    against the restatement; returns the dots"""
    n = len(x)
    xd, vpd = ctx.from_host(x), ctx.from_host(vp)
    ax_ref, bx_ref = spmv_restated(A, x, dt), spmv_restated(B, x, dt)
    P = kk.B200Pencil(dA, dB)
    dots = {}
    for use_prev in (False, True):
        w, bx = ctx.from_host(np.full(n, np.nan, dt)), ctx.from_host(np.full(n, np.nan, dt))
        dots[use_prev] = P.apply_into(xd, w, bx, 0.37, vpd if use_prev else None, 0.61, dot=True)
        assert L.load().b2k_debug_pencil_path() == path
        wref = fma(-0.37, bx_ref, ax_ref, dt)
        if use_prev:
            wref = fma(-0.61, vp, wref, dt)
        assert np.array_equal(bits(bx.to_host()), bits(bx_ref))
        assert np.array_equal(bits(w.to_host()), bits(wref))
        if path == 0:
            assert dots[use_prev] == xd.inner(w)
        dots[use_prev] = (dots[use_prev], wref)
    ax, bx = ctx.from_host(np.full(n, np.nan, dt)), ctx.from_host(np.full(n, np.nan, dt))
    xax, xbx = P.rayleigh_into(xd, ax, bx)
    assert L.load().b2k_debug_pencil_path() == path
    assert np.array_equal(bits(ax.to_host()), bits(ax_ref)) and np.array_equal(bits(bx.to_host()), bits(bx_ref))
    if path == 0:
        assert xax == xd.inner(ax) and xbx == xd.inner(bx)
    P.free()
    return dots, (xax, ax_ref), (xbx, bx_ref)


DIFFS = ["col-first", "col-last", "row-first", "row-mid"]
DIFF_CASES = ([(s, h) for s in SHAPES if s != 1 for h in DIFFS] + [("millions", "col-far")]
              + [("n2", "col"), ("n2", "row")])
_PATS = {}


def pattern(name):
    if name not in _PATS:
        _PATS[name] = shape(name, np.random.default_rng(zlib.crc32(f"pat-{name}".encode())))
    return _PATS[name]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("name,how", DIFF_CASES, ids=[f"{s}-{h}" for s, h in DIFF_CASES])
def test_pattern_differs_takes_composed_path(fma, name, how, dt):
    rng = np.random.default_rng(zlib.crc32(f"{name}-{how}-{np.dtype(dt).name}".encode()))
    if name == "n2":
        A, B = smallest_pairs()[how]
        A, B = A.astype(dt), B.astype(dt)
        A.data[:], B.data[:] = (1.5, -2.25), (0.75, 3.5)
    else:
        P = pattern(name)
        A, _ = with_values(P, rng, dt)
        B = differ(P, how, num_sms())
        B.data = (rng.random(B.nnz) + 0.5).astype(dt)
    n = A.shape[0]
    assert A.nnz == B.nnz
    ctx = kk.B200Context(n, 16, dtype=dt)
    try:
        dA = kk.B200CSR.from_csr_arrays(ctx, n, n, A.indptr, A.indices, A.data)
        dB = kk.B200CSR.from_csr_arrays(ctx, n, n, B.indptr, B.indices, B.data)
        run_pencil(ctx, dA, dB, A, B, rng.standard_normal(n).astype(dt), rng.standard_normal(n).astype(dt), fma,
                   dt, 0)
    finally:
        ctx.close()


ROUTES = ["csc", "transpose-twice", "stencil", "compact-values", "empty", "empty-one"]


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("route", ROUTES)
def test_same_pattern_by_other_routes_takes_fused_path(fma, route, dt):
    rng = np.random.default_rng(zlib.crc32(f"route-{route}-{np.dtype(dt).name}".encode()))
    if route == "stencil":
        nx, ny, nz = 23, 17, 5
        cA, cB = (6.5, -1.25, -0.75, -1.5, -0.5, -1.125, -0.875), (2.0, 0.1, 0.2, 0.3, 0.15, 0.05, 0.25)
        A, B = (csr(*K.stencil_expected(nx, ny, nz, co, dt), nx * ny * nz) for co in (cA, cB))
    elif route in ("empty", "empty-one"):
        n = 1000 if route == "empty" else 1
        A = B = csr(np.zeros(n + 1), [], np.zeros(0, dt), n)
    else:
        A, B = with_values(random_pattern(rng, 3001, 5), rng, dt)
        if route == "compact-values":         # A's values Float32-exact (a compact value stream in Float64), B's not
            A.data = A.data.astype(f32).astype(dt)
    n = A.shape[0]
    ctx = kk.B200Context(n, 16, dtype=dt)
    try:
        if route == "stencil":
            dA = kk.B200CSR.stencil(ctx, nx, ny, nz, cA)
        elif route == "transpose-twice":
            dA = kk.B200CSR.from_csr_arrays(ctx, n, n, A.indptr, A.indices, A.data).transpose().transpose()
        else:
            dA = kk.B200CSR.from_csr_arrays(ctx, n, n, A.indptr, A.indices, A.data)
        if route == "csc":
            Bc = B.tocsc()
            dB = kk.B200CSR.from_julia_csc(ctx, n, n, Bc.indptr.astype(np.int64) + 1,
                                           Bc.indices.astype(np.int64) + 1, Bc.data)
        else:
            dB = kk.B200CSR.from_csr_arrays(ctx, n, n, B.indptr, B.indices, B.data)
        assert same_arrays(arrays(dA), (A.indptr, A.indices, A.data))
        assert same_arrays(arrays(dB), (B.indptr, B.indices, B.data))
        if route == "compact-values" and dt == f64:
            assert ctx.lib.b2k_debug_csr_format(dA.h) & 1 and not ctx.lib.b2k_debug_csr_format(dB.h) & 1
        x = rng.standard_normal(n).astype(dt)
        dots, (xax, ax_ref), (xbx, bx_ref) = run_pencil(ctx, dA, dB, A, B, x, rng.standard_normal(n).astype(dt),
                                                        fma, dt, 1)
        # the fused dots: k_spmv_pipe's order at the pencil's grid (3 CTAs per SM in Float64, 4 in Float32)
        rowblk = device_tiles(dA)
        grid = min(len(rowblk) - 1, (3 if dt == f64 else 4) * num_sms())
        gid, rank = R.csr_threads(rowblk, grid)
        for d, wref in dots.values():
            assert d == R.dot(fma, dt, x, wref, gid, rank, grid, "pipe")
        assert xax == R.dot(fma, dt, x, ax_ref, gid, rank, grid, "pipe")
        assert xbx == R.dot(fma, dt, x, bx_ref, gid, rank, grid, "pipe")
        if A.nnz == 0:
            assert xax == 0.0 and xbx == 0.0 and dots[False][0] == 0.0
    finally:
        ctx.close()


# ================================================================ C. splitmix dense fill ====

def onepass_launch():
    out = (C.c_int32 * 4)()
    assert L.load().b2k_debug_onepass_launch(out) == 0
    return tuple(out)


def unit_vector(n, j, dt):
    e = np.zeros(n, dtype=dt)
    e[j] = 1
    return e


@gpu
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("n", [1, 7, 512])
@pytest.mark.parametrize("m", [1, 31, 32, 33, 4097])
def test_dense_splitmix_fill(fma, m, n, dt):
    seed = SEED + 1000 * m + n
    want = ko.dense_splitmix(seed, m, n, dtype=dt)
    ctx = kk.B200Context(m, 8, dtype=dt)
    try:
        sv = ctx.add_space(n, 8, sharded=False)
        op = kk.B200Dense.splitmix(ctx, m, n, seed, sv)
        for j in range(n):
            col = kk.apply(op, ctx.from_host(unit_vector(n, j, dt), space=sv)).to_host()
            assert np.array_equal(bits(col), bits(want[:, j])), j
        for i in sorted({i for i in (0, 1, 30, 31, 32, 33, m // 2, m - 33, m - 32, m - 2, m - 1) if 0 <= i < m}):
            row = apply_adjoint(op, ctx.from_host(unit_vector(m, i, dt))).to_host()
            assert np.array_equal(bits(row), bits(want[i, :])), i
        # rows [m, ld) are zero: A'(A e_j) over the padded tiles equals the restatement on A padded with zeros
        for j in sorted({0, n - 1}):
            e = unit_vector(n, j, dt)
            y, z = apply_normal_gram(op, ctx.from_host(e, space=sv))
            v, _, grid, _ = onepass_launch()
            assert v == 0
            ry, _, _, rz = rs.apply_normal_gram(np.ascontiguousarray(want), e, 0, grid, fma)
            assert np.array_equal(bits(y.to_host()), bits(ry)) and np.array_equal(bits(z.to_host()), bits(rz)), j
    finally:
        ctx.close()
