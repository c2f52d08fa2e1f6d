"""Operator ingestion cases shared by test_gpu_op_ingest.py (the library) and test_op_ingest_hostsim.py (the numpy
stand-in of the C-ABI, hostsim.py).

1. The device arrays each entry form must build: int32 rowptr / colidx (base 0) and values in T.
   - CSR input (b2k_op_create_csr, from_csr_arrays) keeps its stored order, unsorted and repeated columns included.
   - CSC input (b2k_op_create_csc, from_julia_csc) is a stable counting sort by row: within a row the columns come
     out ascending, a repeated (row, column) in colptr order; rowval / nzval entries past colptr[n_cols] are ignored.
   - Stencils are oracle.krylov_oracle.stencil_matrix with the coefficients rounded to T first ((T)c[k]).
2. The host matrices of every shape the ingestion and tiling code branches on (SHAPES).
3. One table of malformed inputs (BAD), each with the status code it must return.  Both test files run all of it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

BIG = 1 << 31          # the first size the int32 device indices cannot hold
SP_NNZ = 1536          # nonzeros of one SpMV tile; a longer row takes the long-row path


# ---------------------------------------------------------------- expected device arrays ----

def csr_expected(rowptr, colidx, vals, base, dt):
    return ((np.asarray(rowptr, np.int64) - base).astype(np.int32),
            (np.asarray(colidx, np.int64) - base).astype(np.int32), np.asarray(vals).astype(dt))


def csc_expected(n_rows, n_cols, colptr, rowval, nzval, base, dt):
    """the stable counting sort of the CSC entries by row (a stable argsort is one)"""
    cp = np.asarray(colptr, np.int64) - base
    nnz = int(cp[-1])
    rv = np.asarray(rowval, np.int64)[:nnz] - base
    col = np.repeat(np.arange(n_cols, dtype=np.int64), np.diff(cp))
    order = np.argsort(rv, kind="stable")
    rowptr = np.concatenate(([0], np.cumsum(np.bincount(rv, minlength=n_rows))))
    return rowptr.astype(np.int32), col[order].astype(np.int32), np.asarray(nzval)[:nnz].astype(dt)[order]


def stencil_expected(nx, ny, nz, coeffs, dt):
    A = ko.stencil_matrix(nx, ny, nz, tuple(float(dt(c)) for c in coeffs), dtype=dt)
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data


def stencil_nnz(nx, ny, nz):
    """the centre, and both ends of every grid edge along x, y and z"""
    return nx * ny * nz + 2 * ((nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1))


def swapped(c):
    """the coefficients of transpose(stencil(c)): west / east, south / north and down / up exchanged"""
    return (c[0], c[2], c[1], c[4], c[3], c[6], c[5])


# ---------------------------------------------------------------- host matrices ----

@dataclass
class Shape:
    """A host matrix as COO triplets in CSR stored order: rows ascending, within a row the columns as generated
    (unsorted, some repeated)."""
    n_rows: int
    n_cols: int
    rows: np.ndarray
    cols: np.ndarray
    vals: np.ndarray
    apply: bool = True          # False: only built and read back (x of n_cols entries does not fit a context)

    @property
    def nnz(self):
        return len(self.vals)

    def csr(self):
        rowptr = np.concatenate(([0], np.cumsum(np.bincount(self.rows, minlength=self.n_rows)))).astype(np.int64)
        return rowptr, self.cols.astype(np.int64), self.vals

    def csc(self, seed=0):
        """(colptr, rowval, nzval), base 0; within a column the entries in a shuffled order"""
        rng = np.random.default_rng(seed)
        perm = rng.permutation(self.nnz)
        order = perm[np.argsort(self.cols[perm], kind="stable")]
        colptr = np.concatenate(([0], np.cumsum(np.bincount(self.cols, minlength=self.n_cols)))).astype(np.int64)
        return colptr, self.rows[order].astype(np.int64), self.vals[order]


def _from_lengths(lens, n_cols, rng, long_rows=()):
    """rows of the given lengths with random columns; every 5th row of two or more entries repeats its first column,
    and the rows in long_rows hold distinct shuffled columns (plus one repeat)"""
    lens = np.asarray(lens, dtype=np.int64)
    rows = np.repeat(np.arange(len(lens)), lens)
    cols = rng.integers(0, n_cols, int(lens.sum()))
    starts = np.concatenate(([0], np.cumsum(lens)[:-1]))
    for r in np.flatnonzero(lens >= 2)[::5]:
        cols[starts[r] + 1] = cols[starts[r]]
    for r in long_rows:
        c = rng.choice(n_cols, int(lens[r]), replace=False)
        c[-1] = c[0]
        cols[starts[r]:starts[r] + lens[r]] = c
    vals = rng.standard_normal(len(cols))
    return rows, cols, vals


def _shape(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "n1":
        return Shape(1, 1, np.array([0]), np.array([0]), np.array([-1.75]))
    if name == "nnz0":
        return Shape(40, 40, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0))
    if name in ("edge-rows", "gap2k", "gap64k"):
        n, gap = {"edge-rows": (500, None), "gap2k": (3000, (400, 2600)), "gap64k": (67000, (300, 66600))}[name]
        lens = rng.integers(1, 9, n)
        if gap is None:
            lens[:7] = 0
            lens[-11:] = 0
        else:
            lens[gap[0]:gap[1]] = 0
        return Shape(n, n, *_from_lengths(lens, n, rng))
    if name in ("maxrow768", "maxrow769", "longrow"):
        n, r, k = {"maxrow768": (4000, 1234, 768), "maxrow769": (4000, 1234, 769), "longrow": (5000, 77, 2000)}[name]
        lens = rng.integers(0, 9, n)
        lens[r] = k
        return Shape(n, n, *_from_lengths(lens, n, rng, long_rows=(r,)))
    if name in ("tall", "wide"):
        m, n = (900, 300) if name == "tall" else (300, 900)
        return Shape(m, n, *_from_lengths(rng.integers(0, 7, m), n, rng))
    if name == "corners":
        n = 200
        lens = rng.integers(0, 5, n)
        lens[50] = 2
        rows, cols, vals = _from_lengths(lens, n, rng)
        s = int(lens[:50].sum())
        cols[s:s + 2] = (n - 1, 0)
        return Shape(n, n, rows, cols, vals)
    if name == "huge-ncols":
        n_cols = BIG - 1
        lens = np.zeros(64, np.int64)
        lens[5], lens[9] = 3, 1
        return Shape(64, n_cols, np.repeat(np.arange(64), lens), np.array([n_cols - 1, 0, 7, n_cols - 1]),
                     np.array([0.5, -2.0, 1.25, 3.0]), apply=False)
    raise KeyError(name)


SHAPE_NAMES = ["n1", "nnz0", "edge-rows", "gap2k", "gap64k", "maxrow768", "maxrow769", "longrow", "tall", "wide",
               "corners", "huge-ncols"]
_SHAPES: dict[str, Shape] = {}


def shape(name) -> Shape:
    if name not in _SHAPES:
        _SHAPES[name] = _shape(name)
    return _SHAPES[name]


# ---------------------------------------------------------------- entry forms ----

# from_csr_arrays with int32 / int64 indices and base 0 / 1, from_scipy; from_julia_csc, the raw CSC entry with int32
# base-0 indices, and from_julia_csc with rowval / nzval longer than nnz (spare capacity, filled with an out-of-range
# row and NaN that must never be read)
CSR_FORMS = ["csr-i32-b0", "csr-i32-b1", "csr-i64-b0", "csr-i64-b1", "scipy"]
CSC_FORMS = ["julia", "csc-raw-i32", "julia-spare"]
FORMS = CSR_FORMS + CSC_FORMS


def form_shape_pairs():
    """every (form, shape); a CSC colptr of 2^31 entries is not built"""
    return [(f, s) for f in FORMS for s in SHAPE_NAMES if f in CSR_FORMS or shape(s).apply]


def context(s: Shape, dt):
    """(ctx, space of y) for y = A x: a square A in space 0; a rectangular one maps space 0 (its columns) to a
    second space (its rows); an A whose x cannot be allocated gets its rows as space 0"""
    import krylovkit_jl_b200 as kk
    if s.n_rows == s.n_cols or not s.apply:
        return kk.B200Context(s.n_rows, 4, dtype=dt), 0
    ctx = kk.B200Context(s.n_cols, 4, dtype=dt)
    return ctx, ctx.add_space(s.n_rows, 4, sharded=False)


def build(ctx, form, s: Shape, dt):
    """(B200CSR built by `form` from s, the expected device (rowptr, colidx, vals))"""
    import scipy.sparse as sp

    import krylovkit_jl_b200 as kk
    if form.startswith("csr-"):
        idx, base = (np.int32 if "i32" in form else np.int64), int(form[-1])
        rp, ci, va = s.csr()
        op = kk.B200CSR.from_csr_arrays(ctx, s.n_rows, s.n_cols, rp.astype(idx) + idx(base),
                                        ci.astype(idx) + idx(base), va, index_base=base)
        return op, csr_expected(rp, ci, va, 0, dt)
    if form == "scipy":
        A = sp.csr_matrix((s.vals, s.cols, s.csr()[0]), shape=(s.n_rows, s.n_cols))
        sent = A if A.has_sorted_indices else A.sorted_indices()
        return kk.B200CSR.from_scipy(ctx, A), csr_expected(sent.indptr, sent.indices, sent.data, 0, dt)
    cp, rv, nz = s.csc()
    want = csc_expected(s.n_rows, s.n_cols, cp, rv, nz, 0, dt)
    if form == "julia":
        return kk.B200CSR.from_julia_csc(ctx, s.n_rows, s.n_cols, cp + 1, rv + 1, nz), want
    if form == "julia-spare":
        rv2 = np.concatenate((rv + 1, np.full(5, s.n_rows + 7)))
        nz2 = np.concatenate((nz, np.full(5, np.nan)))
        return kk.B200CSR.from_julia_csc(ctx, s.n_rows, s.n_cols, cp + 1, rv2, nz2), want
    assert form == "csc-raw-i32"
    cp32, rv32, nzt = cp.astype(np.int32), rv.astype(np.int32), np.ascontiguousarray(nz, dtype=dt)
    h = L.c_op()
    ctx.check(ctx.lib.b2k_op_create_csc(ctx.h, C.byref(h), s.n_rows, s.n_cols, s.nnz, cp32.ctypes.data,
                                        rv32.ctypes.data, nzt.ctypes.data, 4, 0))
    return kk.B200CSR(ctx, h), want


def download(op):
    """(n_rows, n_cols, nnz, kind) and the device (rowptr, colidx, vals) of a CSR operator"""
    ctx = op.ctx
    nr, nc, nnz, kind = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    ctx.check(ctx.lib.b2k_op_info(op.h, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(kind)))
    rp = np.empty(nr.value + 1, dtype=np.int32)
    ci = np.empty(nnz.value, dtype=np.int32)
    va = np.empty(nnz.value, dtype=ctx.np_dtype)
    ctx.check(ctx.lib.b2k_op_csr_download(ctx.h, op.h, rp.ctypes.data, ci.ctypes.data, va.ctypes.data))
    return (nr.value, nc.value, nnz.value, kind.value), (rp, ci, va)


def same(a, b):
    """equal dtype, shape and bytes (values compared by their bits)"""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


# ---------------------------------------------------------------- malformed inputs ----

# The context every row runs in: space 0 of N0 entries and one more space of N1.
N0, N1 = 6, 4
# A valid 6 x 6 CSR / CSC pattern, base 0, and the stencil grid of N0 points.
RP = [0, 2, 3, 3, 5, 6, 7]
IX = [0, 5, 1, 2, 4, 3, 0]
NNZ = 7
COEFFS = (4.0, -1.0, -1.5, -0.5, -2.0, -0.25, -0.75)


@dataclass
class Bad:
    id: str
    entry: str          # csr, csc, stencil, dense
    args: dict
    code: int


def _idx(kind, ptr=RP, ix=IX, n_rows=N0, n_cols=N0, nnz=NNZ, dtype=np.int64, base=0, idx_bytes=None):
    return Bad("", kind, dict(n_rows=n_rows, n_cols=n_cols, nnz=nnz,
                              ptr=np.asarray(ptr, np.int64).astype(dtype) + dtype(base),
                              ix=np.asarray(ix, np.int64).astype(dtype) + dtype(base),
                              idx_bytes=np.dtype(dtype).itemsize if idx_bytes is None else idx_bytes,
                              base=base), 0)


def _rows():
    EINVAL, EDIM, ENOTSUP = L.EINVAL, L.EDIM, L.ENOTSUP
    out = []

    def add(id_, code, row):
        row.id, row.code = id_, code
        out.append(row)

    for k in ("csr", "csc"):
        p = "rowptr" if k == "csr" else "colptr"
        add(f"{k}-idx-bytes-2", EINVAL, _idx(k, idx_bytes=2))
        add(f"{k}-base-2", EINVAL, _idx(k, base=2))
        add(f"{k}-{p}-first", EINVAL, _idx(k, ptr=[1] + RP[1:]))
        add(f"{k}-{p}-first-i32-base1", EINVAL, _idx(k, ptr=[-1] + RP[1:], dtype=np.int32, base=1))
        add(f"{k}-{p}-last-above-nnz", EINVAL, _idx(k, ptr=RP[:-1] + [NNZ + 1]))
        add(f"{k}-{p}-last-below-nnz", EINVAL, _idx(k, ptr=RP[:-1] + [NNZ - 1]))
        add(f"{k}-{p}-decreasing-i64", EINVAL, _idx(k, ptr=[0, 3, 2, 3, 5, 6, 7]))
        add(f"{k}-{p}-decreasing-i32", EINVAL, _idx(k, ptr=[0, 3, 2, 3, 5, 6, 7], dtype=np.int32, base=1))
        add(f"{k}-{p}-entry-above-nnz", EINVAL, _idx(k, ptr=[0, 2, 9, 3, 5, 6, 7]))
        # an int64 entry that the int32 cast makes look in range and monotone (2 + 2^32 -> 2, 2 - 2^32 -> 2)
        add(f"{k}-{p}-entry-2^32-i64", EINVAL, _idx(k, ptr=[0, 2 + (1 << 32), 3, 3, 5, 6, 7]))
        add(f"{k}-{p}-entry-negative-i64", EINVAL, _idx(k, ptr=[0, 2 - (1 << 32), 3, 3, 5, 6, 7]))
        add(f"{k}-{p}-entry-2^32-i64-base1", EINVAL, _idx(k, ptr=[0, 2 + (1 << 32), 3, 3, 5, 6, 7], base=1))
        # the same without nonzeros, where no column check runs
        add(f"{k}-{p}-entry-2^32-i64-nnz0", EINVAL, _idx(k, ptr=[0, 0, 1 << 32, 0, 0, 0, 0], ix=[], nnz=0))
        add(f"{k}-index-n", EINVAL, _idx(k, ix=IX[:3] + [N0] + IX[4:]))
        add(f"{k}-index-minus1", EINVAL, _idx(k, ix=IX[:3] + [-1] + IX[4:]))
        add(f"{k}-index-0-base1", EINVAL, _idx(k, ix=IX[:3] + [-1] + IX[4:], dtype=np.int32, base=1))
        add(f"{k}-nnz-2^31", ENOTSUP, _idx(k, nnz=BIG))
        add(f"{k}-nnz-negative", EINVAL, _idx(k, nnz=-1))
        add(f"{k}-ncols-2^31", ENOTSUP, _idx(k, n_cols=BIG))
        add(f"{k}-ncols-negative", EINVAL, _idx(k, ptr=[0], ix=[], n_cols=-1, nnz=0) if k == "csc"
            else _idx(k, ptr=[0] * (N0 + 1), ix=[], n_cols=-1, nnz=0))
        add(f"{k}-nrows-2^31", ENOTSUP, _idx(k, n_rows=BIG))
        add(f"{k}-nrows-negative", EINVAL, _idx(k, n_rows=-1))
        add(f"{k}-nrows-not-a-space", EDIM, _idx(k, n_rows=N0 - 1) if k == "csc"
            else _idx(k, ptr=RP[:-1], ix=IX[:5], nnz=5, n_rows=N0 - 1))
    add("stencil-nx-0", EINVAL, Bad("", "stencil", dict(grid=(0, N0, 1)), 0))
    add("stencil-ny-0", EINVAL, Bad("", "stencil", dict(grid=(N0, 0, 1)), 0))
    add("stencil-nz-0", EINVAL, Bad("", "stencil", dict(grid=(N0, 1, 0)), 0))
    add("stencil-grid-7", EDIM, Bad("", "stencil", dict(grid=(7, 1, 1)), 0))
    add("stencil-grid-2x2x2", EDIM, Bad("", "stencil", dict(grid=(2, 2, 2)), 0))
    add("dense-ld-below-m", EINVAL, Bad("", "dense", dict(m=N0, n=N1, ld=N0 - 1), 0))
    add("dense-m-not-space0", EDIM, Bad("", "dense", dict(m=N1, n=N1, ld=N1), 0))
    add("dense-n-0", EINVAL, Bad("", "dense", dict(m=N0, n=0, ld=N0), 0))
    return out


BAD = _rows()
BAD_IDS = [b.id for b in BAD]
assert len(set(BAD_IDS)) == len(BAD_IDS)


def call(lib, ctx, row: Bad, out):
    """the status of the entry point on one malformed row; out is a c_op the caller checks is still NULL"""
    a = row.args
    if row.entry in ("csr", "csc"):
        vals = np.arange(1, max(len(a["ix"]), 1) + 1, dtype=ctx.np_dtype)
        fn = lib.b2k_op_create_csr if row.entry == "csr" else lib.b2k_op_create_csc
        return fn(ctx.h, C.byref(out), a["n_rows"], a["n_cols"], a["nnz"], a["ptr"].ctypes.data,
                  a["ix"].ctypes.data if len(a["ix"]) else vals.ctypes.data, vals.ctypes.data,
                  a["idx_bytes"], a["base"])
    if row.entry == "stencil":
        c = (C.c_double * 7)(*COEFFS)
        return lib.b2k_op_create_stencil(ctx.h, C.byref(out), *a["grid"], c)
    A = np.ones((max(a["ld"], 1), max(a["n"], 1)), dtype=ctx.np_dtype, order="F")
    return lib.b2k_op_create_dense(ctx.h, C.byref(out), a["m"], a["n"], A.ctypes.data, a["ld"])


def valid_csr():
    """the valid 6 x 6 operator each refusal is followed by: (rowptr, colidx, vals)"""
    return np.array(RP, np.int64), np.array(IX, np.int64), np.arange(1, NNZ + 1) * 0.75
