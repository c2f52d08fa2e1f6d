"""GPU tests of the single-operator SpMV kernels with their fused epilogue (SpmvFuse: the normalised gather, the vout
store, the fused dot with dotv or with the normalised operand, the MGS-order dot_sub, the shift, the L2 hints and the
stop flag) against the exact host restatement of tests/spmv_restate.py: y and vout bit for bit, the dot as a double bit
for bit (signed zeros by their bits, NaNs by position).

Every launch goes through b2k_debug_apply_fused, which builds the SpmvFuse from host arguments and calls the production
b2k_enqueue_apply_fused; b2k_debug_spmv_launch says which kernel and instance ran on which grid, and that grid is the
one the restatement uses.  b2k_debug_op_tiles gives the device's tile boundaries, which must equal finish_csr's rules
as restated.  Kernels: k_spmv_stream, k_spmv_pipe in both variants, the four k_spmv_compact instances and the
matrix-free k_stencil_apply in 2-D and 3-D.
"""
import contextlib
import ctypes as C
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)
from test_gpu_csr_compact import INTS, REALS, banded

import spmv_restate as R

f64, f32 = np.float64, np.float32
STREAM, PIPE, COMPACT, STENCIL = 1, 2, 3, 4                 # b2k_debug_spmv_launch kernel ids
F32V, I16 = 1, 2                                            # b2k_debug_spmv_launch instance bits of k_spmv_compact
COMPACT_INST = {"c_dfi16": F32V | I16, "c_dfi32": F32V, "c_ddi16": I16, "c_ffi16": F32V | I16}
SENTINEL = -1234.25                                         # what the dot slot holds before a launch
XSCALES = [1.0 / 3.0, -0.7]                                 # neither is exact in Float32
COEFFS = (4.0, -1.4, -0.6, -1.2, -0.8, -0.3, -0.7)


@contextlib.contextmanager
def kernel(name):
    """the switches that make the dispatcher pick `name`: stream, pipe24 / pipe33 (variant 1 / 0), compact"""
    lib = L.load()
    lib.b2k_debug_set_spmv_pipe(0 if name == "stream" else 1)
    lib.b2k_debug_set_spmv_variant(0 if name == "pipe33" else 1)
    lib.b2k_debug_set_csr_compact(0 if name.startswith("pipe") else 1)
    try:
        yield
    finally:
        lib.b2k_debug_set_spmv_pipe(1)
        lib.b2k_debug_set_spmv_variant(1)
        lib.b2k_debug_set_csr_compact(1)


def launch():
    out = (C.c_int32 * 4)()
    assert L.load().b2k_debug_spmv_launch(out) == L.OK
    return tuple(out)


def device_tiles(op):
    lib, nblk = L.load(), C.c_int32()
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, None, C.byref(nblk)) == L.OK
    rb = np.empty(nblk.value + 1, dtype=np.int32)
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, rb.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nblk)) == L.OK
    return rb.astype(np.int64)


def fused(op, x, y, a0=0.0, a1=1.0, shifted=False, dotv=None, xscale=None, vout=None, dot_self=False, dsub=None,
          dsc=0.0, l2=False, stop=0, no_slot=False):
    """(status, what the dot slot holds afterwards)"""
    d = C.c_double(SENTINEL)
    xs = C.byref(C.c_double(xscale)) if xscale is not None else None
    h = lambda v: v.handle if v is not None else -1
    st = L.load().b2k_debug_apply_fused(op.ctx.h, op.h, x.handle, y.handle, a0, a1, int(shifted), h(dotv), xs, h(vout),
                                        int(dot_self), h(dsub), dsc, int(l2), int(stop), int(no_slot), C.byref(d))
    return st, d.value


def same(a, b):
    """bit for bit; NaNs by position"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


class Case:
    """one operator with its host form, seeded operands and the kernel that must run on it"""

    def __init__(self, ctx, op, dt, host, kname, seed=1, xspace=0):
        self.ctx, self.op, self.dt, self.kname = ctx, op, dt, kname
        self.host = host                       # ("csr", rowptr, colidx, vals) or ("stencil", nx, ny, nz, coeffs)
        m, n = op.n_rows, op.n_cols
        rng = np.random.default_rng(seed)
        self.xh = rng.standard_normal(n).astype(dt)
        self.xh[rng.integers(0, n, n // 50)] = -0.0
        self.vh, self.dh = rng.standard_normal(m).astype(dt), rng.standard_normal(m).astype(dt)
        self.x = ctx.from_host(self.xh, xspace)
        self.v, self.dsub = ctx.from_host(self.vh), ctx.from_host(self.dh)
        self.y, self.vout = ctx.empty(), ctx.empty()
        self.rowblk = None
        if host[0] == "csr":
            self.rowblk = R.tiles(host[1])
            assert np.array_equal(device_tiles(op), self.rowblk)

    def run(self, fma, *, xscale=None, vout=False, dot=None, dsub=False, shift=False, l2=False):
        """one launch with these features against the restatement; returns the launch record"""
        dt = self.dt
        y0 = np.full(self.op.n_rows, 7.5, dtype=dt)
        self.y.upload(y0)
        self.vout.upload(y0)
        a0, a1 = (0.3, -1.25) if shift else (0.0, 1.0)
        kw = dict(a0=a0, a1=a1, shifted=shift, xscale=xscale, dot_self=dot == "self", dsc=-0.45 if dsub else 0.0)
        with kernel(self.kname):
            st, d = fused(self.op, self.x, self.y, dotv=self.v if dot == "dotv" else None,
                          vout=self.vout if vout else None, dsub=self.dsub if dsub else None, l2=l2, **kw)
            rec = launch()
        assert st == L.OK
        want_k = {"stream": STREAM, "pipe24": PIPE, "pipe33": PIPE, "stencil": STENCIL}.get(self.kname, COMPACT)
        assert rec[0] == want_k, (rec, self.kname)
        if self.kname.startswith("pipe"):
            assert rec[1] == (1 if self.kname == "pipe24" else 0)
        rk = {STREAM: "stream", PIPE: "pipe", COMPACT: "compact", STENCIL: "stencil"}[rec[0]]
        src = dict(stencil=self.host[1:]) if rk == "stencil" else dict(csr=self.host[1:], rowblk=self.rowblk)
        if rk != "stencil":
            assert rec[3] == len(self.rowblk) - 1 and 1 <= rec[2] <= rec[3]
        y, vn, dref = R.apply(fma, dt, rk, rec[2], self.xh, dotv=self.vh if dot == "dotv" else None,
                              dsub=self.dh if dsub else None, **src, **kw)
        assert same(self.y.to_host(), y), ("y", self.kname)
        assert same(self.vout.to_host(), vn if vout else y0), ("vout", self.kname)
        if dot is None:
            assert d == SENTINEL
        else:
            assert same(np.float64(d), np.float64(dref)), ("dot", self.kname, d, dref)
        return rec


# ------------------------------------------------------------------ operators ----

def csr_op(ctx, rowptr, cols, vals, n_cols=None):
    n = len(rowptr) - 1
    op = kk.B200CSR.from_csr_arrays(ctx, n, n if n_cols is None else n_cols, np.asarray(rowptr, np.int64),
                                    np.asarray(cols, np.int64), vals)
    return op, ("csr", np.asarray(rowptr, np.int64), np.asarray(cols, np.int64), np.asarray(vals, ctx.np_dtype))


def scipy_op(ctx, A):
    A = A.tocsr()
    A.sort_indices()
    return csr_op(ctx, A.indptr, A.indices, A.data.astype(ctx.np_dtype))


def mixed(n, seed, long_rows=(2000,), empty=(1500, 3000), rng_vals=None):
    """n rows of about 4 random, unsorted, sometimes repeated columns; rows of the given lengths in front (long ones
    alone in their tile), a run of empty rows (a tile of more than 1024 rows)"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 9, n)
    lens[empty[0]:empty[1]] = 0
    for i, m in enumerate(long_rows):
        lens[3 + 7 * i] = m
    rowptr = np.r_[0, np.cumsum(lens)]
    cols = rng.integers(0, n, rowptr[-1])
    dup = rng.integers(0, rowptr[-1] - 1, rowptr[-1] // 20)
    cols[dup + 1] = cols[dup]                  # repeated columns (within a row where the pair does not straddle one)
    vals = rng_vals(rowptr[-1]) if rng_vals else rng.standard_normal(rowptr[-1])
    return rowptr, cols, vals


def make_case(name, dt=None, seed=1):
    """small operators, one per kernel instance"""
    if name in ("stencil2d", "stencil3d"):
        dims = (61, 47, 1) if name == "stencil2d" else (17, 13, 11)
        n = int(np.prod(dims))
        ctx = kk.B200Context(n, 8, dtype=dt)
        op = kk.B200CSR.stencil_free(ctx, *dims, coeffs=COEFFS)
        return Case(ctx, op, dt, ("stencil", *dims, COEFFS), "stencil", seed)
    if name in ("stream", "pipe24", "pipe33"):
        n = 5000
        ctx = kk.B200Context(n, 8, dtype=dt)
        op, host = csr_op(ctx, *mixed(n, seed))
        return Case(ctx, op, dt, host, name, seed)
    # compact instances <T, VS, IS>: test_gpu_csr_compact's banded matrices at the 16-bit offset limits
    dt, reach, vals = {"c_dfi16": (f64, (32768, 32767), INTS), "c_dfi32": (f64, (32768, 32768), INTS),
                       "c_ddi16": (f64, (32768, 32767), REALS), "c_ffi16": (f32, (32768, 32767), REALS)}[name]
    A = banded(100_000, reach, values=vals)
    ctx = kk.B200Context(A.shape[0], 8, dtype=dt)
    op, host = scipy_op(ctx, A)
    assert L.load().b2k_debug_csr_format(op.h) == 4 | (COMPACT_INST[name] if dt == f64 else I16)
    return Case(ctx, op, dt, host, name, seed)


KCASES = [("stream", f64), ("stream", f32), ("pipe24", f64), ("pipe24", f32), ("pipe33", f64), ("pipe33", f32),
          ("c_dfi16", None), ("c_dfi32", None), ("c_ddi16", None), ("c_ffi16", None),
          ("stencil2d", f64), ("stencil2d", f32), ("stencil3d", f64), ("stencil3d", f32)]
KIDS = [f"{k}-{np.dtype(d).name}" if d else k for k, d in KCASES]


def check_instance(case, rec):
    if case.kname in COMPACT_INST:
        assert rec[1] == COMPACT_INST[case.kname]


FEATURES = [dict(), dict(xscale=XSCALES[0]), dict(xscale=XSCALES[1]), dict(vout=True), dict(dot="dotv"),
            dict(dot="self"), dict(dot="dotv", dsub=True), dict(shift=True), dict(l2=True)]
CALLERS = [dict(xscale=XSCALES[0], vout=True, dot="self", l2=True),                 # chained Lanczos step
           dict(xscale=XSCALES[1], vout=True, dot="self", l2=True, dsub=True),      # ... with the MGS-order alpha
           dict(xscale=XSCALES[0], dot="self", shift=True),                         # MINRES
           dict(dot="dotv", shift=True)]                                            # CG, BiCGStab


@pytest.mark.parametrize("kname,dt", KCASES, ids=KIDS)
def test_each_feature_and_the_callers_sets(fma, kname, dt):
    case = make_case(kname, dt)
    for feats in FEATURES + CALLERS:
        check_instance(case, case.run(fma, **feats))
    case.ctx.close()


@pytest.mark.parametrize("kname,dt", KCASES, ids=KIDS)
def test_full_cross_product(fma, kname, dt):
    """xscale x vout x {none, dotv, dot_self} x dot_sub x shift x l2_hints on a small operator"""
    case = make_case(kname, dt, seed=7)
    for xs, vo, dot, ds, sh, l2 in itertools.product([None, XSCALES[1]], [False, True], [None, "dotv", "self"],
                                                     [False, True], [False, True], [False, True]):
        case.run(fma, xscale=xs, vout=vo, dot=dot, dsub=ds, shift=sh, l2=l2)
    case.ctx.close()


# ------------------------------------------------------------------ shapes ----

CSR_KERNELS = ["stream", "pipe24", "compact"]
ALL = dict(xscale=XSCALES[0], vout=True, dot="self", shift=True)


@pytest.mark.parametrize("kname", CSR_KERNELS + ["stencil"])
def test_n1(fma, kname):
    ctx = kk.B200Context(1, 8)
    if kname == "stencil":
        case = Case(ctx, kk.B200CSR.stencil_free(ctx, 1, 1, 1, COEFFS), f64, ("stencil", 1, 1, 1, COEFFS), kname)
    else:
        op, host = csr_op(ctx, [0, 1], [0], np.array([1.7]))
        case = Case(ctx, op, f64, host, kname)
    for feats in (dict(), ALL, dict(dot="dotv", dsub=True)):
        rec = case.run(fma, **feats)
        assert rec[2] == 1
    ctx.close()


@pytest.mark.parametrize("kname", ["stream", "pipe24"])
def test_no_nonzeros(fma, kname):
    """every row empty: one tile, no compact view (the default dispatch takes k_spmv_pipe)"""
    n = 3000
    ctx = kk.B200Context(n, 8)
    op, host = csr_op(ctx, np.zeros(n + 1, np.int64), np.zeros(0, np.int64), np.zeros(0))
    assert L.load().b2k_debug_csr_format(op.h) == 0
    case = Case(ctx, op, f64, host, kname)
    assert case.rowblk.tolist() == [0, n]
    for feats in (dict(), ALL, dict(dot="dotv", dsub=True, shift=True)):
        case.run(fma, **feats)
    with kernel("compact"):
        st, _ = fused(op, case.x, case.y)
        assert st == L.OK and launch()[0] == PIPE
    ctx.close()


def staged_tiles():
    """greedy tiles (a row of 769) of exactly 1024 and 1025 rows starting at unaligned rows 3 and 1027: the first
    stages its row pointers in shared memory, the second reads them from global memory; then rows of 1536 and 1537"""
    lens = [769, 700, 67] + [1] * 1024 + [600] + [0] * 1024 + [1000, 5, 1536, 1537, 3] + [2] * 500
    rng = np.random.default_rng(11)
    rowptr = np.r_[0, np.cumsum(lens)]
    n = len(lens)
    return rowptr, rng.integers(0, n, rowptr[-1]), rng.standard_normal(rowptr[-1])


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("kname", CSR_KERNELS)
def test_staged_and_global_row_pointers_and_long_row_edges(fma, kname, dt):
    rowptr, cols, vals = staged_tiles()
    ctx = kk.B200Context(len(rowptr) - 1, 8, dtype=dt)
    op, host = csr_op(ctx, rowptr, cols, vals.astype(dt))
    case = Case(ctx, op, dt, host, kname)
    rb = case.rowblk.tolist()
    i = rb.index(3)
    assert rb[i + 1] == 3 + 1024 and rb[i + 2] == 1027 + 1025
    j = rb.index(int(np.flatnonzero(np.diff(rowptr) == 1536)[0]))
    assert rowptr[rb[j + 1]] - rowptr[rb[j]] == 1536 and rb[j + 2] - rb[j + 1] == 1     # 1536: a tile; 1537: alone
    for feats in FEATURES[1:] + CALLERS:
        case.run(fma, **feats)
    ctx.close()


@pytest.mark.parametrize("maxrow", [768, 769])
@pytest.mark.parametrize("kname", CSR_KERNELS)
def test_maxrow_768_and_769(fma, kname, maxrow):
    """the nnz-balanced device partition against the greedy host one: rowblk as restated either way"""
    rng = np.random.default_rng(maxrow)
    lens = rng.integers(0, 12, 20000)
    lens[[5, 9000]] = maxrow
    rowptr = np.r_[0, np.cumsum(lens)]
    ctx = kk.B200Context(len(lens), 8)
    op, host = csr_op(ctx, rowptr, rng.integers(0, len(lens), rowptr[-1]), rng.integers(-8, 9, rowptr[-1]) / 4.0)
    case = Case(ctx, op, f64, host, kname)
    for feats in CALLERS:
        case.run(fma, **feats)
    ctx.close()


@pytest.mark.parametrize("kname", CSR_KERNELS + ["stencil"])
def test_grids_of_one_cta_few_and_several_tiles_per_cta(fma, kname):
    """1 CTA; fewer tiles than the grid cap; about 1M nonzeros, several tiles per CTA (then the ticket of every grid
    size back to back: each dot exact, so the ticket returns to 0 after every launch)"""
    cases = []
    for n, per in ((256, 3), (60000, 5), (500000, 5)):
        if kname == "stencil":
            ctx = kk.B200Context(n, 8)
            dims = {256: (16, 16, 1), 60000: (300, 200, 1), 500000: (100, 50, 100)}[n]
            cases.append(Case(ctx, kk.B200CSR.stencil_free(ctx, *dims, coeffs=COEFFS), f64, ("stencil", *dims, COEFFS),
                              kname))
        else:
            rng = np.random.default_rng(n)
            lens = rng.integers(per - 2, per + 3, n)
            rowptr = np.r_[0, np.cumsum(lens)]
            cols = np.clip(np.repeat(np.arange(n), lens) + rng.integers(-200, 201, rowptr[-1]), 0, n - 1)
            ctx = kk.B200Context(n, 8)
            op, host = csr_op(ctx, rowptr, cols, rng.integers(-8, 9, rowptr[-1]) / 8.0)
            cases.append(Case(ctx, op, f64, host, kname))
    recs = [c.run(fma, **CALLERS[1]) for c in cases]
    assert recs[0][2] == 1 and 1 < recs[1][2] < recs[2][2]
    if kname == "stencil":
        assert 256 * recs[2][2] < 500000                            # several rows per thread
    elif kname != "stream":
        assert recs[1][2] == recs[1][3] and 3 * recs[2][2] <= recs[2][3]
    for _ in range(2):
        for c in cases:
            c.run(fma, dot="dotv", shift=True)
    for c in cases:
        c.ctx.close()


@pytest.mark.parametrize("kname", CSR_KERNELS)
def test_rectangular(fma, kname):
    """a wide and a tall operator: plain, dotv and dot_sub (y-space vectors); vout / dot_self refused"""
    for m, n in ((3000, 7000), (7000, 3000)):
        rng = np.random.default_rng(m)
        lens = rng.integers(0, 9, m)
        rowptr = np.r_[0, np.cumsum(lens)]
        ctx = kk.B200Context(m, 8)
        xsp = ctx.add_space(n, 4)
        op, host = csr_op(ctx, rowptr, rng.integers(0, n, rowptr[-1]), rng.standard_normal(rowptr[-1]), n_cols=n)
        case = Case(ctx, op, f64, host, kname, xspace=xsp)
        for feats in (dict(), dict(dot="dotv"), dict(dot="dotv", dsub=True, xscale=XSCALES[1], l2=True)):
            case.run(fma, **feats)
        with kernel(kname):
            for kw in (dict(vout=case.vout), dict(dot_self=True)):
                assert fused(op, case.x, case.y, **kw) == (L.EDIM, SENTINEL)
        ctx.close()


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("kname", CSR_KERNELS)
def test_infinities_against_stored_zeros(fma, kname, dt):
    """0 * ±Inf = NaN at its position, ±0 products and sums with their signs"""
    rowptr, cols, vals = mixed(4000, 5, long_rows=(1800,), rng_vals=lambda k: np.random.default_rng(9).integers(
        -2, 3, k).astype(np.float64))
    hit = np.flatnonzero(np.isin(cols, [17, 2500]))
    vals[hit[::2]] = 0.0
    cols[rowptr[3]], vals[rowptr[3]] = 17, 0.0             # and in the long row
    ctx = kk.B200Context(4000, 8, dtype=dt)
    op, host = csr_op(ctx, rowptr, cols, vals.astype(dt))
    case = Case(ctx, op, dt, host, kname)
    case.xh[[17, 2500]] = [np.inf, -np.inf]
    case.xh[np.flatnonzero(np.arange(4000) % 5 == 1)] = -0.0
    case.x.upload(case.xh)
    for feats in (dict(), dict(dot="dotv"), ALL):
        case.run(fma, **feats)
    ctx.close()


# ------------------------------------------------------------------ stop flag, refusals ----

@pytest.mark.parametrize("kname", CSR_KERNELS + ["stencil"])
def test_stop_flag_writes_nothing(fma, kname):
    case = make_case({"stream": "stream", "pipe24": "pipe24", "compact": "c_dfi16", "stencil": "stencil2d"}[kname], f64)
    dt = case.dt
    y0 = np.full(case.op.n_rows, 2.5, dtype=dt)
    case.y.upload(y0)
    case.vout.upload(y0)
    with kernel(case.kname):
        st, d = fused(case.op, case.x, case.y, xscale=XSCALES[0], vout=case.vout, dot_self=True, dsub=case.dsub,
                      dsc=0.5, shifted=True, a0=0.2, stop=1)
    assert st == L.OK and d == SENTINEL
    assert same(case.y.to_host(), y0) and same(case.vout.to_host(), y0)
    case.run(fma, **CALLERS[1])
    case.ctx.close()


def test_refusals_write_nothing():
    case = make_case("stream", f64)
    n = case.op.n_rows
    y0 = np.full(n, 2.5)
    dense = kk.B200Dense.from_host(case.ctx, np.eye(n), case.ctx.add_space(n, 2, sharded=False))
    case.y.upload(y0)
    case.vout.upload(y0)
    assert fused(case.op, case.x, case.y, dot_self=True, no_slot=True) == (L.EINVAL, SENTINEL)
    assert fused(dense, case.x, case.y, dotv=case.v) == (L.ENOTSUP, SENTINEL)
    assert fused(case.op, case.x, case.x, dotv=case.v, vout=case.vout) == (L.EINVAL, SENTINEL)
    assert same(case.y.to_host(), y0) and same(case.vout.to_host(), y0) and same(case.x.to_host(), case.xh)
    case.ctx.close()
