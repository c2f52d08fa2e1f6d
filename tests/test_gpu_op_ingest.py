"""GPU tests of operator ingestion: the device CSR each entry form builds, bit for bit, in Float64 and Float32.

Every test of an SpMV kernel restates it from the host matrix; these tests check that the device holds that matrix.
The expected arrays, shapes and the table of malformed inputs are in op_ingest_cases.py.

A. Round trip: b2k_op_info and b2k_op_csr_download of every entry form (from_csr_arrays with int32 / int64 indices
   and base 0 / 1, from_scipy, from_julia_csc, the raw CSC entry, CSC arrays with spare capacity) on every shape (n = 1,
   no nonzeros, empty edge rows, empty runs of more than 2048 and 65 536 rows, longest rows of 768 and 769 for both
   tile partitions, a row past one tile, tall and wide, columns 0 and n_cols - 1 in one row, n_cols = 2^31 - 1), and
   b2k_debug_op_tiles against spmv_restate.tiles.
B. One product per form and shape under the plain pipe kernel and the compact kernel, against spmv_restate.csr_rows
   on the expected arrays: it ties each entry form to what the kernels stream, the compact copy included.
C. Stencil assembly on degenerate, ragged and 3-D grids with seven distinct coefficients (0.1 and others that Float32
   rounds), nnz against its closed form, and transpose(stencil(c)) == stencil(swapped c) array for array.
D. Dense upload through the raw entry with ld > m (NaN padding) and ld = m: A e_j returns column j exactly.
E. Every malformed row returns its code, leaves *out NULL and leaves the context usable.  Malformed values reach the
   device only through the conversion kernels, k_minmax_cols and k_rowptr_stats, which read in bounds whatever the
   values; no refused operator is applied.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L

import op_ingest_cases as K
import spmv_restate as R

f64, f32 = np.float64, np.float32
DTS = [pytest.param(f64, id="f64"), pytest.param(f32, id="f32")]
PAIRS = [pytest.param(f, s, id=f"{f}-{s}") for f, s in K.form_shape_pairs()]


@contextlib.contextmanager
def kernel(name):
    """pipe: the plain TMA kernel (compact copies off); compact: the compact copy where the operator has one"""
    lib = L.load()
    lib.b2k_debug_set_csr_compact(1 if name == "compact" else 0)
    try:
        yield
    finally:
        lib.b2k_debug_set_csr_compact(1)


def tiles(op):
    lib, nblk = op.ctx.lib, C.c_int32()
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, None, C.byref(nblk)) == L.OK
    rb = np.empty(nblk.value + 1, dtype=np.int32)
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, rb.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nblk)) == L.OK
    return rb.astype(np.int64)


def check_arrays(op, want, n_rows, n_cols):
    info, got = K.download(op)
    assert info == (n_rows, n_cols, len(want[2]), 0)
    for g, w, what in zip(got, want, ("rowptr", "colidx", "vals")):
        assert K.same(g, w), what
    assert np.array_equal(tiles(op), R.tiles(want[0]))


# ---------------------------------------------------------------- A. round trip ----

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("form,name", PAIRS)
def test_round_trip(form, name, dt):
    s = K.shape(name)
    ctx, _ = K.context(s, dt)
    op, want = K.build(ctx, form, s, dt)
    check_arrays(op, want, s.n_rows, s.n_cols)
    op.free()
    ctx.close()


# ---------------------------------------------------------------- B. one product per form ----

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("form,name", [p for p in PAIRS if K.shape(p.values[1]).apply])
def test_product(form, name, dt):
    s = K.shape(name)
    ctx, sy = K.context(s, dt)
    op, want = K.build(ctx, form, s, dt)
    if sy != 0:
        op.with_spaces(0, sy)
    lib = ctx.lib
    x = np.random.default_rng(sum(map(ord, form + name))).standard_normal(s.n_cols).astype(dt)
    xv = ctx.from_host(x)
    for name_k in ("pipe", "compact"):
        with kernel(name_k):
            y = kk.apply(op, xv).to_host()
            ran = lib.b2k_debug_spmv_kernel()
        assert K.same(y, R.csr_rows(*want, x, dt, None, name_k)), name_k
        if s.nnz > 0:
            assert ran == (3 if name_k == "compact" and lib.b2k_debug_csr_format(op.h) else 2)
    op.free()
    ctx.close()


# ---------------------------------------------------------------- C. stencil assembly ----

GRIDS = [(1, 1, 1), (9, 1, 1), (1, 9, 1), (1, 1, 9), (257, 3, 1), (17, 5, 9)]
# seven distinct coefficients, so a swapped neighbour shows; 0.1, -1.3, 4.1, ... are rounded by (T)c[k] in Float32
C7 = (4.1, -1.3, -0.7, -1.9, -0.45, -1.1, 0.1)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("grid", GRIDS, ids=["x".join(map(str, g)) for g in GRIDS])
def test_stencil_assembly(grid, dt):
    n = int(np.prod(grid))
    ctx = kk.B200Context(n, 4, dtype=dt)
    op = kk.B200CSR.stencil(ctx, *grid, C7)
    want = K.stencil_expected(*grid, C7, dt)
    assert len(want[2]) == K.stencil_nnz(*grid)
    check_arrays(op, want, n, n)
    # transpose(stencil(c)) is stencil(c) with west / east, south / north and down / up swapped (b200krylov.h)
    t = op.transpose()
    sw = kk.B200CSR.stencil(ctx, *grid, K.swapped(C7))
    want_sw = K.stencil_expected(*grid, K.swapped(C7), dt)
    check_arrays(sw, want_sw, n, n)
    _, got_t = K.download(t)
    assert all(K.same(a, b) for a, b in zip(got_t, want_sw))
    x = np.random.default_rng(n).standard_normal(n).astype(dt)
    with kernel("pipe"):
        y = kk.apply(op, ctx.from_host(x)).to_host()
    assert K.same(y, R.csr_rows(*want, x, dt, None, "pipe"))
    ctx.close()


# ---------------------------------------------------------------- D. dense upload ----

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("pad", [0, 13], ids=["ld=m", "ld>m"])
def test_dense_upload(pad, dt):
    m, n = 77, 11
    ld = m + pad
    A = np.random.default_rng(5).standard_normal((m, n)).astype(dt)
    assert np.all(A != 0)                    # no -0 entry: A e_j returns column j's bits
    H = np.full((ld, n), np.nan, dtype=dt, order="F")
    H[:m] = A
    ctx = kk.B200Context(m, 4, dtype=dt)
    sv = ctx.add_space(n, 4, sharded=False)
    h = L.c_op()
    ctx.check(ctx.lib.b2k_op_create_dense(ctx.h, C.byref(h), m, n, H.ctypes.data, ld))
    op = kk.B200Dense(ctx, h)
    op.space_in, op.space_out = sv, 0
    for j in (0, 1, n // 2, n - 1):
        e = np.zeros(n, dtype=dt)
        e[j] = 1
        assert K.same(kk.apply(op, ctx.from_host(e, space=sv)).to_host(), A[:, j]), j
    ctx.close()


# ---------------------------------------------------------------- E. refusals ----

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("row", K.BAD, ids=K.BAD_IDS)
def test_refusal(row, dt):
    ctx = kk.B200Context(K.N0, 4, dtype=dt)
    ctx.add_space(K.N1, 4, sharded=False)
    out = L.c_op()
    assert K.call(ctx.lib, ctx, row, out) == row.code, ctx.lib.b2k_last_error(ctx.h)
    assert not out.value
    # the context still builds and applies an operator
    rp, ci, va = K.valid_csr()
    op = kk.B200CSR.from_csr_arrays(ctx, K.N0, K.N0, rp, ci, va)
    want = K.csr_expected(rp, ci, va, 0, dt)
    check_arrays(op, want, K.N0, K.N0)
    x = np.linspace(-1, 2, K.N0).astype(dt)
    assert K.same(kk.apply(op, ctx.from_host(x)).to_host(), R.csr_rows(*want, x, dt, None, "compact"))
    ctx.close()
