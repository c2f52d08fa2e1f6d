"""Operator ingestion on the numpy stand-in of the C-ABI (hostsim.py), no GPU:
1. every malformed row of op_ingest_cases.BAD returns the library's code, leaves *out NULL and leaves the context
   usable, so driver tests on the stand-in refuse what the library refuses;
2. every entry form builds the expected arrays of op_ingest_cases (the stand-in converts CSC with scipy, whose
   transpose is the same stable counting sort);
3. B200CSR.from_scipy never changes the caller's matrix, and sends sorted input as it is.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L

import hostsim
import op_ingest_cases as K

f64, f32 = np.float64, np.float32


@pytest.mark.parametrize("dt", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("row", K.BAD, ids=K.BAD_IDS)
def test_refusal(row, dt):
    with hostsim.installed() as lib:
        ctx = kk.B200Context(K.N0, 4, dtype=dt)
        ctx.add_space(K.N1, 4, sharded=False)
        out = L.c_op()
        assert K.call(lib, ctx, row, out) == row.code
        assert not out.value
        rp, ci, va = K.valid_csr()
        op = kk.B200CSR.from_csr_arrays(ctx, K.N0, K.N0, rp, ci, va)
        x = np.linspace(-1, 2, K.N0).astype(dt)
        y = kk.apply(op, ctx.from_host(x)).to_host()
        np.testing.assert_allclose(y, sp.csr_matrix((va, ci, rp), shape=(K.N0, K.N0)) @ x, rtol=1e-6)
        ctx.close()


@pytest.mark.parametrize("form,name", [pytest.param(f, s, id=f"{f}-{s}") for f, s in K.form_shape_pairs()
                                       if s not in ("gap64k", "huge-ncols")])
def test_expected_arrays(form, name):
    s = K.shape(name)
    with hostsim.installed():
        ctx, _ = K.context(s, f64)
        op, want = K.build(ctx, form, s, f64)
        info, got = K.download(op)
        assert info == (s.n_rows, s.n_cols, s.nnz, 0)
        assert all(K.same(g, w) for g, w in zip(got, want))
        ctx.close()


def test_from_scipy_leaves_the_callers_matrix_alone():
    s = K.shape("edge-rows")
    A = sp.csr_matrix((s.vals.copy(), s.cols.copy(), s.csr()[0]), shape=(s.n_rows, s.n_cols))
    indices, data = A.indices.copy(), A.data.copy()
    assert not A.has_sorted_indices
    with hostsim.installed():
        ctx = kk.B200Context(s.n_rows, 4)
        kk.B200CSR.from_scipy(ctx, A)
        ctx.close()
    assert np.array_equal(A.indices, indices) and np.array_equal(A.data, data)
    assert not A.has_sorted_indices


def test_from_scipy_sends_sorted_input_without_a_copy():
    A = sp.random(50, 50, density=0.1, format="csr", random_state=3)
    A.sort_indices()
    sent = {}

    class Spy(hostsim.HostSimLib):
        def b2k_op_create_csr(self, h, out, n_rows, n_cols, nnz, rowptr, colidx, vals, idx_bytes, index_base):
            sent["vals"] = vals
            return super().b2k_op_create_csr(h, out, n_rows, n_cols, nnz, rowptr, colidx, vals, idx_bytes,
                                             index_base)

    with hostsim.installed():
        L._lib = Spy()                                  # restored with the stand-in when the block ends
        ctx = kk.B200Context(50, 4)
        kk.B200CSR.from_scipy(ctx, A)
        ctx.close()
    assert sent["vals"] == A.data.ctypes.data          # the caller's Float64 values, sent in place


def test_row_shard_takes_more_than_2_31_global_columns():
    """A row shard's n_cols is the global column count: its columns become local or halo indices that fit int32, so
    only one GPU's operator is limited to 2^31 columns (the table's csr-ncols-2^31 row)."""
    lib = hostsim.HostSimLib()
    n_global = (1 << 31) + K.N0
    h = C.c_void_p()
    assert lib.b2k_ctx_create_dist(C.byref(h), 0, K.N0, 4, L.F64, 1, 2, None, n_global, n_global - K.N0) == L.OK
    rp = np.array(K.RP, np.int64)
    ci = np.array(K.IX, np.int64) + (n_global - K.N0)          # the shard's own columns, all >= 2^31
    ci[0] = n_global - K.N0 - 1                                   # and one halo column below them
    va = np.arange(1.0, K.NNZ + 1)
    out, nr, nc, nnz, kind = L.c_op(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    assert lib.b2k_op_create_csr(h, C.byref(out), K.N0, n_global, K.NNZ, rp.ctypes.data, ci.ctypes.data,
                                 va.ctypes.data, 8, 0) == L.OK
    assert out.value
    assert lib.b2k_op_info(out, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(kind)) == L.OK
    assert (nr.value, nc.value, nnz.value) == (K.N0, n_global, K.NNZ)
    ci[1] = n_global                                              # a column past the global count is still refused
    out2 = L.c_op()
    assert lib.b2k_op_create_csr(h, C.byref(out2), K.N0, n_global, K.NNZ, rp.ctypes.data, ci.ctypes.data,
                                 va.ctypes.data, 8, 0) == L.EINVAL
    assert not out2.value


@pytest.mark.parametrize("n,colptr,rowval,nzval", [
    (-1, [], [], []),                      # a negative column count
    (2, [1, 2], [1], [1.0]),               # colptr one entry short
    (2, [1, 2, 3], [1], [1.0, 2.0]),       # rowval shorter than colptr's nnz
    (2, [1, 2, 3], [1, 2], [1.0]),         # nzval shorter
], ids=["n-negative", "colptr-short", "rowval-short", "nzval-short"])
def test_from_julia_csc_refuses_inconsistent_arrays(n, colptr, rowval, nzval):
    with hostsim.installed():
        ctx = kk.B200Context(2, 4)
        with pytest.raises(L.B200Error):
            kk.B200CSR.from_julia_csc(ctx, 2, n, colptr, rowval, nzval)
        ctx.close()
