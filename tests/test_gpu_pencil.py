"""GPU tests of the pencil entry points (b2k_pencil_create / _apply / _rayleigh) and the fused two-operator SpMV
k_spmv_pencil, in Float32 and Float64.

ax, bx and w are compared bit for bit with the composition of existing calls (b2k_op_apply with A and B, then
b2k_vec_axpby) and with a host restatement: products rounded in T and summed in CSR order in T; a row longer than the
1536-nonzero tile as a double sum in the kernel's thread / warp order, rounded once; then w = fma(-ρ, bx, ax) and
w = fma(-β, vprev, w) with libm's fma (a gcc-built helper, as in test_gpu_blas1.py).  The dots are checked bit for bit
with spmv_restate's k_spmv_pipe order at the pencil's grid, exactly on small integers and within the Higham bound of
b2k_vec_inner.  Shapes: sizes 1 and 255-257, one tile exactly full, rows
straddling tiles, a long row, and an odd size of millions of rows derived from the SM count.
"""
import ctypes as C
import subprocess
import zlib

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L

import spmv_restate as R

f64, f32 = np.float64, np.float32
SP_NNZ = 1536

_FMA_C = r"""
#include <math.h>
#include <stddef.h>
void vfma_f64(size_t n, const double* a, const double* b, const double* c, double* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fma(a[i], b[i], c[i]);
}
void vfma_f32(size_t n, const float* a, const float* b, const float* c, float* out) {
    for (size_t i = 0; i < n; ++i) out[i] = fmaf(a[i], b[i], c[i]);
}
"""


@pytest.fixture(scope="module")
def fma(tmp_path_factory):
    d = tmp_path_factory.mktemp("pfma")
    src, so = d / "vfma.c", str(d / "libvfma.so")
    src.write_text(_FMA_C)
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, str(src), "-lm"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)

    def f(a, b, c, dt):
        a, b, c = (np.ascontiguousarray(t, dtype=dt) for t in np.broadcast_arrays(
            np.asarray(a, dtype=dt), np.asarray(b, dtype=dt), np.asarray(c, dtype=dt)))
        out = np.empty(a.shape, dtype=dt)
        fn = lib.vfma_f64 if dt == f64 else lib.vfma_f32
        fn(C.c_size_t(out.size), C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), C.c_void_p(c.ctypes.data),
           C.c_void_p(out.ctypes.data))
        return out
    return f


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def spmv_restated(M, x, dt):
    """k_spmv_pipe's rounding: products in T, summed per row in CSR order in T; rows of > SP_NNZ nonzeros: double
    sums over 256 threads (thread t takes t, t + 256, ...), warp butterflies, the 8 warps in order, rounded once."""
    n = M.shape[0]
    lens = np.diff(M.indptr)
    prod = (M.data.astype(dt) * x.astype(dt)[M.indices]).astype(dt)
    y = np.zeros(n, dtype=dt)
    short = lens <= SP_NNZ
    L_ = int(lens[short].max(initial=0))
    for p in range(L_):
        rows = np.nonzero(short & (lens > p))[0]
        y[rows] = (y[rows] + prod[M.indptr[rows] + p]).astype(dt)
    for r in np.nonzero(~short)[0]:
        pr = prod[M.indptr[r]:M.indptr[r + 1]].astype(np.float64)
        acc = np.zeros(256)
        for t in range(256):
            s = 0.0
            for v in pr[t::256]:
                s += v
            acc[t] = s
        tot = 0.0
        for w in range(8):
            v = acc[32 * w:32 * w + 32].copy()
            for o in (16, 8, 4, 2, 1):
                v = v + v[np.arange(32) ^ o]
            tot += v[0]
        y[r] = dt(tot)
    return y


def random_pattern(rng, n, per_row):
    rows = np.repeat(np.arange(n), per_row)
    cols = rng.integers(0, n, size=rows.size)
    M = sp.csr_matrix((np.ones(rows.size), (rows, cols)), shape=(n, n))
    M.sum_duplicates()
    M.sort_indices()
    return M


def shape(name, rng):
    """(pattern, description) for the named shape"""
    if isinstance(name, int):
        return random_pattern(rng, name, 5)
    if name == "full_tile":             # one row of exactly SP_NNZ nonzeros: a tile exactly full
        n = 2 * SP_NNZ
        M = random_pattern(rng, n, 3).tolil()
        M[7, :] = 0.0
        M[7, :SP_NNZ] = 1.0
        return M.tocsr()
    if name == "straddle":              # 700-nonzero rows: two per tile, every third row starts a new one
        n = 3000
        M = random_pattern(rng, n, 3).tolil()
        for r in range(0, 60, 3):
            M[r, rng.choice(n, 700, replace=False)] = 1.0
        return M.tocsr()
    if name == "long":                  # rows longer than a tile take the long-row branch
        n = 5000
        M = random_pattern(rng, n, 4).tolil()
        M[11, :] = 0.0
        M[11, :SP_NNZ + 1] = 1.0
        M[4000, rng.choice(n, 4321, replace=False)] = 1.0
        return M.tocsr()
    if name == "millions":              # an odd size of millions of rows: every CTA runs many tiles
        return random_pattern(rng, 20_000 * num_sms() + 1, 5)
    raise ValueError(name)


SHAPES = [1, 255, 256, 257, "full_tile", "straddle", "long", "millions"]


def with_values(P, rng, dt):
    A = P.copy()
    A.data = rng.standard_normal(P.nnz).astype(dt)
    B = P.copy()
    B.data = (rng.random(P.nnz) + 0.5).astype(dt)
    return A, B


def explicit_zero(B):
    """B with one more stored entry, an explicit zero: the same matrix with another pattern"""
    row0 = set(B.indices[B.indptr[0]:B.indptr[1]].tolist())
    c = next(c for c in range(B.shape[1]) if c not in row0)
    coo = B.tocoo()
    Z = sp.csr_matrix((np.append(coo.data, 0.0).astype(B.dtype), (np.append(coo.row, 0), np.append(coo.col, c))),
                      shape=B.shape)
    Z.sort_indices()
    assert Z.nnz == B.nnz + 1
    return Z


def upload(ctx, M):
    return kk.B200CSR.from_csr_arrays(ctx, M.shape[0], M.shape[1], M.indptr, M.indices, M.data)


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("name", SHAPES)
def test_apply_and_rayleigh_bitwise(fma, dt, name):
    rng = np.random.default_rng(zlib.crc32(f"{name}-{np.dtype(dt).name}".encode()))
    Pat = shape(name, rng)
    n = Pat.shape[0]
    A, B = with_values(Pat, rng, dt)
    ctx = kk.B200Context(n, 16, dtype=dt)
    try:
        dA, dB = upload(ctx, A), upload(ctx, B)
        P = kk.B200Pencil(dA, dB)
        x = rng.standard_normal(n).astype(dt)
        vp = rng.standard_normal(n).astype(dt)
        xd, vpd = ctx.from_host(x), ctx.from_host(vp)
        ax_ref, bx_ref = spmv_restated(A, x, dt), spmv_restated(B, x, dt)
        # the composition of existing calls
        axc, bxc = dA(xd), dB(xd)
        np.testing.assert_array_equal(axc.to_host(), ax_ref)
        np.testing.assert_array_equal(bxc.to_host(), bx_ref)
        for rho in (0.0, 0.37):
            for use_prev in (False, True):
                w, bx = ctx.empty(), ctx.empty()
                l0 = ctx.launches
                dot = P.apply_into(xd, w, bx, rho, vpd if use_prev else None, 0.61, dot=True)
                assert ctx.launches - l0 == 1 and L.load().b2k_debug_pencil_path() == 1
                wref = fma(-rho, bx_ref, ax_ref, dt)
                if use_prev:
                    wref = fma(-0.61, vp, wref, dt)
                wc = axc.copy().add_(bxc, -rho)
                if use_prev:
                    wc = wc.add_(vpd, -0.61)
                np.testing.assert_array_equal(bx.to_host(), bx_ref)
                np.testing.assert_array_equal(w.to_host(), wref)
                np.testing.assert_array_equal(w.to_host(), wc.to_host())
                exact = float(np.dot(x.astype(np.float64), w.to_host().astype(np.float64)))
                bound = 2 * n * np.finfo(dt).eps * float(np.dot(np.abs(x).astype(np.float64),
                                                                  np.abs(w.to_host()).astype(np.float64)))
                assert abs(dot - exact) <= bound + 1e-300
                assert abs(dot - xd.inner(w)) <= 2 * bound + 1e-300
                w2, bx2 = ctx.empty(), ctx.empty()
                dot2 = P.apply_into(xd, w2, bx2, rho, vpd if use_prev else None, 0.61, dot=True)
                assert dot2 == dot
                np.testing.assert_array_equal(w2.to_host(), w.to_host())
        ax, bx = ctx.empty(), ctx.empty()
        xax, xbx = P.rayleigh_into(xd, ax, bx)
        np.testing.assert_array_equal(ax.to_host(), ax_ref)
        np.testing.assert_array_equal(bx.to_host(), bx_ref)
        for d, y in ((xax, ax_ref), (xbx, bx_ref)):
            exact = float(np.dot(x.astype(np.float64), y.astype(np.float64)))
            bound = 2 * n * np.finfo(dt).eps * float(np.dot(np.abs(x).astype(np.float64), np.abs(y).astype(np.float64)))
            assert abs(d - exact) <= bound + 1e-300
        P.free()
    finally:
        ctx.close()


def device_tiles(op):
    lib, nblk = L.load(), C.c_int32()
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, None, C.byref(nblk)) == L.OK
    rb = np.empty(nblk.value + 1, dtype=np.int32)
    assert lib.b2k_debug_op_tiles(op.ctx.h, op.h, rb.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nblk)) == L.OK
    return rb.astype(np.int64)


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("name", SHAPES)
def test_dots_bitwise(fma, dt, name):
    """<x, w> (MODE 0, with and without vprev), <x, Ax> and <x, Bx> (MODE 1) bit for bit with k_spmv_pipe's dot order
    at the pencil's grid (3 CTAs per SM in Float64, 4 in Float32): per consumer thread an fma chain in T over its rows,
    the CTA's warps in order, the last CTA adding the partials in CTA order"""
    rng = np.random.default_rng(zlib.crc32(f"dots-{name}-{np.dtype(dt).name}".encode()))
    Pat = shape(name, rng)
    n = Pat.shape[0]
    A, B = with_values(Pat, rng, dt)
    ctx = kk.B200Context(n, 16, dtype=dt)
    try:
        dA, dB = upload(ctx, A), upload(ctx, B)
        P = kk.B200Pencil(dA, dB)
        x = rng.standard_normal(n).astype(dt)
        vp = rng.standard_normal(n).astype(dt)
        xd, vpd = ctx.from_host(x), ctx.from_host(vp)
        rowblk = device_tiles(dA)
        grid = min(len(rowblk) - 1, (3 if dt == f64 else 4) * num_sms())
        gid, rank = R.csr_threads(rowblk, grid)
        ax_ref, bx_ref = spmv_restated(A, x, dt), spmv_restated(B, x, dt)
        for use_prev in (False, True):
            w, bx = ctx.empty(), ctx.empty()
            dot = P.apply_into(xd, w, bx, 0.37, vpd if use_prev else None, 0.61, dot=True)
            wref = fma(-0.37, bx_ref, ax_ref, dt)
            if use_prev:
                wref = fma(-0.61, vp, wref, dt)
            np.testing.assert_array_equal(w.to_host(), wref)
            assert dot == R.dot(fma, dt, x, wref, gid, rank, grid, "pipe"), use_prev
        ax, bx = ctx.empty(), ctx.empty()
        xax, xbx = P.rayleigh_into(xd, ax, bx)
        assert xax == R.dot(fma, dt, x, ax_ref, gid, rank, grid, "pipe")
        assert xbx == R.dot(fma, dt, x, bx_ref, gid, rank, grid, "pipe")
        P.free()
    finally:
        ctx.close()


@pytest.mark.parametrize("dt", [f64, f32])
def test_dots_exact_on_small_integers(dt):
    rng = np.random.default_rng(5)
    Pat = random_pattern(rng, 100_003, 5)
    A, B = Pat.copy(), Pat.copy()
    A.data = rng.integers(-3, 4, Pat.nnz).astype(dt)
    B.data = rng.integers(1, 4, Pat.nnz).astype(dt)
    x = rng.integers(-2, 3, Pat.shape[0]).astype(dt)
    ctx = kk.B200Context(Pat.shape[0], 8, dtype=dt)
    try:
        P = kk.B200Pencil(upload(ctx, A), upload(ctx, B))
        xd = ctx.from_host(x)
        ax, bx = ctx.empty(), ctx.empty()
        xax, xbx = P.rayleigh_into(xd, ax, bx)
        assert xax == float(x.astype(np.float64) @ (A @ x.astype(np.float64)))
        assert xbx == float(x.astype(np.float64) @ (B @ x.astype(np.float64)))
        w, bx = ctx.empty(), ctx.empty()
        dot = P.apply_into(xd, w, bx, 2.0, None, 0.0, dot=True)
        assert dot == float(x.astype(np.float64) @ (A @ x - 2.0 * (B @ x)).astype(np.float64))
    finally:
        ctx.close()


@pytest.mark.parametrize("dt", [f64, f32])
def test_path_hook_and_composed_bits(fma, dt):
    rng = np.random.default_rng(9)
    nx, ny = 40, 30
    n = nx * ny
    ctx = kk.B200Context(n, 24, dtype=dt)
    try:
        K = kk.B200CSR.stencil(ctx, nx, ny)
        M = kk.B200CSR.stencil(ctx, nx, ny, coeffs=(1.5, -0.125, -0.125, -0.125, -0.125, 0, 0))
        Kf = kk.B200CSR.stencil_free(ctx, nx, ny)
        Ms = M.to_scipy()
        Mz = upload(ctx, explicit_zero(Ms))
        D = kk.B200Dense.from_host(ctx, np.diag(np.arange(1.0, n + 1)), 0)
        x = ctx.from_host(rng.standard_normal(n).astype(dt))
        outs = {}
        for label, pair, path in (("same", (K, M), 1), ("pattern", (K, Mz), 0), ("free", (Kf, M), 0),
                                  ("dense", (K, D), 0)):
            P = kk.B200Pencil(*pair)
            w, bx = ctx.empty(), ctx.empty()
            P.apply_into(x, w, bx, 0.3)
            assert L.load().b2k_debug_pencil_path() == path, label
            outs[label] = (w.to_host(), bx.to_host())
            P.free()
        for label in ("pattern", "free"):
            np.testing.assert_array_equal(outs[label][0], outs["same"][0])
            np.testing.assert_array_equal(outs[label][1], outs["same"][1])
    finally:
        ctx.close()


def test_refusals_write_nothing():
    rng = np.random.default_rng(3)
    Pat = random_pattern(rng, 1000, 4)
    A, B = with_values(Pat, rng, f64)
    ctx = kk.B200Context(1000, 16)
    other = kk.B200Context(1000, 8)
    try:
        sp_short = ctx.add_space(999, 4)
        dA, dB = upload(ctx, A), upload(ctx, B)
        oA = upload(other, A)
        P = kk.B200Pencil(dA, dB)
        vs = [ctx.from_host(rng.standard_normal(1000)) for _ in range(4)]
        short = ctx.from_host(np.ones(999), space=sp_short)
        ov = [other.from_host(np.ones(1000)) for _ in range(3)]
        before = [v.to_host() for v in vs] + [short.to_host()] + [v.to_host() for v in ov]
        lib, h = ctx.lib, ctx.h
        x, w, bx, vp = (v.handle for v in vs)
        d = C.c_double(12345.0)
        h_out = C.c_void_p()
        cases = [
            (L.EINVAL, lambda: lib.b2k_pencil_apply(h, None, x, w, bx, 1.0, -1, 0.0, C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_apply(h, P.h, x, x, bx, 1.0, -1, 0.0, C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_apply(h, P.h, x, w, w, 1.0, -1, 0.0, C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_apply(h, P.h, x, w, bx, 1.0, x, 0.5, C.byref(d))),
            (L.EDIM, lambda: lib.b2k_pencil_apply(h, P.h, x, w, short.handle, 1.0, -1, 0.0, C.byref(d))),
            (L.EDIM, lambda: lib.b2k_pencil_apply(h, P.h, x, w, bx, 1.0, short.handle, 0.5, C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_rayleigh(h, P.h, x, x, bx, C.byref(d), C.byref(d))),
            (L.EDIM, lambda: lib.b2k_pencil_rayleigh(h, P.h, short.handle, w, bx, C.byref(d), C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_apply(other.h, P.h, *(v.handle for v in ov), 1.0, -1, 0.0,
                                                    C.byref(d))),
            (L.EINVAL, lambda: lib.b2k_pencil_create(h, C.byref(h_out), dA.h, dA.h)),
            (L.EINVAL, lambda: lib.b2k_pencil_create(h, C.byref(h_out), dA.h, oA.h)),
            (L.EINVAL, lambda: lib.b2k_pencil_create(h, None, dA.h, dB.h)),
        ]
        launches = ctx.launches
        for code, call in cases:
            assert call() == code
        assert ctx.launches == launches and d.value == 12345.0 and h_out.value is None
        after = [v.to_host() for v in vs] + [short.to_host()] + [v.to_host() for v in ov]
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
        with pytest.raises(L.DimensionMismatch):
            kk.B200Pencil(dA, upload(ctx, sp.identity(1000, format="csr")[:, :999].tocsr()))
    finally:
        other.close()
        ctx.close()
