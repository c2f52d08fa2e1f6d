"""Host restatement of the summation order of the one-pass dense Golub-Kahan-Lanczos step (csrc/onepass_kernels.cuh,
driven from csrc/spmv.cu: b2k_op_apply_normal_gram): y = A x and z = A'(A x), bit for bit in Float32 and Float64.

`fma` is fma(a, b, c, T): the correctly rounded a·b + c elementwise in T, arguments broadcast and cast to T first
(`load_fma` builds one from libm; test_gpu_blas1.py's module fixture is the same function).  Every other operation is
a numpy operation in T or in float64, each rounded once, every accumulator starts at +0.

Matrix.  A is m x n column-major with leading dimension ld = 32 ceil(m / 32); rows [m, ld) are zero (alloc_dense
memsets them), and the kernels read them: their y is 0 and their products enter z as zeros.

VARIANT A, k_dense_onepass<T, NZ> (NZ = 1, 2, 4, 7 for n <= 256, 512, 1024, else).  32-row tiles, ntiles = ld / 32,
grid = min(ntiles, occupancy · #SMs) CTAs of 256 threads; CTA b takes tiles b, b + grid, ... in order.
VEC = 16 / sizeof(T) rows per load, VPC = 32 / VEC loads per tile column, CSTEP = 256 / VPC (32 f32, 16 f64) column
classes.  Thread tid holds rows VEC·(tid % VPC) ... + VEC - 1 of the tile and column class c0 = tid / VPC:
    y:  acc = fma(A[row, c], x[c], acc) over c = c0, c0 + CSTEP, ... < n (increasing);
        butterfly acc += shfl_xor(acc, off), off = VPC, 2 VPC, ... < 32: warp w holds classes CW·w ... CW·w + CW - 1
        (CW = 32 / VPC: 4 f32, 2 f64) and gives (a0 + a1) + (a2 + a3) in f32, a0 + a1 in f64;
        y_row = ((0 + W0) + W1) + ... + W7 over the 8 warps, in T (rows >= m are formed, not stored).
    z:  per tile, thread <-> column c: p = fma(A[row, c], y_row, p) over the tile's rows 0 ... 31 in T;
        per CTA, zacc += (double) p over its tiles in order: zpart[b, c].
VARIANT B, k_dense_onepass_w (Float32, n <= 512, b2k_debug_set_onepass_variant(1)).  64-row tiles,
ntiles = ceil(ld / 64) (the last tile is half outside A when ld = 32 mod 64: those rows load as zero),
grid = min(ntiles, #SMs) CTAs of 512 threads.  VPC = 16, CSTEP = 32: class c0 = tid / 16 takes columns c0 + 32 u,
u < 16; butterfly off = 16 only (a0 + a1); y in order over the 16 warps; z per tile: p0 over the even rows, p1 over
the odd rows (fma chains in f32), zacc += (double)(p0 + p1).
REDUCTION, k_onepass_reduce.  Column c, group g = 0 ... 7 takes partials g, g + 8, ...: while p + 24 < grid four
running sums take p, p + 8, p + 16, p + 24 and p advances by 32; the rest goes into s0 in steps of 8;
red_g = (s0 + s1) + (s2 + s3); dres = ((red0 + red1) + ...) + red7 (starting from red0); z = T(dres).
ROW-SHARDED (onepass_finish with a sharded y): the ranks' dres are summed in rank order from 0.0 (peer_sum1, in
slot-sized pieces of 1024 columns: the order per column is the same), then z = T(sum) on every rank (k_onepass_store).

`butterfly` and `grouped` switch to a different, equally plausible order (a sequential warp sum, a plain in-order sum
of the partials): the negative controls that show a comparison tells the orders apart.
"""
import ctypes as C
import os
import subprocess

import numpy as np

f64, f32 = np.float64, np.float32
OP_T, OP_ROWS, OP_ZMAX = 256, 32, 7
OPW_T, OPW_ROWS = 512, 64

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


def load_fma(directory):
    """fma(a, b, c, T) through libm's fma / fmaf, from a helper compiled into `directory`"""
    src, so = os.path.join(directory, "vfma.c"), os.path.join(directory, "libvfma.so")
    with open(src, "w") as f:
        f.write(_FMA_C)
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stderr)
    lib = C.CDLL(so)

    def fma(a, b, c, dt):
        a, b, c = (np.ascontiguousarray(t, dtype=dt) for t in np.broadcast_arrays(
            np.asarray(a, dtype=dt), np.asarray(b, dtype=dt), np.asarray(c, dtype=dt)))
        out = np.empty(a.shape, dtype=dt)
        fn = lib.vfma_f64 if dt == f64 else lib.vfma_f32
        fn(C.c_size_t(out.size), C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), C.c_void_p(c.ctypes.data),
           C.c_void_p(out.ctypes.data))
        return out
    return fma


def ld_of(m):
    return 32 * -(-m // 32)


def nz_of(n):
    """columns per thread in phase 2 of variant A: the template instance"""
    return 1 if n <= OP_T else 2 if n <= 2 * OP_T else 4 if n <= 4 * OP_T else OP_ZMAX


def ntiles_of(m, variant):
    ld = ld_of(m)
    return ld // OP_ROWS if variant == 0 else -(-ld // OPW_ROWS)


def padded(A, rows):
    """A (m x n, T) with zero rows appended up to `rows`"""
    P = np.zeros((rows, A.shape[1]), dtype=A.dtype)
    P[:A.shape[0]] = A
    return P


def _xor_tree(v, axis_len, butterfly):
    """the shuffle butterfly over the CW column classes of a warp (last axis); element 0 is what lane < VPC stores"""
    if not butterfly:                                    # negative control: a sequential sum of the classes
        s = v[..., 0]
        for k in range(1, axis_len):
            s = s + v[..., k]
        return s
    idx = np.arange(axis_len)
    o = 1
    while o < axis_len:
        v = v + v[..., idx ^ o]
        o <<= 1
    return v[..., 0]


def _y_rows(Ap, x, cstep, nwarps, fma, butterfly):
    """y of every row of the padded matrix: per-class fma chains, the warp butterfly, the warps in order"""
    dt = Ap.dtype.type
    rows, n = Ap.shape
    acc = np.zeros((rows, cstep), dtype=dt)
    c0 = np.arange(cstep)
    for k in range(-(-n // cstep)):
        cols = c0 + k * cstep
        ok = cols < n
        cv = cols[ok]
        acc[:, ok] = fma(Ap[:, cv], x[cv][None, :], acc[:, ok], dt)
    cw = cstep // nwarps
    W = _xor_tree(acc.reshape(rows, nwarps, cw), cw, butterfly)
    y = np.zeros(rows, dtype=dt)
    for w in range(nwarps):
        y = y + W[:, w]
    return y


def _cta_partials(P, grid):
    """zpart[b] = sum over CTA b's tiles b, b + grid, ... of (double) P[tile], in order, from 0.0"""
    ntiles, n = P.shape
    zpart = np.zeros((grid, n))
    for tt in range(-(-ntiles // grid)):
        tiles = np.arange(grid) + tt * grid
        ok = tiles < ntiles
        zpart[ok] = zpart[ok] + P[tiles[ok]].astype(f64)
    return zpart


def variant_a(A, x, grid, fma, butterfly=True):
    """(y, zpart) of k_dense_onepass<T, NZ> on A (m x n, T) and x (n, T) with `grid` CTAs"""
    dt = A.dtype.type
    m, n = A.shape
    ld = ld_of(m)
    assert 1 <= grid <= ld // OP_ROWS
    vec = 16 // np.dtype(dt).itemsize
    cstep = OP_T // (OP_ROWS // vec)
    Ap = padded(A, ld)
    y = _y_rows(Ap, np.asarray(x, dtype=dt), cstep, OP_T // 32, fma, butterfly)
    At = Ap.reshape(ld // OP_ROWS, OP_ROWS, n)
    yt = y.reshape(ld // OP_ROWS, OP_ROWS)
    p = np.zeros((ld // OP_ROWS, n), dtype=dt)
    for r in range(OP_ROWS):
        p = fma(At[:, r, :], yt[:, r, None], p, dt)
    return y[:m], _cta_partials(p, grid)


def variant_b(A, x, grid, fma, butterfly=True):
    """(y, zpart) of k_dense_onepass_w on A (m x n, float32, n <= 512) and x with `grid` CTAs"""
    assert A.dtype == f32 and A.shape[1] <= 512
    m, n = A.shape
    ntiles = ntiles_of(m, 1)
    assert 1 <= grid <= ntiles
    rows = ntiles * OPW_ROWS                             # rows >= ld load as zero
    Ap = padded(A, rows)
    y = _y_rows(Ap, np.asarray(x, dtype=f32), OPW_T // (OPW_ROWS // 4), OPW_T // 32, fma, butterfly)
    At = Ap.reshape(ntiles, OPW_ROWS, n)
    yt = y.reshape(ntiles, OPW_ROWS)
    p0 = np.zeros((ntiles, n), dtype=f32)
    p1 = np.zeros((ntiles, n), dtype=f32)
    for r in range(0, OPW_ROWS, 2):
        p0 = fma(At[:, r, :], yt[:, r, None], p0, f32)
        p1 = fma(At[:, r + 1, :], yt[:, r + 1, None], p1, f32)
    return y[:m], _cta_partials(p0 + p1, grid)


def reduce(zpart, grouped=True):
    """dres of k_onepass_reduce over the grid x n partials"""
    G, n = zpart.shape
    if not grouped:                                      # negative control: the partials in CTA order
        s = np.zeros(n)
        for b in range(G):
            s = s + zpart[b]
        return s
    red = []
    for g in range(8):
        s0, s1, s2, s3 = (np.zeros(n) for _ in range(4))
        p = g
        while p + 24 < G:
            s0, s1, s2, s3 = s0 + zpart[p], s1 + zpart[p + 8], s2 + zpart[p + 16], s3 + zpart[p + 24]
            p += 32
        while p < G:
            s0 = s0 + zpart[p]
            p += 8
        red.append((s0 + s1) + (s2 + s3))
    s = red[0]
    for w in range(1, 8):
        s = s + red[w]
    return s


def rank_sum(dres_per_rank):
    """the peer all-reduce of the ranks' dres: rank order, from 0.0"""
    s = np.zeros_like(dres_per_rank[0])
    for d in dres_per_rank:
        s = s + d
    return s


def apply_normal_gram(A, x, variant, grid, fma, butterfly=True, grouped=True):
    """(y, zpart, dres, z) of one b2k_op_apply_normal_gram call with `grid` CTAs (variant 0 = A, 1 = B)"""
    y, zpart = (variant_a if variant == 0 else variant_b)(A, x, grid, fma, butterfly)
    dres = reduce(zpart, grouped)
    return y, zpart, dres, dres.astype(A.dtype)
