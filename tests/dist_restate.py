"""Host restatement of the row-sharded path (csrc/dist.cu, the halo plan and reads of spmv.cu, the rank-ordered sums of
csrc/tsk.cuh and csrc/basis.cu), composed from the single-GPU restatements spmv_restate.py and tsk_restate.py, bit for
bit in Float64 and Float32.

Rank p owns the rows [r0_p, r0_p + n_p) of every vector and of the operator; its sums are the single-GPU ones over
those rows, and every cross-rank value is the rank-order fold of the ranks' doubles:
    fold(d) = ((0.0 + d_0) + d_1) + ... + d_{R-1}
which is what peer_sum1 (SpMV alpha, ||w||^2), k_peer_allreduce (b2k_allreduce over the peer window: inner, norm,
b2k_op_apply_dot, the synchronous step's coefficients) and, since coef_ranksum, the chained step's coefficients compute.
Every rank adds the same doubles in the same order, so every rank holds the same bits.

SpMV.  Rank p's rows gather from the global operand with the global columns (the halo holds exactly the entries of
the neighbours' rows the local rows reference, and localising the columns keeps the CSR order inside each row), so
y_p = spmv_restate.apply(..., x_p, gather=(x, r0_p)): the rows of the global restatement, with the epilogue (shift,
xscale, vout, dot_self, dot_sub) on the rank's row-aligned slices.  The tiles are finish_csr's partition of the local
row pointer, the grid the one rank p launched.  b2k_debug_apply_fused returns this local partial d_p (no cross-rank
sum: its SpmvFuse carries no alpha sequence); b2k_op_apply_dot returns fold(d).  The matrix-free stencil is the global
grid's rows r0_p, r0_p + 1, ... (shards of whole grid lines or planes).

BLAS-1.  inner and norm: rank p's partial is the double a one-rank context on the same device gives for the same
local slice (same n, so the same grid); inner = fold(partials), norm = sqrt(fold(squared-norm partials)).

One CGS2 Lanczos step (b2k_lanczos_expand, one classical pass, K1 <= kcap).  With P = [V, v] the local panel:
    v_p    = rn(T(1 / beta_old) r_p)
    w_p, d_p = the SpMV rows and fused dot (dotv = v) of rank p;      alpha0 = fold(d)
    x_p    = tsk_restate.prologue(w_p, V_p[:, -1], v_p, beta_old, alpha0)
    c_p    = tsk_restate.colsum(project_partials(P_p, x_p)) with rank p's sweep grid min(#SMs, ceil(n_p / 256))
    h      = fold(c) elementwise;   w'_p = tsk_restate.update(P_p, x_p, coefs(h, -1))
    ||w||^2 = fold(normsum(norm_partials(w'_p)));   alpha = alpha0 + h[k];   beta = sqrt(||w||^2)
The synchronous step reduces c_p with k_finalize and all-reduces the K1 doubles (k_peer_allreduce).  The chained step
(b2k_lanczos_expand_many) forms c_p in peer_boundary: the last CTA of rank p to reach the phase boundary runs
coef_colsum over the rank's per-CTA partials (G = the local grid, stride B2K_KSTRIDE, coef_lanes(K1) lanes: lane l adds
partials l, l + L, ... from 0.0, then an xor tree) and stores the K1 doubles into slot [COEF][parity][p] of every
rank's window; the update phase and the finaliser read the R sets (stride PEER_SLOT) through coef_ranksum, the same
fold.  The finaliser's ||w||^2 is finalize_block's 16-lane partial_lane_sum over the local part_n (normsum), folded by
peer_sum1; alpha0 is peer_sum1 of the SpMV partials; so the record {alpha0, alpha, beta, 1/beta, ||w||^2} is the
synchronous step's, on every rank.
"""
import numpy as np

import spmv_restate as R
import tsk_restate as ts

f64 = np.float64


def fold(parts):
    """((0.0 + d_0) + d_1) + ...: the rank-order sum of doubles (elementwise for arrays)"""
    a = np.zeros_like(np.asarray(parts[0], dtype=f64))
    for d in parts:
        a = a + np.asarray(d, dtype=f64)
    return a


def offsets(sizes):
    return np.r_[0, np.cumsum(sizes)].astype(np.int64)


def local_csr(rowptr, cols, vals, r0, n):
    """rank rows [r0, r0 + n) of a global CSR: local row pointer, the GLOBAL columns, the values"""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    a, b = rowptr[r0], rowptr[r0 + n]
    return rowptr[r0:r0 + n + 1] - a, np.asarray(cols[a:b], dtype=np.int64), np.asarray(vals[a:b])


def spmv(fma, dt, kernel, grid, xg, r0, n, *, csr=None, stencil=None, dotv=None, dsub=None, **kw):
    """(y, vout, dot partial) of rank rows [r0, r0 + n): csr = the rank's local_csr, stencil = the global grid;
    dotv / dsub are global vectors (the rank uses their slices)"""
    sl = slice(r0, r0 + n)
    xg = np.asarray(xg, dtype=dt)
    src = dict(stencil=stencil) if kernel == "stencil" else dict(csr=csr, rowblk=R.tiles(csr[0]))
    return R.apply(fma, dt, kernel, grid, xg[sl], gather=(xg, r0),
                   dotv=None if dotv is None else np.asarray(dotv)[sl],
                   dsub=None if dsub is None else np.asarray(dsub)[sl], **src, **kw)


def band_csr(n, lo, hi, seed, ints=False):
    """about 6 random columns per row in [r - lo, r + hi] (lo != hi: unequal lower and upper halos)"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 9, n)
    rowptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    rows = np.repeat(np.arange(n), lens)
    cols = np.clip(rows + rng.integers(-lo, hi + 1, rowptr[-1]), 0, n - 1)
    vals = rng.integers(-4, 5, rowptr[-1]).astype(f64) if ints else rng.standard_normal(rowptr[-1])
    return rowptr, cols, vals


def fold_case(dt, nranks):
    """the data on which the rank-order fold of the SpMV dot partials differs from the reverse fold, from
    coef_colsum's lane tree and from the unsharded launch (test_dist_restate.py pins it): shards of 2100, 1300 and
    2600 rows (two ranks: 3400 and 2600), a band operator with halos of 57 rows below and 9 above, and a dot vector
    scaled by 1, 2^-20 and -1 on the three shards.  (sizes, csr, x, v)"""
    sizes3 = [2100, 1300, 2600]
    n = sum(sizes3)
    rowptr, cols, vals = band_csr(n, 57, 9, 7)
    rng = np.random.default_rng(28)
    x = rng.standard_normal(n).astype(dt)
    v = rng.standard_normal(n)
    off = offsets(sizes3)
    for p, s in enumerate([1.0, 2.0 ** -20, -1.0]):
        v[off[p]:off[p + 1]] *= s
    sizes = sizes3 if nranks == 3 else [3400, 2600]
    return sizes, (rowptr, cols, vals.astype(dt)), x, v.astype(dt)


def stencil_csr(nx, ny, nz, coeffs, dt):
    """the assembled stencil of b2k_op_create_stencil as a global CSR (k_stencil_fill's order: ascending columns)"""
    n, plane = nx * ny * nz, nx * ny
    g = np.arange(n)
    ix, iy, iz = g % nx, (g // nx) % ny, g // plane
    terms = [((nz > 1) & (iz > 0), 5, -plane), (iy > 0, 3, -nx), (ix > 0, 1, -1), (g >= 0, 0, 0),
             (ix < nx - 1, 2, 1), (iy < ny - 1, 4, nx), ((nz > 1) & (iz < nz - 1), 6, plane)]
    cnt = sum(m.astype(np.int64) for m, _, _ in terms)
    rowptr = np.r_[0, np.cumsum(cnt)].astype(np.int64)
    cols = np.empty(rowptr[-1], dtype=np.int64)
    vals = np.empty(rowptr[-1], dtype=dt)
    pos = rowptr[:-1].copy()
    for m, c, off in terms:
        cols[pos[m]] = g[m] + off
        vals[pos[m]] = dt(coeffs[c])
        pos[m] += 1
    return rowptr, cols, vals


def lanczos_step(fma, dt, sizes, V, r, beta_old, csr, spmv_kernel, spmv_grids, nsm):
    """one synchronous CGS2 step on the row shards (module docstring).  V: global n x k (q_0 ... q_{k-2}, v_prev),
    r: global residual, csr: the global operator, spmv_grids[p]: rank p's SpMV grid.  Returns (per-rank w, global v,
    alpha0, alpha, beta, ||w||^2)"""
    off = offsets(sizes)
    v = (dt(1.0 / beta_old) * np.asarray(r, dtype=dt)).astype(dt)
    ws, ds = [], []
    for p, n in enumerate(sizes):
        w, _, d = spmv(fma, dt, spmv_kernel, spmv_grids[p], v, off[p], n, csr=local_csr(*csr, off[p], n), dotv=v)
        ws.append(w)
        ds.append(d)
    alpha0 = float(fold(ds))
    xs, cs = [], []
    for p, n in enumerate(sizes):
        sl = slice(off[p], off[p] + n)
        x = ts.prologue(ws[p], V[sl, -1], v[sl], beta_old, alpha0, fma)
        Q = np.column_stack([V[sl], v[sl]])
        xs.append(x)
        cs.append(ts.colsum(ts.project_partials(Q, x, nsm, fma)))
    h = fold(cs)
    out, n2s = [], []
    for p, n in enumerate(sizes):
        sl = slice(off[p], off[p] + n)
        Q = np.column_stack([V[sl], v[sl]])
        w = ts.update(Q, xs[p], ts.coefs(h, -1.0, dt), fma)
        out.append(w)
        n2s.append(ts.normsum(ts.norm_partials(w, nsm, fma)))
    n2 = float(fold(n2s))
    return out, v, alpha0, alpha0 + float(h[-1]), float(np.sqrt(n2)), n2
