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


# ------------------------------------------------------------------------------ the other sharded entry points ----
#
# Every sharded entry point below sums across ranks only through b2k_allreduce, so each restatement is rank p's
# single-GPU order on its row slice (G_p = the local grid), folded where the device all-reduces:
#   b2k_basis_project     h = fold(tsk_restate.project(Q_p, x_p)), per pass of kcap columns the colsum of that pass,
#                         one all-reduce of all k doubles (slot-sized pieces past PEER_SLOT = 1024);
#   classical pass        cgs_pass_unfused_t: h = that fold, v_p = update(Q_p, v_p, coefs(h, -1)), ||v||^2 =
#                         fold(normsum(norm_partials(v_p))); fused_ok() is false on a sharded panel, so CGS, CGS2,
#                         CGSIR and MGS2B always take it;
#   k_dot                 s = fold(lsmr_restate.blas1_sum(a_p, b_p, grid_for(n_p, 8))): inner, norm, every ||v||^2
#                         of the MGS family and the vector orthogonalizer, and each s_j of mgs_sweep, which is folded
#                         before the next pipelined k_dot subtracts it (x = fma(-T(s_{j-1}), q_{j-1}, x));
#   CG / BiCGStab steps   the SpMV's fused dot (this module's spmv) and the k_cg_xr / k_bicg_s / k_bicg_xr sums, the
#                         latter in blas1_sum's order on grid_for(n_p, 8);
#   the IR loops          decide on the folded norms only, so every rank runs the same number of passes.
# A replicated space (sharded = 0) is summed on no rank: every rank's value is the one-rank restatement of the full
# vectors.

import math  # noqa: E402

import lsmr_restate as LS  # noqa: E402

EPS = {f64: 2.0 ** -52, np.float32: 2.0 ** -23}


def rows(sizes, a):
    """the rank slices of a global vector or row panel"""
    off = offsets(sizes)
    return [a[off[p]:off[p + 1]] for p in range(len(sizes))]


def dot(fma, dt, sizes, a, b, nsm):
    """k_dot on the shards, all-reduced: the fold of every rank's blas1_sum on its grid_for(n_p, 8)"""
    return float(fold([LS.blas1_sum(fma, dt, ap, bp, LS.grid_for(len(ap), 8, nsm))
                       for ap, bp in zip(rows(sizes, a), rows(sizes, b))]))


def project(fma, sizes, Q, x, nsm):
    """b2k_basis_project (and the projection of a classical pass): the fold of the ranks' per-pass colsums"""
    return fold([ts.project(Qp, xp, nsm, fma) for Qp, xp in zip(rows(sizes, Q), rows(sizes, x))])


def cgs_pass(fma, sizes, Q, v, nsm):
    """one unfused classical pass (cgs_pass_unfused_t): (h, v', ||v'||^2)"""
    dt = Q.dtype.type
    h = project(fma, sizes, Q, v, nsm)
    cs = ts.coefs(h, -1.0, dt)
    out = [ts.update(Qp, vp, cs, fma) for Qp, vp in zip(rows(sizes, Q), rows(sizes, v))]
    n2 = float(fold([ts.normsum(ts.norm_partials(w, nsm, fma)) for w in out]))
    return h, np.concatenate(out), n2


def mgs_sweep(fma, sizes, Q, v, nsm):
    """mgs_sweep: each s_j folded before the next launch subtracts it.  (s, v')"""
    dt = Q.dtype.type
    xs = [np.asarray(x, dtype=dt) for x in rows(sizes, v)]
    Qs = rows(sizes, Q)
    s = []
    for j in range(Q.shape[1]):
        if j > 0:
            xs = [fma(-dt(s[-1]), Qp[:, j - 1], x, dt) for Qp, x in zip(Qs, xs)]
        s.append(float(fold([LS.blas1_sum(fma, dt, Qp[:, j], x, LS.grid_for(len(x), 8, nsm))
                             for Qp, x in zip(Qs, xs)])))
    xs = [fma(-dt(s[-1]), Qp[:, -1], x, dt) for Qp, x in zip(Qs, xs)]
    return np.array(s), np.concatenate(xs)


def orthogonalize(fma, sizes, Q, v, alg, eta, nsm):
    """b2k_basis_orthogonalize on the shards: (h, ||v'||, passes, v')"""
    dt = Q.dtype.type
    CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)

    def one(v):
        if alg in (CGS, CGS2, MGS2B, CGSIR):
            return cgs_pass(fma, sizes, Q, v, nsm)
        s, v = mgs_sweep(fma, sizes, Q, v, nsm)
        return s, v, None

    def norm2(v, n2):
        return dot(fma, dt, sizes, v, v, nsm) if n2 is None else n2

    if alg in (CGSIR, MGSIR):
        nold = math.sqrt(dot(fma, dt, sizes, v, v, nsm))
        h, passes = np.zeros(Q.shape[1]), 0
        while True:
            hp, v, n2 = one(v)
            passes += 1
            h = h + hp
            nnew = math.sqrt(norm2(v, n2))
            if not (EPS[dt] < nnew < eta * nold):
                return h, nnew, passes, v
            nold = nnew
    passes = 2 if alg in (CGS2, MGS2, MGS2B) else 1
    h, v, n2 = one(v)
    if passes == 2:
        h2, v, n2 = one(v)
        h = h + h2
    return h, math.sqrt(norm2(v, n2)), passes, v


def vec_orthogonalize(fma, sizes, q, v, alg, eta, nsm):
    """b2k_vec_orthogonalize on the shards (every s and ||v||^2 a k_dot, all-reduced): (s, ||v'||, v', passes)"""
    dt = np.asarray(v).dtype.type
    CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)

    def step(v):
        s = dot(fma, dt, sizes, q, v, nsm)
        return s, fma(-dt(s), q, v, dt)

    if alg in (CGSIR, MGSIR):
        nold = math.sqrt(dot(fma, dt, sizes, v, v, nsm))
        s, v = step(v)
        nnew = math.sqrt(dot(fma, dt, sizes, v, v, nsm))
        passes = 1
        while EPS[dt] < nnew < eta * nold:
            nold = nnew
            s1, v = step(v)
            passes += 1
            s += s1
            nnew = math.sqrt(dot(fma, dt, sizes, v, v, nsm))
        return s, nnew, v, passes
    s, v = step(v)
    passes = 1
    if alg in (CGS2, MGS2, MGS2B):
        s1, v = step(v)
        passes = 2
        s = s + s1
    return s, math.sqrt(dot(fma, dt, sizes, v, v, nsm)), v, passes


def lanczos_expand(fma, dt, sizes, V, r, beta_old, csr, spmv_kernel, spmv_grids, nsm, alg, eta=0.0):
    """b2k_lanczos_expand on the shards for every orthogonalizer but CGS2 (lanczos_step): (w, v, alpha, beta,
    passes), w and v global, passes = 1 + the reorthogonalisation passes of CGSIR / MGSIR (1 otherwise).  CGS /
    CGSIR: the SpMV with the fused dot gives alpha0, the prologue is axpy2; CGSIR decides on beta = ||w'|| first and
    then runs classical passes over [V, v] without a prologue.  The MGS family: w -= beta_old v_prev (axpby),
    alpha0 = <v, w>, w -= alpha0 v, then nothing (MGS), one classical pass (MGS2B), one MGS sweep (MGS2) or the MGSIR
    loop of sweeps; alpha += the coefficient of v.  MGS2B takes alpha0 from the SpMV epilogue (dotv = v, dot_sub_vec
    = v_prev scaled by beta_old: the chained step's order), the others from k_dot after the SpMV."""
    CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)
    off = offsets(sizes)
    v = (dt(1.0 / beta_old) * np.asarray(r, dtype=dt)).astype(dt)
    Q = np.column_stack([V, v])
    classical = alg in (CGS, CGSIR)
    fused = classical or alg == MGS2B
    sub = dict(dsub=V[:, -1], dsc=beta_old) if alg == MGS2B else {}
    ws, ds = [], []
    for p, n in enumerate(sizes):
        w, _, d = spmv(fma, dt, spmv_kernel, spmv_grids[p], v, off[p], n, csr=local_csr(*csr, off[p], n),
                       dotv=v if fused else None, **sub)
        ws.append(w)
        ds.append(d)
    w = np.concatenate(ws)
    eps = EPS[dt]
    passes = 1
    if classical:
        alpha = float(fold(ds))
        w = ts.prologue(w, V[:, -1], v, beta_old, alpha, fma)
        beta = math.sqrt(dot(fma, dt, sizes, w, w, nsm))
        if alg == CGS:
            return w, v, alpha, beta, passes
        nold = math.sqrt(beta * beta + (alpha * alpha + beta_old * beta_old))
        if not (eps < beta < eta * nold):
            return w, v, alpha, beta, passes
        nold = beta
        while True:
            h, w, n2 = cgs_pass(fma, sizes, Q, w, nsm)
            passes += 1
            alpha += float(h[-1])
            beta = math.sqrt(n2)
            if not (eps < beta < eta * nold):
                return w, v, alpha, beta, passes
            nold = beta
    w = fma(-beta_old, V[:, -1], w, dt)
    alpha = float(fold(ds)) if alg == MGS2B else dot(fma, dt, sizes, v, w, nsm)
    w = fma(-dt(alpha), v, w, dt)
    if alg == MGS2B:
        h, w, n2 = cgs_pass(fma, sizes, Q, w, nsm)
        return w, v, alpha + float(h[-1]), math.sqrt(n2), passes
    if alg == MGS2:
        s, w = mgs_sweep(fma, sizes, Q, w, nsm)
        return w, v, alpha + float(s[-1]), math.sqrt(dot(fma, dt, sizes, w, w, nsm)), passes
    beta = math.sqrt(dot(fma, dt, sizes, w, w, nsm))
    if alg == MGSIR:
        nold = math.sqrt(beta * beta + alpha * alpha + beta_old * beta_old)
        while eps < beta < eta * nold:
            nold = beta
            s, w = mgs_sweep(fma, sizes, Q, w, nsm)
            passes += 1
            alpha += float(s[-1])
            beta = math.sqrt(dot(fma, dt, sizes, w, w, nsm))
    return w, v, alpha, beta, passes


def sharded_apply(fma, dt, sizes, xg, csr, spmv_kernel, spmv_grids, dotv=None, **kw):
    """the halo SpMV on every rank: (global y, the ranks' dot partials)"""
    off = offsets(sizes)
    ys, ds = [], []
    for p, n in enumerate(sizes):
        y, _, d = spmv(fma, dt, spmv_kernel, spmv_grids[p], xg, off[p], n, csr=local_csr(*csr, off[p], n),
                       dotv=dotv, **kw)
        ys.append(y)
        ds.append(d)
    return np.concatenate(ys), ds


def shift_kw(a0, a1):
    return dict(a0=a0, a1=a1, shifted=(a0 != 0.0) or (a1 != 1.0))


def cg_step(fma, dt, sizes, x, r, p, csr, spmv_kernel, spmv_grids, nsm, a0, a1, beta, rho):
    """b2k_cg_step on the shards: p' = r (beta = 0) or rn(r + rn(T(beta) p)); q' = (a0 + a1 A) p' with <p', q'>
    fused (folded); alpha = T(rho / <p', q'>); x' = fma(alpha, p', x); r' = fma(-alpha, q', r); ||r'||^2 the fold of
    k_cg_xr's sums.  (x', r', p', q', <p', q'>, ||r'||, the ranks' <p', q'> partials, the ranks' ||r'||^2 partials)"""
    pn = np.asarray(r, dtype=dt).copy() if beta == 0.0 else (r + dt(beta) * p).astype(dt)
    q, dpq = sharded_apply(fma, dt, sizes, pn, csr, spmv_kernel, spmv_grids, dotv=pn, **shift_kw(a0, a1))
    pq = float(fold(dpq))
    al = dt(rho / pq)
    xn, rn = fma(al, pn, x, dt), fma(-al, q, r, dt)
    drr = [LS.blas1_sum(fma, dt, a, a, LS.grid_for(len(a), 8, nsm)) for a in rows(sizes, rn)]
    return xn, rn, pn, q, pq, math.sqrt(float(fold(drr))), dpq, drr


def bicgstab_half(fma, dt, sizes, rs, r, p, v, csr, spmv_kernel, spmv_grids, nsm, a0, a1, beta, omega, rho, first):
    """b2k_bicgstab_half on the shards: p' = r (first) or rn(r + rn(T(beta) fma(-T(omega), v, p))); v' = (a0 + a1 A)
    p' with sigma = <rs, v'> fused (folded); s' = fma(-T(rho / sigma), v', r); ||s'||^2 the fold of k_bicg_s's sums.
    (p', v', s', sigma, ||s'||, the sigma partials, the ||s'||^2 partials)"""
    if first:
        pn = np.asarray(r, dtype=dt).copy()
    else:
        pn = (r + dt(beta) * fma(-dt(omega), v, p, dt)).astype(dt)
    vn, ds = sharded_apply(fma, dt, sizes, pn, csr, spmv_kernel, spmv_grids, dotv=rs, **shift_kw(a0, a1))
    sigma = float(fold(ds))
    sn = fma(-dt(rho / sigma), vn, r, dt)
    dss = [LS.blas1_sum(fma, dt, a, a, LS.grid_for(len(a), 8, nsm)) for a in rows(sizes, sn)]
    return pn, vn, sn, sigma, math.sqrt(float(fold(dss))), ds, dss


def bicgstab_full(fma, dt, sizes, x, rs, p, s, csr, spmv_kernel, spmv_grids, nsm, a0, a1, alpha):
    """b2k_bicgstab_full on the shards: t' = (a0 + a1 A) s with <t', s> fused, <t', t'> by k_dot (both folded, one
    all-reduce of two doubles); omega = <t', s> / <t', t'>; x' = fma(T(omega), s, fma(T(alpha), p, x));
    r' = fma(-T(omega), t', s); ||r'||^2 and <rs, r'> the folds of k_bicg_xr's sums.
    (x', r', t', omega, ||r'||, next rho, the partials of <t', s>, <t', t'>, ||r'||^2 and <rs, r'>)"""
    tn, dts = sharded_apply(fma, dt, sizes, s, csr, spmv_kernel, spmv_grids, dotv=s, **shift_kw(a0, a1))
    dtt = [LS.blas1_sum(fma, dt, a, a, LS.grid_for(len(a), 8, nsm)) for a in rows(sizes, tn)]
    omega = float(fold(dts)) / float(fold(dtt))
    w = dt(omega)
    xn = fma(w, s, fma(dt(alpha), p, x, dt), dt)
    rn = fma(-w, tn, s, dt)
    drr = [LS.blas1_sum(fma, dt, a, a, LS.grid_for(len(a), 8, nsm)) for a in rows(sizes, rn)]
    drho = [LS.blas1_sum(fma, dt, a, b, LS.grid_for(len(a), 8, nsm)) for a, b in zip(rows(sizes, rs), rows(sizes, rn))]
    return xn, rn, tn, omega, math.sqrt(float(fold(drr))), float(fold(drho)), (dts, dtt, drr, drho)


def dense_adjoint(fma, sizes, A, x, nsm):
    """b2k_op_apply_adjoint of a row-sharded dense A (m x n): y = T(fold of the ranks' per-pass project colsums of
    their row blocks against x_p), the same on every rank"""
    dt = A.dtype.type
    return project(fma, sizes, A, x, nsm).astype(dt)
