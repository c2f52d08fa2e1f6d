"""Host restatement of the summation order of the tall-skinny engine (csrc/tsk.cuh, driven from csrc/basis.cu): the
projection, coefficient and norm reductions and the update fold, bit for bit in Float64 and Float32.

`fma` is the module fixture of test_gpu_blas1.py (libm fma / fmaf, correctly rounded, broadcasting, arguments cast to
T first).  `nsm` is the device's SM count: the grid of every sweep is G = min(#SMs, ceil(n / 256)) CTAs.

Geometry.  A row tile is R = 256 rows; tile t belongs to CTA t mod G, which visits its tiles in increasing order.  A
ring chunk holds C = 8 (f64) / 16 (f32) columns, the consumer lanes read VEC = 2 / 4 elements per 128-bit load and
NLD = 256 / (32 VEC) loads per column.  One pass takes at most kcap = 16 C columns (128 / 256); the cooperative fused
sweep holds at most 12 C (96 / 192).

PROJECT (consumer_phase, VecOps::fma_acc): column j, CTA b, lane l keep an accumulator in T, from +0:
    for b's tiles t, for i < NLD, for e < VEC:  row = 256 t + VEC l + 32 VEC i + e,  row < n:  acc = fma(Q[row, j], x[row], acc)
then (double) acc is summed over the warp by warp_sum (butterfly o = 16 ... 1, each lane adds its xor partner); lane 0
gives part[b, j].
Coefficient (coef_colsum, partial_lane_sum; every UPDATE phase and finalize_block): with L = coef_lanes(k) the largest
power of two <= 16 with L k <= 256 (k the pass width), lane l adds part[g, j] for g = l, l + L, ... to 0.0 in order,
then an xor tree o = L/2 ... 1; lane 0's value.  CGS2 fused reports colsum(A) + colsum(B); the unfused passes and
b2k_basis_project add on the host.
UPDATE: cs_j = T(alphac) * T(h_j) rounded in T (h_j = 0.0 + c_j when the coefficients come from one set of doubles).
acc starts at 0, x or rn(T(beta) x) (beta_mode 0 / 1 / 2), then acc = fma(Q[:, j], cs_j, acc) over the pass's columns
in list order.  Passes past kcap continue from the stored vector with beta_mode 1.
Norm: thread <-> row, nrm = fma(acc, acc, nrm) in T over the CTA's tiles, warp_sum per warp, the 8 warps added to 0.0
in order: part_n[b].  The finaliser: 16 lanes of partial_lane_sum over the G partials, then an xor tree o = 8 ... 1.
Lanczos prologue: x' = fma(T(-alpha0), v, fma(T(-beta_old), v_prev, w)); the update runs over q_0 ... q_{k-2} and then
v_prev, v (the unrotated column order); partials keep the original column index.
"""
import numpy as np

R = 256
NS = 12            # ring slots
f64, f32 = np.float64, np.float32


def cfg(dt):
    """(C, VEC, NLD, kcap, fused limit) of the vector type"""
    c, vec = (8, 2) if np.dtype(dt) == f64 else (16, 4)
    return c, vec, R // (32 * vec), 16 * c, 12 * c


def grid(n, nsm):
    return int(max(1, min(nsm, -(-n // R))))


def coef_lanes(k):
    lanes = 16
    while lanes > 1 and lanes * k > 256:
        lanes //= 2
    return lanes


def warp_sum(v, axis):
    """butterfly over a 32-lane axis: v += shfl_xor(v, o), o = 16 ... 1"""
    idx = np.arange(v.shape[axis])
    for o in (16, 8, 4, 2, 1):
        v = v + np.take(v, idx ^ o, axis=axis)
    return v


def project_partials(Q, x, nsm, fma):
    """part[b, j] of one PROJECT phase over the columns of Q (n x k, T) against x (n, T)"""
    dt = Q.dtype.type
    n, k = Q.shape
    _, vec, nld, _, _ = cfg(dt)
    G = grid(n, nsm)
    ntiles = -(-n // R)
    lanes = np.arange(32)
    acc = np.zeros((G, 32, k), dtype=dt)
    for tt in range(-(-ntiles // G)):
        tile = np.arange(G) + tt * G
        for i in range(nld):
            for e in range(vec):
                rows = R * tile[:, None] + vec * lanes[None, :] + 32 * vec * i + e
                valid = rows < n
                rc = np.where(valid, rows, 0)
                acc = np.where(valid[..., None], fma(Q[rc], x[rc][..., None], acc, dt), acc)
    return warp_sum(acc.astype(f64), 1)[:, 0, :]


def colsum(P):
    """coef_colsum over the G x k partials of one pass"""
    G, k = P.shape
    lanes = coef_lanes(k)
    a = np.zeros((lanes, k))
    for l in range(lanes):
        for g in range(l, G, lanes):
            a[l] = a[l] + P[g]
    idx = np.arange(lanes)
    o = lanes // 2
    while o > 0:
        a = a + a[idx ^ o]
        o //= 2
    return a[0]


def project(Q, x, nsm, fma):
    """d_res of project_t: per pass of kcap columns, the finaliser's colsum of that pass's partials"""
    kcap = cfg(Q.dtype.type)[3]
    k = Q.shape[1]
    return np.concatenate([colsum(project_partials(Q[:, o:o + kcap], x, nsm, fma)) for o in range(0, k, kcap)])


def coefs(h, alphac, dt, one_set=True):
    """cs_j = T(alphac) * T(h_j); from one set of doubles (unfused passes, unproject) h_j is 0.0 + c_j"""
    h = np.asarray(h, dtype=f64)
    if one_set:
        h = 0.0 + h
    return (dt(alphac) * h.astype(dt)).astype(dt)


def update(Q, x, cs, fma, beta_mode=1, beta=1.0):
    """the UPDATE fold over the columns of Q in order (all passes: the later ones start from the stored vector)"""
    dt = Q.dtype.type
    x = np.asarray(x, dtype=dt)
    if beta_mode == 0:
        acc = np.zeros_like(x)
    elif beta_mode == 1:
        acc = x.copy()
    else:
        acc = (dt(beta) * x).astype(dt)
    for j in range(Q.shape[1]):
        acc = fma(Q[:, j], cs[j], acc, dt)
    return acc


def norm_partials(y, nsm, fma):
    """part_n[b]: thread <-> row fma chains over the CTA's tiles, warp_sum, the 8 warps added to 0.0 in order"""
    dt = y.dtype.type
    n = len(y)
    G = grid(n, nsm)
    ntiles = -(-n // R)
    nrm = np.zeros((G, R), dtype=dt)
    for tt in range(-(-ntiles // G)):
        rows = R * (np.arange(G) + tt * G)[:, None] + np.arange(R)[None, :]
        valid = rows < n
        yr = y[np.where(valid, rows, 0)]
        nrm = np.where(valid, fma(yr, yr, nrm, dt), nrm)
    red = warp_sum(nrm.astype(f64).reshape(G, 8, 32), 2)[:, :, 0]
    s = np.zeros(G)
    for w in range(8):
        s = s + red[:, w]
    return s


def normsum(part_n):
    """the finaliser's ||x||^2: 16 lanes of partial_lane_sum, xor tree o = 8 ... 1"""
    a = np.zeros(16)
    for l in range(16):
        for g in range(l, len(part_n), 16):
            a[l] = a[l] + part_n[g]
    idx = np.arange(16)
    for o in (8, 4, 2, 1):
        a = a + a[idx ^ o]
    return a[0]


def cgs(Q, v, passes, nsm, fma):
    """`passes` classical passes (fused or unfused: the same bits): (h, v_out, ||v_out||^2); h sums the passes in
    double.  The fused sweep sums the partials itself, the unfused update takes the finaliser's doubles: equal."""
    dt = Q.dtype.type
    h = np.zeros(Q.shape[1])
    for _ in range(passes):
        hp = project(Q, v, nsm, fma)
        v = update(Q, v, coefs(hp, -1.0, dt), fma)
        h = h + hp
    return h, v, normsum(norm_partials(v, nsm, fma))


def prologue(w, vprev, v, beta_old, alpha0, fma):
    """x' = fma(T(-alpha0), v, fma(T(-beta_old), v_prev, w)): lanczos.jl:313-319 as the sweeps and axpy2 round it"""
    dt = w.dtype.type
    return fma(-alpha0, v, fma(-beta_old, vprev, w, dt), dt)


def lanczos_step(V, v, w, beta_old, alpha0, passes, nsm, fma):
    """the engine part of a CGS2 Lanczos step (prologue, then `passes` classical passes over [V, v] in the original
    column order): (w_out, alpha, ||w_out||^2, h of the last pass); alpha = alpha0 + h[k] per pass, added on the host"""
    Q = np.column_stack([V, v])
    x = prologue(w, V[:, -1], v, beta_old, alpha0, fma)
    alpha = alpha0
    for _ in range(passes):
        h, x, n2 = cgs(Q, x, 1, nsm, fma)
        alpha = alpha + h[-1]
    return x, alpha, n2, h


def slot_of(local_tile, chunk, nch):
    """ring slot of a chunk in a single-phase launch: slots advance by one per chunk, NS slots in a ring"""
    return (local_tile * nch + chunk) % NS
