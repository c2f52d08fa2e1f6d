"""Host restatement of the single-operator SpMV kernels of spmv.cu (k_spmv_stream, k_spmv_pipe, k_spmv_compact,
k_stencil_apply) with every SpmvFuse feature: y, the stored normalised operand and the fused dot, bit for bit.

Every vector operation is rounded in the vector type T (numpy arithmetic in float32 / float64 is correctly rounded per
operation; fused multiply-adds go through the correctly rounded `fma(a, b, c, T)` of the test_gpu_blas1 fixture), in
the order the kernels use:
  tiles      finish_csr: maxrow <= 768: rowblk[b] = lower_bound(rowptr, b T) with T = 1537 - maxrow; otherwise greedy
             runs of at most 1536 nonzeros and 2048 rows, a longer row alone in its tile;
  products   rn(v rn(x_c T(sc))); a row of a tile of <= 1536 nonzeros summed from (T)0 in stored CSR order;
  long rows  consumer thread i sums the rounded products i, i + 256, ... in double, then a warp butterfly (xor 16 .. 1),
             then the 8 warp sums in order from 0.0 (pipe, compact) or block_sum (stream), rounded to T once;
  shift      fma(T(a0), rn(x_r T(sc)), rn(T(a1) s));   vout_r = rn(x_r T(sc));
  dot        per thread dacc = fma(dv, sd, dacc) in T, sd = s or fma(-T(dsc), dsub_r, s), dv = dotv_r or the normalised
             x_r.  Pipe / compact: CTA b takes tiles b, b + G, ...; consumer t rows r0 + t, r0 + t + 256, ...; in a long
             tile thread 0 alone.  Stream: one tile per CTA.  Stencil: rows t, t + 256 G, ... of global thread t.
             Each CTA reduces its threads (pipe / compact: butterflies, then the warps in order; stream / stencil:
             block_sum); the last CTA has thread t add partials t, t + 256, ... from 0.0 and reduces those the same way.
The grid G is the one the device reports (b2k_debug_spmv_launch).
k_spmm_pipe (apply to a block, test_gpu_spmm.py) forms every row of every vector as k_spmv_pipe does without xscale:
csr_rows(..., xscale=None, kernel="pipe").  Its long row is the same strided double sums, warp_sum butterflies and
red[0 .. 7] added in order from 0.0 by thread 0, so it needs no variant of its own.
"""
import numpy as np

SP_NNZ, SP_ROWS, BT, WARPS = 1536, 2048, 256, 8
f64 = np.float64
KERNELS = ("stream", "pipe", "compact", "stencil")


def tiles(rowptr):
    """rowblk of finish_csr for a row pointer array (int64 array of nblk + 1 boundaries)"""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    n, nnz = len(rowptr) - 1, int(rowptr[-1])
    maxrow = int(np.diff(rowptr).max(initial=0))
    if maxrow <= SP_NNZ // 2:
        T = SP_NNZ - maxrow + 1
        nblk = max(1, -(-nnz // T))
        return np.append(np.searchsorted(rowptr[:n], np.arange(nblk) * T, side="left"), n).astype(np.int64)
    blk, r = [0], 0
    while r < n:
        start, p0 = r, rowptr[r]
        if rowptr[r + 1] - p0 > SP_NNZ:
            r += 1
        else:
            while r < n and rowptr[r + 1] - p0 <= SP_NNZ and r - start < SP_ROWS:
                r += 1
        blk.append(r)
    return np.array(blk, dtype=np.int64)


def butterfly(v):
    """warp_sum over the last axis (32 lanes): lane i adds lane i ^ o for o = 16, 8, 4, 2, 1; every lane ends equal"""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    return v[..., 0]


def cta_reduce(v, kernel):
    """the sum of a CTA's 256 per-thread doubles (last axis) as `kernel` forms it"""
    w = butterfly(v.reshape(v.shape[:-1] + (WARPS, 32)))
    if kernel in ("pipe", "compact"):
        tot = np.zeros(v.shape[:-1])
        for i in range(WARPS):
            tot = tot + w[..., i]
        return tot
    pad = np.zeros(v.shape[:-1] + (32,))          # block_sum: warp 0 butterflies the warp sums, padded with zeros
    pad[..., :WARPS] = w
    return butterfly(pad)


def strided_sums(terms):
    """thread i of a 256-thread CTA adds terms i, i + 256, ... in double from 0.0 (the padding adds +0.0 to a sum that
    started at +0.0, which changes nothing)"""
    trips = max(1, -(-len(terms) // BT))
    t = np.zeros(trips * BT)
    t[:len(terms)] = terms
    acc = np.zeros(BT)
    for k in range(trips):
        acc = acc + t[k * BT:(k + 1) * BT]
    return acc


def last_cta(part, kernel):
    """the last CTA's sum of the CTA partials, in CTA order"""
    return float(cta_reduce(strided_sums(np.asarray(part, dtype=f64)), kernel))


def row_sums(rowptr, prod, dt):
    """each row's rounded products summed from (T)0 in stored order (rows of any length); step k touches only the
    rows longer than k, so the work is O(nnz) whatever the longest row"""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    lens = np.diff(rowptr)
    s = np.zeros(len(lens), dtype=dt)
    rows, k = np.flatnonzero(lens > 0), 0
    while rows.size:
        s[rows] = s[rows] + prod[rowptr[rows] + k]
        k += 1
        rows = rows[lens[rows] > k]
    return s


def csr_rows(rowptr, colidx, vals, x, dt, xscale, kernel):
    """(A x)_r, the operand normalised by T(xscale) when given"""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    with np.errstate(all="ignore"):
        xv = np.asarray(x, dtype=dt)[np.asarray(colidx, dtype=np.int64)]
        if xscale is not None:
            xv = xv * dt(xscale)
        prod = np.asarray(vals, dtype=dt) * xv
        s = row_sums(rowptr, prod, dt)
        for r in np.flatnonzero(np.diff(rowptr) > SP_NNZ):
            acc = strided_sums(prod[rowptr[r]:rowptr[r + 1]].astype(f64))
            s[r] = dt(cta_reduce(acc, kernel))
    return s


def stencil_rows(nx, ny, nz, coeffs, x, dt, xscale):
    """k_stencil_apply's row sums: the products of the 5- / 7-point stencil in ascending column order"""
    n, plane = nx * ny * nz, nx * ny
    c0, cw, ce, cs, cn, cd, cu = (dt(c) for c in coeffs)
    with np.errstate(all="ignore"):
        X = np.asarray(x, dtype=dt)
        if xscale is not None:
            X = X * dt(xscale)
        g = np.arange(n)
        ix, iy, iz = g % nx, (g // nx) % ny, g // plane
        terms = [((nz > 1) & (iz > 0), cd, -plane), (iy > 0, cs, -nx), (ix > 0, cw, -1), (g >= 0, c0, 0),
                 (ix < nx - 1, ce, 1), (iy < ny - 1, cn, nx), ((nz > 1) & (iz < nz - 1), cu, plane)]
        s = np.zeros(n, dtype=dt)
        for m, c, off in terms:
            s[m] = s[m] + c * X[g[m] + off]
    return s


def epilogue(fma, dt, s, x, a0, a1, shifted, xscale, dotv, dot_self, dsub, dsc):
    """(y, vout, dv, sd) of every row from its sum s"""
    with np.errstate(all="ignore"):
        xn = None                               # the normalised operand, row r <-> x_r (square operators)
        if len(x) == len(s):
            xn = np.asarray(x, dtype=dt)
            if xscale is not None:
                xn = xn * dt(xscale)
        y = fma(dt(a0), xn, dt(a1) * s, dt) if shifted else s
        dv = xn if dot_self else (np.asarray(dotv, dtype=dt) if dotv is not None else None)
        sd = fma(-dt(dsc), dsub, y, dt) if dsub is not None else y
    return y, xn, dv, sd


def csr_threads(rowblk, grid):
    """(global consumer thread, position in that thread's row sequence) of every row; k_spmv_stream is the case
    grid = nblk"""
    rowblk = np.asarray(rowblk, dtype=np.int64)
    n = int(rowblk[-1])
    tile = np.repeat(np.arange(len(rowblk) - 1), np.diff(rowblk))
    local = np.arange(n) - rowblk[tile]
    gid = (tile % grid) * BT + local % BT
    order = np.lexsort((local // BT, tile // grid, gid))
    sg = gid[order]
    starts = np.r_[0, np.flatnonzero(np.diff(sg)) + 1]
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n) - np.repeat(starts, np.diff(np.r_[starts, n]))
    return gid, rank


def stencil_threads(n, grid):
    g = np.arange(n)
    return g % (grid * BT), g // (grid * BT)


def dot(fma, dt, dv, sd, gid, rank, grid, kernel, plain=None):
    """the fused dot: the per-thread fma chains in T, the CTA sums, the last CTA's sum.  plain: rows whose term is
    rn(dv sd) rather than an fma into the chain (k_spmv_stream's long row, the first and only term of its thread)"""
    dacc = np.zeros(grid * BT, dtype=dt)
    with np.errstate(all="ignore"):
        for k in range(int(rank.max(initial=-1)) + 1):
            m = rank == k
            dacc[gid[m]] = fma(dv[m], sd[m], dacc[gid[m]], dt)
        if plain is not None and plain.any():
            dacc[gid[plain]] = dv[plain] * sd[plain]
        part = cta_reduce(dacc.astype(f64).reshape(grid, BT), kernel)
        return last_cta(part, kernel)


def apply(fma, dt, kernel, grid, x, *, csr=None, stencil=None, rowblk=None, a0=0.0, a1=1.0, shifted=False,
          xscale=None, dotv=None, dot_self=False, dsub=None, dsc=0.0, gather=None):
    """(y, vout, dot) of one launch; csr = (rowptr, colidx, vals), stencil = (nx, ny, nz, coeffs); vout is the
    normalised operand (what a launch with vout stores), dot is None without a dot.
    gather = (xg, r0): a row shard.  The rows gather from the global operand xg (CSR columns are global, the stencil is
    the global grid's rows r0, r0 + 1, ...), and x, dotv and dsub are the shard's row-aligned slices the epilogue uses."""
    assert kernel in KERNELS
    xg, r0 = (x, 0) if gather is None else gather
    if kernel == "stencil":
        nrows = len(x) if gather is not None else int(np.prod(stencil[:3]))
        s = stencil_rows(*stencil, xg, dt, xscale)[r0:r0 + nrows]
        gid, rank = stencil_threads(len(s), grid)
        plain = None
    else:
        rowptr, colidx, vals = csr
        s = csr_rows(rowptr, colidx, vals, xg, dt, xscale, kernel)
        assert kernel != "stream" or grid == len(rowblk) - 1
        gid, rank = csr_threads(rowblk, grid)
        plain = (np.diff(np.asarray(rowptr, dtype=np.int64)) > SP_NNZ) if kernel == "stream" else None
    y, vout, dv, sd = epilogue(fma, dt, s, x, a0, a1, shifted, xscale, dotv, dot_self, dsub, dsc)
    d = dot(fma, dt, dv, sd, gid, rank, grid, kernel, plain) if dv is not None else None
    return y, vout, d
