"""GPU tests of the block path: the multi-right-hand-side kernels of block.cu (block_inner, block_axpy, the block
classical Gram-Schmidt orthogonalisation in its fused and unfused forms, CholeskyQR2 with every k_block_rmul width)
and the reference modified Gram-Schmidt block_qr / block_reorthogonalize of basis.cu, in Float64 and Float32, each
against a float64 restatement of the same operation on the values as stored on the device; then Float32 BlockLanczos
end to end.

Every branch test asserts which branch ran, from the per-class launch counts of b2k_prof_read: 5 = block project
(k_block_phase PROJECT), 6 = block update, Gram matrix or triangular transform (k_block_phase UPDATE and
UPDATE + PROJECT, k_block_rmul).  The register block of the block dimension follows p (PP = 4 for p <= 4, else 8), so
the p grids below run both.

Tolerances.  u is the unit roundoff of the vector type (2^-53 / 2^-24).  Unless a test states otherwise, a sum of m
rounded terms may be off by LAM * sqrt(m) * u * sum(|terms|): the probabilistic bound of Higham & Mary (SIAM J. Sci.
Comput. 41(5), 2019), which a sum violates with probability below 2 m exp(-LAM^2 / 2) (< 1e-9 here).  Bounds are
doubled where the float64 restatement rounds too.

Exact inputs.  A bound scaled by sum(|terms|) cannot see one missing or duplicated row of a long vector, so every
projection and update case also runs on small integers whose partial sums all stay below 2^24.  Every operation is
then exact in both types, and the device must return the float64 result bit for bit.  Columns with a single nonzero
at rows 0, 255, 256, 257, n - 1 and inside a ragged last row tile pin the row <-> thread mapping.
"""
import contextlib
import ctypes as C
import itertools
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.vectors import handles
from oracle import krylov_oracle as ko

LAM = 8.0
BPROJ, BUPD = 5, 6
QMAX = 48                # basis columns per block pass (block.cu BK_QMAX)
PMAX = 8                 # block columns per launch (BK_PMAX)
HCAP = 3968              # coefficients per block call: k * p (B2K_BLK_HCAP)
RES = 8192               # results one block_inner call returns: p * q (B2K_RES_DOUBLES)
EXACT = 2.0 ** 24        # integers up to here are exact in Float32
f64, f32 = np.float64, np.float32

SIZES = [(f64, n) for n in (1, 255, 256, 257, 70_001)] + \
        [(f32, n) for n in (1, 255, 256, 257, 70_001, 4097, 4098, 4099)]      # n % 4 = 1, 2, 3 for the float4 paths
SIZE_IDS = [f"{np.dtype(d).name}-n{n}" for d, n in SIZES]
LAYOUT = pytest.mark.parametrize("contiguous", [True, False], ids=["contiguous", "strided"])


def unit(dtype):
    return 2.0 ** -53 if dtype == f64 else 2.0 ** -24


def cdiv(a, b):
    return -(-a // b)


def dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@contextlib.contextmanager
def profiled(ctx):
    """launch counts of the block classes for what runs inside the block"""
    counts = {}
    ctx.check(ctx.lib.b2k_prof_reset(ctx.h))
    ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 1))
    try:
        yield counts
    finally:
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 0))
        for cls in (BPROJ, BUPD):
            c = C.c_int64()
            ctx.check(ctx.lib.b2k_prof_read(ctx.h, cls, C.byref(c), None, None))
            counts[cls] = c.value


def alloc(ctx, m, contiguous):
    """m device vectors: one slab range, or every other column of 2 m single allocations (all kept alive)"""
    if contiguous:
        return ctx.empty_range(m)
    vecs = [ctx.empty() for _ in range(2 * m)]
    ctx._keep = getattr(ctx, "_keep", []) + vecs
    return vecs[::2]


def put(vecs, A, dtype):
    """upload the columns of A; returns them as stored (Float32 rounds), in float64"""
    At = np.ascontiguousarray(np.asarray(A).T, dtype=dtype)
    for j, v in enumerate(vecs):
        v.upload(At[j])
    return At.T.astype(f64)


def get(vecs):
    return np.column_stack([v.to_host() for v in vecs]).astype(f64)


def spike_rows(n):
    """rows 0, 255, 256, 257, n - 1, and the first and a middle row of the last row tile (ragged unless 256 | n)"""
    last = (n - 1) // 256 * 256
    rows = {0, 255, 256, 257, n - 1, last, last + (n - 1 - last) // 2}
    return sorted(r for r in rows if 0 <= r < n)


def int_block(rng, n, m, spikes=()):
    """n x m integers in [-3, 3]; column c < len(spikes) has the single nonzero +-(c % 3 + 1) at row spikes[c]"""
    A = rng.integers(-3, 4, size=(n, m)).astype(f64)
    for c, r in enumerate(list(spikes)[:m]):
        A[:, c] = 0.0
        A[r, c] = (-1) ** c * (c % 3 + 1)
    return A


def spike_basis(rng, n, k):
    """k columns +-e_r, the rows cycling through spike_rows(n) then random rows (repeated when k > n): an integer
    basis that touches the special rows and keeps every Gram-Schmidt quantity a small integer"""
    rows = spike_rows(n) + list(rng.permutation(n))
    rows = [rows[j % len(rows)] for j in range(k)]
    V = np.zeros((n, k))
    V[rows, np.arange(k)] = rng.choice([-1.0, 1.0], size=k)
    return V


_Q = {}


def qbasis(n, k):
    """n x k orthonormal columns (float64), a prefix of one cached QR factor"""
    if n not in _Q or _Q[n].shape[1] < k:
        _Q[n] = np.linalg.qr(np.random.default_rng(n).standard_normal((n, max(k, 97))))[0]
    return _Q[n][:, :k]


# ------------------------------------------------------------------------------------------ wrappers ---------------

def block_inner(ctx, X, Y):
    M = np.zeros((len(X), len(Y)), order="F")
    ctx.check(ctx.lib.b2k_block_inner(ctx.h, handles(X), len(X), handles(Y), len(Y), dptr(M)))
    return M


def block_axpy(ctx, Y, X, M, ldm):
    """Y[j] -= sum_i X[i] M[i, j], M passed with leading dimension ldm (rows past p are NaN: never read)"""
    p, q = len(X), len(Y)
    Mh = np.full((ldm, q), np.nan, order="F")
    Mh[:p] = M
    ctx.check(ctx.lib.b2k_block_axpy(ctx.h, handles(Y), q, handles(X), p, dptr(Mh), ldm))


def block_orth(ctx, R, V, passes, want_gram=True):
    p, k = len(R), len(V)
    H = np.zeros((max(k, 1), p), order="F")
    G = np.zeros((p, p), order="F")
    ctx.check(ctx.lib.b2k_block_orthogonalize(ctx.h, handles(R), p, handles(V) if k else None, k, passes,
                                              dptr(H) if k else None, dptr(G) if want_gram else None))
    return H[:k], G


def block_cholqr(ctx, X, tol, G0=None):
    p = len(X)
    R = np.zeros((p, p), order="F")
    ok = C.c_int32()
    g0 = np.asfortranarray(G0, dtype=f64) if G0 is not None else None
    ctx.check(ctx.lib.b2k_block_cholqr(ctx.h, handles(X), p, float(tol), dptr(g0) if g0 is not None else None,
                                       dptr(R), C.byref(ok)))
    return R, ok.value


def block_qr(ctx, X, tol):
    p = len(X)
    R = np.zeros((p, p), order="F")
    good = (C.c_int32 * p)()
    drift = C.c_int32()
    ctx.check(ctx.lib.b2k_block_qr(ctx.h, handles(X), p, float(tol), dptr(R), good, C.byref(drift)))
    return R, [int(g) for g in good], drift.value


def mgs_once(ctx, w, Q):
    """one modified Gram-Schmidt sweep of w against Q, as b2k_block_qr runs it; returns (h, ||w||)"""
    h = np.zeros(len(Q))
    beta, passes = C.c_double(), C.c_int32()
    ctx.check(ctx.lib.b2k_basis_orthogonalize(ctx.h, w.handle, handles(Q), len(Q), dptr(h), L.MGS, 0.0,
                                              C.byref(beta), C.byref(passes)))
    return h, beta.value


# ------------------------------------------------------------------------------------------ 1. block_inner ---------

PS = (1, 47, 48, 49, 96, 97, 496)
QS = (1, 3, 4, 5, 8, 9, 17)


@LAYOUT
@pytest.mark.parametrize("dtype,n", SIZES, ids=SIZE_IDS)
def test_block_inner(dtype, n, contiguous):
    """M = X'Y for p in PS (both sides of the 48-column pass) and q in QS (both sides of the 8-column launch), one
    launch per 8 columns of Y and 48 of X; the Gram matrix X'X; the refusals past p = 496 and p * q = 8192."""
    u = unit(dtype)
    rng = np.random.default_rng(n + 7 * contiguous)
    pm, qm = max(PS) + 1, max(QS)
    ctx = kk.B200Context(n, 2 * (pm + qm) + 8, dtype=dtype)
    X, Y = alloc(ctx, pm, contiguous), alloc(ctx, qm, contiguous)
    spikes = spike_rows(n)
    for kind in ("normal", "integer"):
        if kind == "normal":
            Xs, Ys = put(X, rng.standard_normal((n, pm)), dtype), put(Y, rng.standard_normal((n, qm)), dtype)
        else:
            Xs, Ys = put(X, int_block(rng, n, pm, spikes), dtype), put(Y, int_block(rng, n, qm, spikes[::-1]), dtype)
        ref, absum = Xs.T @ Ys, np.abs(Xs).T @ np.abs(Ys)
        if kind == "integer":
            assert absum.max() < EXACT
        for p in PS:
            for q in QS:
                if p * q > RES:
                    with pytest.raises(kk.B200Error):
                        block_inner(ctx, X[:p], Y[:q])
                    continue
                with profiled(ctx) as cnt:
                    M = block_inner(ctx, X[:p], Y[:q])
                assert (cnt[BPROJ], cnt[BUPD]) == (cdiv(q, PMAX) * cdiv(p, QMAX), 0), (p, q, cnt)
                if kind == "integer":
                    assert np.array_equal(M, ref[:p, :q]), (p, q, np.argwhere(M != ref[:p, :q])[:8])
                else:
                    # n products summed per entry
                    err = np.abs(M - ref[:p, :q]) - 2 * LAM * math.sqrt(n) * u * absum[:p, :q]
                    assert err.max() <= 0, (p, q, err.max())
        # block_inner(Y, Y): entry (i, j) sums the same products in the same row order as (j, i) (the basis and the
        # block side of a tile are read alike, fma(q, x, acc) == fma(x, q, acc)), so the Gram matrix is symmetric
        G = block_inner(ctx, Y, Y)
        gref, gabs = Ys.T @ Ys, np.abs(Ys).T @ np.abs(Ys)
        if kind == "integer":
            assert np.array_equal(G, gref)
        else:
            assert np.all(np.abs(G - gref) <= 2 * LAM * math.sqrt(n) * u * gabs)
        assert np.array_equal(G, G.T)
    # p * 8 > 3968 coefficients: refused before anything runs; the context stays usable
    with pytest.raises(kk.B200Error):
        block_inner(ctx, X[:497], Y[:1])
    assert np.array_equal(block_inner(ctx, X[:3], Y[:2]), ref[:3, :2])
    ctx.close()


# ------------------------------------------------------------------------------------------ 2. block_axpy ----------

@LAYOUT
@pytest.mark.parametrize("dtype,n", SIZES, ids=SIZE_IDS)
def test_block_axpy(dtype, n, contiguous):
    """Y -= X M for the (p, q) grid of test_block_inner, with ldm = p and ldm > p; an aliased Y is refused."""
    u = unit(dtype)
    rng = np.random.default_rng(2 * n + contiguous)
    pm, qm = max(PS) + 1, max(QS)
    ctx = kk.B200Context(n, 2 * (pm + qm) + 8, dtype=dtype)
    X, Y = alloc(ctx, pm, contiguous), alloc(ctx, qm, contiguous)
    spikes = spike_rows(n)
    for kind in ("normal", "integer"):
        if kind == "normal":
            Xs = put(X, rng.standard_normal((n, pm)), dtype)
            Y0 = rng.standard_normal((n, qm)).astype(dtype)
            Mf = rng.standard_normal((pm, qm))
        else:
            Xs = put(X, int_block(rng, n, pm, spikes), dtype)
            Y0 = int_block(rng, n, qm, spikes[::-1]).astype(dtype)
            Mf = rng.integers(-3, 4, size=(pm, qm)).astype(f64)
        Ys = Y0.astype(f64)
        Mt = Mf.astype(dtype).astype(f64)      # the device rounds the coefficients to the vector type
        # prefix products X[:, :p] M[:p, :] for every p of the grid, accumulated in column blocks
        prod, aprod, lo = {}, {}, 0
        acc, aacc = np.zeros((n, qm)), np.zeros((n, qm))
        for p in PS:
            acc = acc + Xs[:, lo:p] @ Mt[lo:p]
            aacc = aacc + np.abs(Xs[:, lo:p]) @ np.abs(Mt[lo:p])
            prod[p], aprod[p], lo = acc, aacc, p
        for p in PS:
            if kind == "integer":
                assert (np.abs(Ys) + aprod[p]).max() < EXACT
            for q in QS:
                for c, y in enumerate(Y[:q]):
                    y.upload(Y0[:, c])
                with profiled(ctx) as cnt:
                    block_axpy(ctx, Y[:q], X[:p], Mf[:p, :q], p if kind == "integer" else p + 3)
                assert (cnt[BUPD], cnt[BPROJ]) == (cdiv(q, PMAX) * cdiv(p, QMAX), 0), (p, q, cnt)
                out = get(Y[:q])
                ref = Ys[:, :q] - prod[p][:, :q]
                if kind == "integer":
                    assert np.array_equal(out, ref), (p, q, np.argwhere(out != ref)[:8])
                else:
                    # per entry a chain of p fused multiply-adds onto y: p + 1 terms
                    bound = 2 * LAM * math.sqrt(p + 1) * u * (np.abs(Ys[:, :q]) + aprod[p][:, :q])
                    assert np.all(np.abs(out - ref) <= bound), (p, q, np.abs(out - ref).max())
    with pytest.raises(ValueError):
        block_axpy(ctx, [Y[0], X[2]], X[:3], np.ones((3, 2)), 3)
    with pytest.raises(kk.B200Error):
        block_axpy(ctx, Y[:1], X[:497], np.ones((497, 1)), 497)
    ctx.close()


# ------------------------------------------------------------------------------------------ 3. block_orthogonalize -

@contextlib.contextmanager
def block_fuse(on):
    """B2K_BLOCK_FUSE for the contexts created inside.  b2k_block_init copies the variable into a process-wide flag at
    every context creation, but only when it is set: unsetting it would leave the flag as it is, so the exit sets it
    back to 1 and creates a context before restoring the environment."""
    saved = os.environ.get("B2K_BLOCK_FUSE")
    os.environ["B2K_BLOCK_FUSE"] = "1" if on else "0"
    try:
        yield
    finally:
        os.environ["B2K_BLOCK_FUSE"] = "1"
        kk.B200Context(8, 2).close()
        if saved is None:
            del os.environ["B2K_BLOCK_FUSE"]
        else:
            os.environ["B2K_BLOCK_FUSE"] = saved


def bcgs_ref(V, R, passes):
    """R - V (V'R), `passes` times, in float64; returns (R_out, summed coefficients, the largest sum of |terms| any
    partial sum of the coefficients or the update saw)"""
    H = np.zeros((V.shape[1], R.shape[1]))
    W, big = R.copy(), 0.0
    for _ in range(passes):
        h = V.T @ W
        big = max(big, (np.abs(V).T @ np.abs(W)).max(initial=0), (np.abs(W) + np.abs(V) @ np.abs(h)).max(initial=0))
        W = W - V @ h
        H += h
    return W, H, big


def orth_tols(n, k, u, nv, passes):
    """Bounds on the coefficients and the result of `passes` block Gram-Schmidt passes of a column of norm nv against
    k orthonormal columns.  Per pass, for the column w it starts from (|w| <= nv, |h| <= |w|):
      coefficient <v_j, w>, n terms:               |dh_j| <= LAM sqrt(n) u nv             (sum |v_ij w_i| <= |w|)
      update w - sum_j v_j h_j, h rounded to T,    |dw|   <= (LAM sqrt(k+1) + 1) u (1 + sqrt(k)) nv
      k + 1 terms:                                           + sqrt(k) max_j |dh_j|
    A later pass's coefficients see the earlier update's rounding but not its coefficient errors (V'V dh = dh, which
    the pass removes).  Summed over the passes, doubled for the float64 restatement.  Returns (max |dH|, |d R_out|)."""
    eh = LAM * math.sqrt(n) * u * nv
    eu = (LAM * math.sqrt(k + 1) + 1) * u * (1 + math.sqrt(k)) * nv
    return 2 * passes * (eh + eu), 2 * passes * (math.sqrt(k) * eh + eu)


def expected_orth_launches(p, k, passes, fuse=True):
    """(block project, block update) launches: k = 0 is one Gram pass; the fused BCGS2 sweep (passes 2, p <= 4,
    k <= 48) is project | update + project | update; otherwise one launch of each per 48 columns and pass"""
    if k == 0:
        return 0, 1
    if fuse and passes == 2 and p <= 4 and k <= QMAX:
        return 1, 2
    return passes * cdiv(k, QMAX), passes * cdiv(k, QMAX)


KS = (0, 1, 47, 48, 49, 97)


def check_orth(ctx, R, V, Rs, Vs, passes, kind, dtype):
    """run block_orthogonalize on R (stored values Rs) against V (Vs) and check it; returns (R_out, H, G)"""
    n, p, k = Rs.shape[0], Rs.shape[1], Vs.shape[1]
    u = unit(dtype)
    with profiled(ctx) as cnt:
        H, G = block_orth(ctx, R, V, passes)
    case = (kind, p, k, passes)
    assert (cnt[BPROJ], cnt[BUPD]) == expected_orth_launches(p, k, passes), (case, cnt)
    out = get(R)
    if k == 0:
        assert np.array_equal(out, Rs), case           # Gram matrix only: the block is not written
    ref, href, big = bcgs_ref(Vs, Rs, passes)
    gref = out.T @ out                                  # the Gram matrix of what the device stored
    gabs = np.abs(out).T @ np.abs(out)
    if kind == "integer":
        assert big < EXACT
        assert np.array_equal(out, ref), (case, np.argwhere(out != ref)[:8])
        assert np.array_equal(H, href), case
        # a basis column repeated m times scales a row by (1 - m)^passes: its squares can pass 2^24 (n = 1, k = 97)
        if dtype == f64 or gabs.max() < EXACT:
            assert np.array_equal(G, gref), case
            return out, H, G
    # G: n products per entry, from the downloaded block
    assert np.all(np.abs(G - gref) <= 2 * LAM * math.sqrt(n) * u * gabs), case
    if kind == "integer":
        return out, H, G
    for i in range(p):
        nv = float(np.linalg.norm(Rs[:, i]))
        tx, tv = orth_tols(n, k, u, nv, passes)
        assert np.abs(H[:, i] - href[:, i]).max(initial=0) <= tx, (case, i, np.abs(H[:, i] - href[:, i]).max(), tx)
        assert np.linalg.norm(out[:, i] - ref[:, i]) <= tv, (case, i, np.linalg.norm(out[:, i] - ref[:, i]), tv)
    return out, H, G


@LAYOUT
@pytest.mark.parametrize("dtype,n", SIZES, ids=SIZE_IDS)
def test_block_orthogonalize(dtype, n, contiguous):
    """BCGS of p = 1..8 columns against k in KS basis columns (0: Gram matrix only; both sides of the 48-column pass),
    one and two passes: R_out, the summed coefficients H and G = R_out'R_out against the float64 restatement, on an
    orthonormal basis (k <= n) and, exactly, on an integer basis of +-unit columns.  With two passes a block that
    lies in span(V) up to 1e-8 (where the second pass is what orthogonalises it) comes out orthogonal to V at the
    rounding level."""
    u = unit(dtype)
    rng = np.random.default_rng(3 * n + contiguous)
    km = max(KS)
    with block_fuse(True):
        ctx = kk.B200Context(n, 2 * (km + 8) + 16, dtype=dtype)
    V, R, W = alloc(ctx, km, contiguous), alloc(ctx, PMAX, contiguous), alloc(ctx, PMAX, contiguous)
    Vq = put(V, qbasis(n, km) if n >= km else np.zeros((n, km)), dtype)
    E = np.linalg.norm(Vq.T @ Vq - np.eye(km), 2) if n >= km else None    # V'V - I of the stored basis
    for p in range(1, PMAX + 1):
        for k in KS:
            for passes in (1, 2):
                if k <= n:                              # the orthonormal basis needs k <= n
                    Vs = Vq[:, :k]
                    Rs = put(R[:p], rng.standard_normal((n, p)), dtype)
                    check_orth(ctx, R[:p], V[:k], Rs, Vs, passes, "normal", dtype)
                    if passes == 2 and k > 0 and n >= km:
                        # R = V C + 1e-8 noise.  Pass 1 leaves w1 of norm ~1e-8 |R| (Float64) or ~u |R| (Float32:
                        # the noise is below the stored precision), already rounding-level in V'w1 relative to |R|,
                        # not to |w1|.  Pass 2 starts from w1: V'R_out = -E V'w1 - (I + E) dh + V'dw with
                        # |dh| <= LAM sqrt(n) u |w1| and |dw| <= the update bound of orth_tols on |w1|.
                        near = Vs @ rng.standard_normal((k, p)) + 1e-8 * rng.standard_normal((n, p))
                        Rs = put(R[:p], near, dtype)
                        put(W[:p], near, dtype)
                        block_orth(ctx, W[:p], V[:k], 1, want_gram=False)
                        w1 = np.linalg.norm(get(W[:p]), axis=0)          # the device's first pass
                        out, _, _ = check_orth(ctx, R[:p], V[:k], Rs, Vs, 2, "near", dtype)
                        f = E + 1.01 * LAM * math.sqrt(n) * u + 2 * (LAM * math.sqrt(k + 1) + 1) * u * (1 + math.sqrt(k))
                        lhs = np.abs(Vs.T @ out).max(axis=0)
                        rhs = f * w1 + 2 * LAM * math.sqrt(n) * 2.0 ** -53 * np.linalg.norm(out, axis=0)
                        assert np.all(lhs <= rhs), (p, k, lhs, rhs)
                # exact: +-unit basis columns (repeated rows when k > n), integer block
                Vi = spike_basis(rng, n, k)
                Vis = put(V[:k], Vi, dtype)
                Rs = put(R[:p], int_block(rng, n, p, spike_rows(n)[::-1]), dtype)
                check_orth(ctx, R[:p], V[:k], Rs, Vis, passes, "integer", dtype)
                put(V[:k], Vq[:, :k], dtype)            # restore the orthonormal basis
    ctx.close()


FUSE_SIZES = [(f64, 257), (f64, 70_001), (f32, 255), (f32, 70_001)]


@pytest.mark.parametrize("dtype,n", FUSE_SIZES, ids=[f"{np.dtype(d).name}-n{n}" for d, n in FUSE_SIZES])
def test_fused_bcgs2_equals_unfused(dtype, n):
    """The fused BCGS2 sweep (launch_update_project: the updated block is projected from the resident tile) against the
    four separate sweeps of B2K_BLOCK_FUSE=0 on the same inputs.  Both project the updated block tile by tile with the
    same per-CTA accumulation order and round it to the vector type first (the fused sweep projects the values it
    stores), so R_out, H and G are bit-identical."""
    rng = np.random.default_rng(n)
    cases = []
    Q = qbasis(n, QMAX)
    for p in range(1, 5):
        for k in (1, 47, 48):
            cases.append((p, k, rng.standard_normal((n, p))))
            cases.append((p, k, Q[:, :k] @ rng.standard_normal((k, p)) + 1e-8 * rng.standard_normal((n, p))))
            cases.append((p, k, int_block(rng, n, p, spike_rows(n))))
    runs = {}
    for fuse in (True, False):
        with block_fuse(fuse):
            ctx = kk.B200Context(n, 2 * QMAX + 16, dtype=dtype)
            V, R = ctx.empty_range(QMAX), ctx.empty_range(4)
            put(V, Q, dtype)
            res = []
            for p, k, A in cases:
                put(R[:p], A, dtype)
                with profiled(ctx) as cnt:
                    H, G = block_orth(ctx, R[:p], V[:k], 2)
                assert (cnt[BPROJ], cnt[BUPD]) == expected_orth_launches(p, k, 2, fuse), (fuse, p, k, cnt)
                res.append((get(R[:p]), H, G))
            ctx.close()
        runs[fuse] = res
    for (p, k, _), a, b in zip(cases, runs[True], runs[False]):
        for x, y, what in zip(a, b, ("R", "H", "G")):
            assert np.array_equal(x, y), (p, k, what, np.abs(x - y).max())


@pytest.mark.parametrize("dtype", [f64, f32])
def test_block_orthogonalize_limits(dtype):
    """k * p = 3968 (p = 8, k = 496: eleven unfused 48-column passes, twice) works and is exact on integer inputs;
    k * p = 3976 is refused before anything runs; a block column that is also a basis column is refused."""
    n = 257
    assert 496 * PMAX == HCAP
    rng = np.random.default_rng(3968)
    with block_fuse(True):
        ctx = kk.B200Context(n, 520, dtype=dtype)
    V, R = ctx.empty_range(497), ctx.empty_range(8)
    Vs = put(V, spike_basis(rng, n, 497), dtype)
    Rs = put(R, int_block(rng, n, 8, spike_rows(n)), dtype)
    check_orth(ctx, R, V[:496], Rs, Vs[:, :496], 2, "integer", dtype)
    out = get(R)
    with profiled(ctx) as cnt:
        with pytest.raises(kk.B200Error):
            block_orth(ctx, R, V, 2)
    assert (cnt[BPROJ], cnt[BUPD]) == (0, 0) and np.array_equal(get(R), out)
    with pytest.raises(ValueError):
        block_orth(ctx, [R[0], V[5]], V[:8], 2)
    assert np.array_equal(get(R), out)
    ctx.close()


@pytest.mark.parametrize("dtype", [f64, f32])
def test_block_gram_of_a_ragged_tile_after_the_ring_wraps(dtype):
    """The rows of a ragged last tile past n hold what an earlier tile of the same CTA left in the shared-memory ring
    once the ring has wrapped (here: every CTA walks at least 13 row tiles, the ring has 12 slots).  The Gram matrix
    (k = 0) and one pass against a +-unit basis must not see them: exact on integers."""
    n = 256 * 132 * 13 + 129
    rng = np.random.default_rng(13)
    with block_fuse(True):
        ctx = kk.B200Context(n, 24, dtype=dtype)
    V, R = ctx.empty_range(4), ctx.empty_range(PMAX)
    Vs = put(V, spike_basis(rng, n, 4), dtype)
    for p in (3, PMAX):
        for k in (0, 1, 4):
            Rs = put(R[:p], int_block(rng, n, p, spike_rows(n)), dtype)
            check_orth(ctx, R[:p], V[:k], Rs, Vs[:, :k], 1, "integer", dtype)
    ctx.close()


# ------------------------------------------------------------------------------------------ 4. block_cholqr --------

def cholqr_tols(n, p, u, kappa, Xnorm):
    """Bounds for an accepted CholeskyQR2 of an n x p block of condition kappa and Frobenius norm Xnorm.
      Q'Q - I, per entry: round 2 starts from Q1 with |Q1'Q1 - I| < 1/2 (what the acceptance threshold buys); its
        Gram matrix (n products per entry, |q_i||q_j| <= 1.5) and its transform (p + 1 terms per entry, |U2| <= 2)
        leave LAM (sqrt(n) + sqrt(p + 1)) u, times 4 for those norms.
      |QR - X|_F: fl(X U) = X U + E with |E| <= LAM sqrt(p+1) u |X||U|, so Q1 L1' = X + E L1' with
        |E L1'|_F <= LAM sqrt(p+1) u |X|_F kappa(L1) and kappa(L1) = kappa(X); round 2 adds the same with kappa ~ 1;
        doubled for the float64 product QR."""
    return 4 * LAM * (math.sqrt(n) + math.sqrt(p + 1)) * u, 2 * LAM * math.sqrt(p + 1) * u * (kappa + 1) * Xnorm


def check_cholqr(ctx, X, Xs, Q, R, u):
    """orthogonality, QR = X and R against the positive-diagonal QR factor of the stored block; returns a list of
    what failed"""
    n, p = Xs.shape
    kappa = float(np.linalg.cond(Xs))
    torth, tres = cholqr_tols(n, p, u, kappa, float(np.linalg.norm(Xs)))
    bad = []
    eo = np.abs(Q.T @ Q - np.eye(p)).max()
    if not eo <= torth:
        bad.append(f"|Q'Q - I| = {eo:.3g} > {torth:.3g}")
    er = np.linalg.norm(Q @ R - Xs)
    if not er <= tres:
        bad.append(f"|QR - X| = {er:.3g} > {tres:.3g}")
    if not (np.all(np.tril(R, -1) == 0) and np.all(np.diag(R) > 0)):
        bad.append("R is not upper triangular with a positive diagonal")
    # R is the exact factor of X + dX with |dX|_F <= |QR - X|_F + |Q'Q - I|_F |X|_2 (first order), and the
    # factor moves by at most sqrt(2) kappa |dX|_F / |X|_2 relative to |X|_2 (Sun 1991); doubled for second order
    # and the float64 factorisation
    Rr = np.linalg.qr(Xs)[1]
    Rr = Rr * np.sign(np.diag(Rr))[:, None]
    dX = er + np.linalg.norm(Q.T @ Q - np.eye(p)) * np.linalg.norm(Xs, 2)
    eR = np.linalg.norm(R - Rr)
    if not eR <= 2 * math.sqrt(2) * kappa * dX + 1e-14 * kappa * np.linalg.norm(Xs):
        bad.append(f"|R - R_qr| = {eR:.3g}")
    return bad


@LAYOUT
@pytest.mark.parametrize("dtype,n", SIZES, ids=SIZE_IDS)
def test_block_cholqr(dtype, n, contiguous):
    """CholeskyQR2 of well-conditioned blocks of p = 1..8 columns (every k_block_rmul width; n covers every n % VEC
    tail), with the first Gram matrix passed in and computed: one Gram pass and two transforms, or two transforms.
    A block with more columns than rows (n = 1) is refused and left untouched."""
    u = unit(dtype)
    rng = np.random.default_rng(5 * n + contiguous)
    ctx = kk.B200Context(n, 2 * PMAX + 8, dtype=dtype)
    X = alloc(ctx, PMAX, contiguous)
    for p in range(1, PMAX + 1):
        for with_g0 in (False, True):
            Xs = put(X[:p], rng.standard_normal((n, p)) + 0.5, dtype)
            with profiled(ctx) as cnt:
                R, ok = block_cholqr(ctx, X[:p], 1e-12, Xs.T @ Xs if with_g0 else None)
            case = (p, with_g0)
            assert ok == (n >= p), case
            if not ok:
                assert (cnt[BUPD], cnt[BPROJ]) == (0 if with_g0 else 1, 0), (case, cnt)
                assert np.array_equal(get(X[:p]), Xs), case
                continue
            assert (cnt[BUPD], cnt[BPROJ]) == (2 if with_g0 else 3, 0), (case, cnt)
            bad = check_cholqr(ctx, X[:p], Xs, get(X[:p]), R, u)
            assert not bad, (case, bad)
    ctx.close()


KAPPAS = (1e1, 1e3, 1e4, 1e5, 1e6, 1e8)


@pytest.mark.parametrize("dtype", [f64, f32])
def test_block_cholqr_conditioning_sweep(dtype):
    """Blocks X = Q diag(s) W' with s geometric from 1 to 1/kappa, Q spread over all rows or supported on 16 rows (then
    the Gram entries are sums of few products and carry the full relative noise u of the type).  Contract: no error
    for finite input; ok = 1 only with Q orthonormal to the rounding level of the type (X untouched otherwise); Float64
    accepts every kappa up to 1e5 (its smallest pivot, >= s_min^2 = 1e-10, is above the threshold 1e-11 |x_j|^2) and
    refuses 1e8."""
    u = unit(dtype)
    n = 70_001
    rng = np.random.default_rng(10 ** 8)
    ctx = kk.B200Context(n, 2 * PMAX + 8, dtype=dtype)
    X = ctx.empty_range(PMAX)
    bad, accepted = [], {}
    rows = rng.choice(n, size=16, replace=False)
    Q16 = np.zeros((n, PMAX))
    Q16[rows] = np.linalg.qr(rng.standard_normal((16, PMAX)))[0]
    for kappa, p, shape, with_g0 in itertools.product(KAPPAS, (2, 4, 8), ("spread", "rows16"), (False, True)):
        W = np.linalg.qr(rng.standard_normal((p, p)))[0]
        Qb = qbasis(n, p) if shape == "spread" else Q16[:, :p]
        A = Qb @ np.diag(np.geomspace(1.0, 1.0 / kappa, p)) @ W.T
        Xs = put(X[:p], A, dtype)
        case = f"kappa={kappa:g} p={p} {shape} G0={with_g0}"
        try:
            R, ok = block_cholqr(ctx, X[:p], 1e-12, Xs.T @ Xs if with_g0 else None)
        except kk.B200Error as e:
            bad.append(f"{case}: raised {e}")
            put(X[:p], A, dtype)
            continue
        accepted[case] = (kappa, ok)
        if ok:
            bad += [f"{case}: {b}" for b in check_cholqr(ctx, X[:p], Xs, get(X[:p]), R, u)]
        elif not np.array_equal(get(X[:p]), Xs):
            bad.append(f"{case}: refused but X changed")
    assert not bad, "\n".join(bad)
    if dtype == f64:
        for case, (kappa, ok) in accepted.items():
            if kappa <= 1e5:
                assert ok, case
            if kappa >= 1e8:
                assert not ok, case
    ctx.close()


# ------------------------------------------------------------------------------------------ 5. block_qr, reorth ----

QR_TOL = {f64: 1e-8, f32: 1e-3}      # unit-size columns: the f32 drift band (1e-3, 1e-1) is far above its rounding


def qr_block(rng, n, p, tol, layout):
    """p columns of size ~1 with the roles of `layout` (a string, one letter a column): r random, z zero, s below tol,
    d dependent on the earlier columns (dropped), g 3 x column 0 plus 10 tol orthogonal to every earlier column (its
    residual lies inside (tol, 100 tol): the DGKS pass)"""
    A = np.zeros((n, p))
    for j, c in enumerate(layout):
        if c == "r":
            A[:, j] = rng.standard_normal(n) / math.sqrt(n)
        elif c == "s":
            A[:, j] = 0.1 * tol * rng.standard_normal(n) / math.sqrt(n)
        elif c == "d":
            A[:, j] = 2.0 * A[:, 0] if j == 1 else A[:, j - 1] - 2.0 * A[:, j - 2]
        elif c == "g":
            e = rng.standard_normal(n)
            if j:
                Qp = np.linalg.qr(A[:, :j])[0]
                e -= Qp @ (Qp.T @ e)
                e -= Qp @ (Qp.T @ e)
            A[:, j] = 3.0 * A[:, 0] + 10.0 * tol * e / np.linalg.norm(e)
    return A


QR_LAYOUTS = {1: ("r", "z", "s"), 2: ("rr", "rg", "rd", "zr", "sr"), 8: ("rrrdrgrr", "zrrrgrdr"),
              12: ("rrrdrgrrsrgr", "srrrrrrrrrdr")}


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("p", sorted(QR_LAYOUTS))
def test_block_qr_branches(dtype, p):
    """b2k_block_qr against the oracle's block_qr on the stored columns: good, drift, R and the orthonormal columns,
    for blocks whose first column is zero or below tol, with dependent columns and with a column whose residual lies
    strictly inside (tol, 100 tol).  For that column R holds the first and the DGKS sweep's coefficients: R[:j, j]
    equals, bit for bit, the sum of two MGS sweeps of the input column against the returned columns."""
    n = 4099
    u = unit(dtype)
    tol = QR_TOL[dtype]
    rng = np.random.default_rng(p)
    ctx = kk.B200Context(n, 2 * p + 8, dtype=dtype)
    X = ctx.empty_range(p)
    for layout in QR_LAYOUTS[p]:
        Xs = put(X, qr_block(rng, n, p, tol, layout), dtype)
        R, good, drift = block_qr(ctx, X, tol)
        blk = [Xs[:, j].copy() for j in range(p)]
        Rg, gidx, odrift = ko.block_qr(blk, tol)
        oQ = np.column_stack(blk)
        assert good == [int(j in gidx) for j in range(p)], (layout, good, gidx)
        assert drift == int(odrift) == int("g" in layout[1:]), (layout, drift, odrift)
        Q = get(X)
        # Each column goes through at most p - 1 projections (n products each) and updates: 2 p LAM (sqrt(n) +
        # sqrt(p)) u |x|, doubled for the oracle.  Normalising a column by beta amplifies its error by |x| / beta, and
        # later columns inherit it through their coefficients: amp multiplies those factors over the kept columns.
        xmax = np.linalg.norm(Xs, axis=0).max()
        amp = math.prod(max(1.0, xmax / Rg[r, gidx[r]]) for r in range(len(gidx)))
        bound = 2 * p * LAM * (math.sqrt(n) + math.sqrt(p)) * u * xmax * amp
        assert np.abs(R[gidx, :] - Rg).max(initial=0) <= bound * xmax, (layout, np.abs(R[gidx, :] - Rg).max())
        dropped = [j for j in range(p) if j not in gidx]
        assert np.all(R[dropped, :] == 0) and np.all(Q[:, dropped] == 0), layout
        assert np.abs(Q - oQ).max() <= bound, (layout, np.abs(Q - oQ).max())
        for j, c in enumerate(layout):
            if c == "g" and j > 0:
                w = ctx.from_host(Xs[:, j])
                h1, _ = mgs_once(ctx, w, X[:j])
                h2, beta = mgs_once(ctx, w, X[:j])
                assert np.any(h2 != 0), layout                  # the DGKS sweep had something to correct
                assert np.array_equal(R[:j, j], h1 + h2) and R[j, j] == beta, layout
                assert tol < beta < 100 * tol
                w.free()
    ctx.close()


@pytest.mark.parametrize("dtype", [f64, f32])
@pytest.mark.parametrize("k", [1, 96, 97, 300])
def test_block_reorthogonalize(dtype, k):
    """b2k_block_reorthogonalize (one MGS sweep per block column) against the oracle's block_reorthogonalize on the
    stored values, p = 1, 2, 8, 12; bound: orth_tols for one pass (its coefficients and updates are those of a
    classical pass, taken one basis column at a time)."""
    n = 9973
    u = unit(dtype)
    rng = np.random.default_rng(k)
    ctx = kk.B200Context(n, k + 24, dtype=dtype)
    V = ctx.empty_range(k)
    Vs = put(V, qbasis(n, k), dtype)
    Vl = list(Vs.T)
    for p in (1, 2, 8, 12):
        R = ctx.empty_range(p)
        A = rng.standard_normal((n, p)) + Vs[:, :1] * 3.0
        Rs = put(R, A, dtype)
        ctx.check(ctx.lib.b2k_block_reorthogonalize(ctx.h, handles(R), p, handles(V), k))
        out = get(R)
        ref = ko.block_reorthogonalize([Rs[:, i].copy() for i in range(p)], Vl)
        for i in range(p):
            _, tv = orth_tols(n, k, u, float(np.linalg.norm(Rs[:, i])), 1)
            assert np.linalg.norm(out[:, i] - ref[i]) <= tv, (p, i, np.linalg.norm(out[:, i] - ref[i]), tv)
        del R
    ctx.close()


# ------------------------------------------------------------------------------------------ 6. Float32 end to end --

@pytest.mark.parametrize("fast", [False, True], ids=["reference", "fast_block"])
def test_float32_blocklanczos_toric_code(fast):
    """Float32 BlockLanczos with a block of 5 on -H of the 3 x 3 toric code (integer spectrum; the four-fold -16 is
    two units below the next level).  A converged Ritz value has an eigenvalue within its residual norm (<= tol) plus
    the rounding of the projected problem (~ krylovdim u |H|, |H| <= 16); with tol = 1e-3 that eigenvalue is -16.
    The Ritz vectors are orthonormal to the loss of orthogonality of a Float32 basis: krylovdim LAM sqrt(n) u."""
    H = ko.toric_code_hamiltonian(3, 3)
    n = H.shape[0]
    u = unit(f32)
    rng = np.random.default_rng(1)
    X0 = [rng.random(n) for _ in range(5)]
    ctx = kk.B200Context(n, 120, dtype=f32)
    op = kk.B200CSR.from_scipy(ctx, (-H).tocsr())
    kd, tol = 40, 1e-3
    alg = kk.BlockLanczos(tol=tol, krylovdim=kd, maxiter=30, verbosity=0, fast_block=fast)
    with profiled(ctx) as cnt:
        D, U, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
    assert cnt[BPROJ] > 0 and cnt[BUPD] > 0, cnt
    assert info.converged >= 4
    assert np.all(np.abs(np.asarray(D[:4]) + 16.0) <= tol + kd * u * 16.0 * 16), D[:4]
    G = np.column_stack([x.to_host() for x in U[:4]]).astype(f64)
    assert np.abs(G.T @ G - np.eye(4)).max() <= kd * LAM * math.sqrt(n) * u
    ctx.close()


@pytest.mark.parametrize("fast", [False, True], ids=["reference", "fast_block"])
def test_float32_blocklanczos_block_of_8(fast):
    """Float32 BlockLanczos with p = 8 on the 5-point Laplacian, so the PP = 8 block kernels run inside a solve (its
    clustered low end converges slowly in Float32: 40 restarts leave the first two pairs converged): each of the four
    Ritz values lies within its residual norm (plus krylovdim u |A|, |A| <= 8) of an eigenvalue of the closed
    form, and the Ritz vectors are orthonormal to krylovdim LAM sqrt(n) u."""
    nx, ny = 61, 47
    n = nx * ny
    u = unit(f32)
    X0 = [ko.splitmix_vector(300 + i, n) for i in range(8)]
    ctx = kk.B200Context(n, 120, dtype=f32)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    kd = 48
    alg = kk.BlockLanczos(tol=1e-3, krylovdim=kd, maxiter=40, verbosity=0, fast_block=fast)
    with profiled(ctx) as cnt:
        D, U, info = kk.eigsolve(op, kk.Block([ctx.from_host(x) for x in X0]), 4, "SR", alg)
    assert cnt[BPROJ] > 0 and cnt[BUPD] > 0, cnt
    assert info.converged >= 1
    lam = np.sort(ko.laplace_eigenvalues(nx, ny))
    for d, r in zip(D[:4], info.normres[:4]):
        assert np.abs(lam - d).min() <= r + kd * u * 8.0 * 8, (d, r)
    G = np.column_stack([x.to_host() for x in U[:4]]).astype(f64)
    assert np.abs(G.T @ G - np.eye(4)).max() <= kd * LAM * math.sqrt(n) * u
    ctx.close()
