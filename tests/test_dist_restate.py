"""CPU tests of the row-sharded composition (tests/dist_restate.py) that test_gpu_zz_dist_restate.py holds the sharded
kernels to: with one rank it is the single-GPU restatement; on small integers every composed value is exact; and on
the data the GPU test uses, the rank-order fold gives different bits than the reverse fold, than a fold that starts
from d_0 instead of 0.0, than the lane tree coef_colsum forms over three rank sets, and than the unsharded order, so
a kernel or transport that moves a cross-rank sum fails there.  The same three kinds of test hold the compositions
of the other sharded entry points (project, the orthogonalizers, the Lanczos families, the CG / BiCGStab steps and
the dense adjoint): one rank is the single-GPU restatement, integers are exact, and on the worker's data a sum that is
missing, doubled, reversed or unsharded changes the records."""
import numpy as np
import pytest

import dist_restate as D
import spmv_restate as R
import tsk_restate as ts
from test_gpu_blas1 import fma  # noqa: F401  (fixture: correctly rounded fused multiply-add on the host)

f64, f32 = np.float64, np.float32
BIG = 1e16          # ulp(1e16) = 2


@pytest.mark.parametrize("dt", [f64, f32])
@pytest.mark.parametrize("kernel", ["stream", "pipe"])
def test_one_rank_is_the_single_gpu_restatement(fma, dt, kernel):
    n = 3000
    rowptr, cols, vals = D.band_csr(n, 40, 40, 1)
    vals = vals.astype(dt)
    rng = np.random.default_rng(2)
    x, v, s = (rng.standard_normal(n).astype(dt) for _ in range(3))
    rb = R.tiles(rowptr)
    grid = len(rb) - 1 if kernel == "stream" else 1
    for kw in (dict(dotv=v), dict(xscale=-0.7, dot_self=True, shifted=True, a0=0.3, a1=-1.25),
               dict(dotv=v, dsub=s, dsc=-0.45)):
        want = R.apply(fma, dt, kernel, grid, x, csr=(rowptr, cols, vals), rowblk=rb, **kw)
        got = D.spmv(fma, dt, kernel, grid, x, 0, n, csr=D.local_csr(rowptr, cols, vals, 0, n), **kw)
        for a, b in zip(got[:2], want[:2]):
            assert np.array_equal(a, b)
        assert (got[2] is None and want[2] is None) or D.fold([got[2]]) == want[2]
    nx, ny = 50, 60
    st = (nx, ny, 1, (4.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0))
    xs = rng.standard_normal(nx * ny).astype(dt)
    want = R.apply(fma, dt, "stencil", 2, xs, stencil=st, dot_self=True)
    got = D.spmv(fma, dt, "stencil", 2, xs, 0, nx * ny, stencil=st, dot_self=True)
    assert np.array_equal(got[0], want[0]) and got[2] == want[2]


def test_stencil_csr_is_the_assembled_order(fma):
    """the host CSR of the assembled stencil gives the matrix-free stencil's rows, shard by shard"""
    dims, co = (17, 13, 11), (4.0, -1.4, -0.6, -1.2, -0.8, -0.3, -0.7)
    csr = D.stencil_csr(*dims, co, f64)
    n = int(np.prod(dims))
    x = np.random.default_rng(4).standard_normal(n)
    sizes = [3 * 17 * 13, 8 * 17 * 13]
    off = D.offsets(sizes)
    for p, m in enumerate(sizes):
        a = D.spmv(fma, f64, "pipe", 3, x, off[p], m, csr=D.local_csr(*csr, off[p], m))[0]
        b = D.spmv(fma, f64, "stencil", 3, x, off[p], m, stencil=(*dims, co))[0]
        assert np.array_equal(a, b)


@pytest.mark.parametrize("dt", [f64, f32])
def test_integer_data_is_exact(fma, dt):
    """every row, halo entry and rank partial counted once: the composed y and dot are A x and <v, A x>"""
    sizes = [700, 1900, 1100]
    n = sum(sizes)
    rowptr, cols, vals = D.band_csr(n, 57, 9, 3, ints=True)
    A = np.zeros((n, n))
    np.add.at(A, (np.repeat(np.arange(n), np.diff(rowptr)), cols), vals)
    rng = np.random.default_rng(5)
    x, v = rng.integers(-3, 4, n).astype(dt), rng.integers(-3, 4, n).astype(dt)
    off = D.offsets(sizes)
    ys, ds = [], []
    for p, m in enumerate(sizes):
        y, _, d = D.spmv(fma, dt, "pipe", 2, x, off[p], m, csr=D.local_csr(rowptr, cols, vals.astype(dt), off[p], m),
                         dotv=v, shifted=True, a0=2.0, a1=-1.0)
        ys.append(y)
        ds.append(d)
    want = 2.0 * x.astype(f64) - A @ x.astype(f64)
    assert np.array_equal(np.concatenate(ys).astype(f64), want)
    assert D.fold(ds) == v.astype(f64) @ want


def test_lanczos_step_on_integers_is_exact(fma):
    """the composed step on a diagonal operator with integer data: alpha0 = <v, A v>, the coefficients <q_j, x>, the
    update x - sum_j h_j q_j and ||w||^2 all exact"""
    sizes = [600, 1000, 800]
    n = sum(sizes)
    rng = np.random.default_rng(6)
    d = rng.integers(-2, 3, n).astype(f64)
    csr = (np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64), d)
    V = np.zeros((n, 3))
    for j in range(3):                       # disjoint unit-like columns: every h_j an integer
        V[j * 7:(j + 1) * 7 + 1, j] = 1.0
    r = rng.integers(-2, 3, n).astype(f64)
    ws, v, a0, alpha, beta, n2 = D.lanczos_step(fma, f64, sizes, V, r, 1.0, csr, "pipe", [1, 1, 1], 132)
    w = d * r
    assert a0 == r @ w
    x = w - V[:, -1] * 1.0 - a0 * r
    Q = np.column_stack([V, r])
    h = Q.T @ x
    assert alpha == a0 + h[-1]
    x2 = x - Q @ h
    assert np.array_equal(np.concatenate(ws), x2) and n2 == x2 @ x2 and beta == np.sqrt(x2 @ x2)


def test_the_fold_tells_the_orders_apart():
    """three rank partials: the rank-order fold from 0.0 against the reverse fold and against coef_colsum's lane tree
    (lanes 0, 1, 2 hold the sets; xor 2 adds sets 0 and 2 first); two: against a fold that starts from d_0 (signed
    zeros)"""
    d = [1.0, BIG, -BIG]
    assert D.fold(d) == (1.0 + BIG) - BIG == 0.0
    assert D.fold(d[::-1]) == (-BIG + BIG) + 1.0 == 1.0
    d = [BIG, 1.0, -BIG]
    assert D.fold(d) == 0.0
    assert ts.colsum(np.array(d)[:, None])[0] == (BIG - BIG) + 1.0 == 1.0
    d2 = [-0.0, -0.0]
    assert np.signbit(d2[0] + d2[1]) and not np.signbit(D.fold(d2))


@pytest.mark.parametrize("nranks", [2, 3])
@pytest.mark.parametrize("dt", [f64, f32])
def test_the_gpu_data_tells_the_orders_apart(fma, dt, nranks):
    """on the data of the GPU test's fold case the composed dot differs from the single-GPU launch over all rows and,
    at three ranks, from the reverse fold and from the lane tree"""
    sizes, csr, x, v = D.fold_case(dt, nranks)
    off = D.offsets(sizes)
    ds = [D.spmv(fma, dt, "pipe", 2, x, off[p], m, csr=D.local_csr(*csr, off[p], m), dotv=v)[2]
          for p, m in enumerate(sizes)]
    composed = D.fold(ds)
    if nranks == 3:
        assert composed != D.fold(ds[::-1])
        assert composed != ts.colsum(np.array(ds)[:, None])[0]
    _, _, whole = R.apply(fma, dt, "pipe", 2, x, csr=csr, rowblk=R.tiles(csr[0]), dotv=v)
    assert composed != whole


# ------------------------------------------------------------------------------ the other sharded entry points ----

NSM = 132
ETA = 1.0 / np.sqrt(2.0)
TINY = {f64: 1e-9, f32: 1e-4}          # well above the rounding of T: IR runs a second pass
KCAP = {f64: 128, f32: 256}
CGS, MGS, CGS2, MGS2, CGSIR, MGSIR, MGS2B = range(7)


def ragged(nranks):
    """the worker's shards: fold_case's, with n_p % 256 != 0 and n_p % 4 != 0 on the last ranks"""
    return [2100, 1303, 2597] if nranks == 3 else [3403, 2597]


def scaled(sizes, a):
    a = np.array(a, dtype=f64)
    off = D.offsets(sizes)
    for p in range(len(sizes)):
        a[off[p]:off[p + 1]] *= (1.0, 2.0 ** -20, -1.0)[p % 3]
    return a


def test_one_rank_is_the_single_gpu_engine_and_blas1(fma):
    """with one rank every new composition is the single-GPU restatement: tsk_restate's project and classical passes,
    lsmr_restate's k_dot sum and pipelined MGS sweep"""
    import lsmr_restate as LS
    for dt in (f64, f32):
        n = 3001
        rng = np.random.default_rng(8)
        Q = rng.standard_normal((n, KCAP[dt] + 3)).astype(dt)
        v = rng.standard_normal(n).astype(dt)
        assert np.array_equal(D.project(fma, [n], Q, v, NSM), ts.project(Q, v, NSM, fma))
        h, w, n2 = D.cgs_pass(fma, [n], Q, v, NSM)
        wh, ww, wn2 = ts.cgs(Q, v, 1, NSM, fma)
        assert np.array_equal(h, wh) and np.array_equal(w, ww) and n2 == wn2
        h, nrm, passes, w = D.orthogonalize(fma, [n], Q[:, :9], v, CGS2, 0.0, NSM)
        wh, ww, wn2 = ts.cgs(Q[:, :9], v, 2, NSM, fma)
        assert np.array_equal(h, wh) and np.array_equal(w, ww) and nrm == np.sqrt(wn2) and passes == 2
        assert D.dot(fma, dt, [n], v, Q[:, 0], NSM) == LS.blas1_sum(fma, dt, v, Q[:, 0], LS.grid_for(n, 8, NSM))
        _, w = D.mgs_sweep(fma, [n], Q[:, :6], v, NSM)
        assert np.array_equal(w, LS.mgs(fma, dt, Q[:, :6].T, v, NSM))


@pytest.mark.parametrize("dt", [f64, f32])
def test_one_rank_cg_and_bicgstab_steps_are_the_single_gpu_formulas(fma, dt):
    """one rank: the steps are test_gpu_blas1's restatement with the SpMV's fused dot and the blas1_sum sums"""
    import lsmr_restate as LS
    n = 3001
    csr = D.band_csr(n, 20, 20, 9)
    csr = (csr[0], csr[1], csr[2].astype(dt))
    rng = np.random.default_rng(10)
    x, r, p, v, rs = (rng.standard_normal(n).astype(dt) for _ in range(5))
    rb = R.tiles(csr[0])
    g = LS.grid_for(n, 8, NSM)
    xn, rn, pn, q, pq, nr, _, _ = D.cg_step(fma, dt, [n], x, r, p, csr, "pipe", [3], NSM, 0.3, 1.5, 0.6, 1.3)
    wq, _, wpq = R.apply(fma, dt, "pipe", 3, pn, csr=csr, rowblk=rb, dotv=pn, shifted=True, a0=0.3, a1=1.5)
    assert np.array_equal(pn, (r + dt(0.6) * p).astype(dt)) and np.array_equal(q, wq) and pq == wpq
    al = dt(1.3 / pq)
    assert np.array_equal(xn, fma(al, pn, x, dt)) and np.array_equal(rn, fma(-al, wq, r, dt))
    assert nr == np.sqrt(LS.blas1_sum(fma, dt, rn, rn, g))
    pn, vn, sn, sg, ns, _, _ = D.bicgstab_half(fma, dt, [n], rs, r, p, v, csr, "pipe", [3], NSM, 0.0, 1.0, 0.9, 0.45,
                                               1.1, 0)
    wv, _, wsg = R.apply(fma, dt, "pipe", 3, pn, csr=csr, rowblk=rb, dotv=rs)
    assert np.array_equal(vn, wv) and sg == wsg
    assert np.array_equal(sn, fma(-dt(1.1 / sg), wv, r, dt)) and ns == np.sqrt(LS.blas1_sum(fma, dt, sn, sn, g))
    xn, rn, tn, om, nr, rho, _ = D.bicgstab_full(fma, dt, [n], x, rs, pn, sn, csr, "pipe", [3], NSM, 0.0, 1.0,
                                                 1.1 / sg)
    wt, _, wts = R.apply(fma, dt, "pipe", 3, sn, csr=csr, rowblk=rb, dotv=sn)
    assert np.array_equal(tn, wt) and om == wts / LS.blas1_sum(fma, dt, wt, wt, g)
    assert nr == np.sqrt(LS.blas1_sum(fma, dt, rn, rn, g)) and rho == LS.blas1_sum(fma, dt, rs, rn, g)


@pytest.mark.parametrize("dt", [f64, f32])
def test_integer_orthogonalizers_and_steps_are_exact(fma, dt):
    """small integers on three unequal shards: every coefficient, norm and update of the composed orthogonalizers,
    vector orthogonalizers, CG step and dense adjoint is the exact value, so every rank partial is counted once"""
    sizes = [700, 1903, 1097]
    n = sum(sizes)
    rng = np.random.default_rng(11)
    Q = np.zeros((n, 4), dtype=dt)
    Q[[5, 800, 2599, 3600], [0, 1, 2, 3]] = 1.0      # unit columns on every shard: h = v at those rows, exactly
    v = rng.integers(-3, 4, n).astype(dt)
    h = Q.astype(f64).T @ v.astype(f64)
    w = v.astype(f64) - Q.astype(f64) @ h
    for alg in range(7):
        gh, gn, _, gv = D.orthogonalize(fma, sizes, Q, v, alg, 0.0, NSM)
        assert np.array_equal(gv.astype(f64), w) and np.array_equal(gh, h) and gn == np.sqrt(w @ w), alg
    assert np.array_equal(D.project(fma, sizes, Q, v, NSM), h)
    q = Q[:, 1]
    s = float(q.astype(f64) @ v.astype(f64))
    for alg in range(7):
        gs, gn, gv, _ = D.vec_orthogonalize(fma, sizes, q, v, alg, 0.0, NSM)
        ww = v.astype(f64) - s * q.astype(f64)
        assert gs == s and np.array_equal(gv.astype(f64), ww) and gn == np.sqrt(ww @ ww), alg
    A = rng.integers(-3, 4, (n, 5)).astype(dt)
    assert np.array_equal(D.dense_adjoint(fma, sizes, A, v, NSM).astype(f64), A.astype(f64).T @ v.astype(f64))
    # CG with rho = <p, q>: alpha = 1, so x' = x + p and r' = r - q exactly
    csr = (np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64), rng.integers(-2, 3, n).astype(dt))
    x, r = rng.integers(-3, 4, n).astype(dt), rng.integers(-3, 4, n).astype(dt)
    q = csr[2].astype(f64) * r
    pq = float(r.astype(f64) @ q)
    xn, rn, _, _, gpq, nr, _, _ = D.cg_step(fma, dt, sizes, x, r, r, csr, "pipe", [1, 1, 1], NSM, 0.0, 1.0, 0.0, pq)
    assert gpq == pq and np.array_equal(xn.astype(f64), x + r.astype(f64))
    assert np.array_equal(rn.astype(f64), r - q) and nr == np.sqrt((r - q) @ (r - q))


def compositions(fma, dt, nranks, unsharded=False):
    """the worker's compositions on its data (one per group the host restates): name -> () -> every double and
    vector they produce; unsharded: the same data restated on one rank"""
    sizes = ragged(nranks)
    n = sum(sizes)
    rng = np.random.default_rng([61, int(dt == f64)])
    Q = np.linalg.qr(rng.standard_normal((n, 12)))[0].astype(dt)
    v = scaled(sizes, rng.standard_normal(n)).astype(dt)
    Qk = rng.standard_normal((n, KCAP[dt] + 1)).astype(dt)
    q = scaled(sizes, rng.standard_normal(n))
    q = (q / np.linalg.norm(q)).astype(dt)
    _, csr, _, _ = D.fold_case(dt, 3)
    V = (rng.standard_normal((n, 8)) / np.sqrt(n)).astype(dt)
    r = scaled(sizes, rng.standard_normal(n))
    r = (1.7 * r / np.linalg.norm(r)).astype(dt)
    x, p, s = (scaled(sizes, rng.standard_normal(n)).astype(dt) for _ in range(3))
    near = (Q[:, :8] @ rng.standard_normal(8) + TINY[dt] * rng.standard_normal(n)).astype(dt)
    nearq = (3.0 * q + TINY[dt] * rng.standard_normal(n)).astype(dt)
    grids = [3] * nranks
    if unsharded:
        sizes, grids = [n], [3]
    out = {"project": lambda: D.project(fma, sizes, Qk, v, NSM),
           "dense adjoint": lambda: D.dense_adjoint(fma, sizes, Qk[:, :40], v, NSM)}
    for alg in range(7):
        out[f"orthogonalize {alg}"] = lambda alg=alg: D.orthogonalize(fma, sizes, Q[:, :8], v, alg, 0.0, NSM)
        out[f"vec_orthogonalize {alg}"] = lambda alg=alg: D.vec_orthogonalize(fma, sizes, q, v, alg, 0.0, NSM)
    for alg in (CGSIR, MGSIR):
        out[f"orthogonalize {alg} near span"] = lambda alg=alg: D.orthogonalize(fma, sizes, Q[:, :8], near, alg,
                                                                                ETA, NSM)
        out[f"vec_orthogonalize {alg} near q"] = lambda alg=alg: D.vec_orthogonalize(fma, sizes, q, nearq, alg, ETA,
                                                                                     NSM)
    for alg in (CGS, CGSIR, MGS, MGS2, MGSIR, MGS2B):
        out[f"lanczos_expand {alg}"] = lambda alg=alg: D.lanczos_expand(
            fma, dt, sizes, V, r, 1.7, csr, "pipe", grids, NSM, alg, 0.95 if alg in (CGSIR, MGSIR) else 0.0)
    out["cg_step"] = lambda: D.cg_step(fma, dt, sizes, x, v, p, csr, "pipe", grids, NSM, 0.3, 1.5, 0.6, 1.3)[:6]
    out["bicgstab_half"] = lambda: D.bicgstab_half(fma, dt, sizes, v, x, p, s, csr, "pipe", grids, NSM, 0.0, 1.0,
                                                   0.9, 0.45, 1.1, 0)[:5]
    out["bicgstab_full"] = lambda: D.bicgstab_full(fma, dt, sizes, x, v, p, s, csr, "pipe", grids, NSM, 0.2, 0.9,
                                                   0.7)[:6]
    return out


def flat(res):
    return b"".join(np.asarray(t, dtype=np.asarray(t).dtype).tobytes() for t in
                    (res if isinstance(res, tuple) else (res,)))


FOLD = D.fold
FOLDS = {
    "reverse": lambda parts: FOLD(parts[::-1]),
    "missing": lambda parts: FOLD(parts[:1]),
    "doubled": lambda parts: FOLD(list(parts) + list(parts)),
}


# where these partials add exactly in either order (Float32 partials carry about 30 bits, so 1 + 2^-20 + -1 rounds
# nowhere) or the one-rank launch happens to round alike, the other alterations still tell the sums apart
SAME_REVERSED = {"lanczos_expand 1", "vec_orthogonalize 4 near q", "vec_orthogonalize 5 near q",
                 "bicgstab_half", "bicgstab_full"}
SAME_UNSHARDED = {("float64", 2): {"cg_step"}}


@pytest.mark.parametrize("nranks", [2, 3])
@pytest.mark.parametrize("dt", [f64, f32])
def test_the_gpu_data_tells_the_sums_apart(fma, dt, nranks, monkeypatch):
    """on the worker's data every composition changes when its cross-rank sums are missing (rank 0's partial alone)
    or doubled, and nearly every one when they are left unsharded (one rank over all rows) or, at three ranks in
    Float64, folded in reverse (with two the addition commutes).  (A fold that starts from d_0 instead of 0.0
    differs only on signed zeros: test_the_fold_tells_the_orders_apart.)"""
    base = {k: flat(f()) for k, f in compositions(fma, dt, nranks).items()}
    for name, alt in FOLDS.items():
        if name == "reverse" and (nranks == 2 or dt == f32):
            continue
        monkeypatch.setattr(D, "fold", alt)
        for k, f in compositions(fma, dt, nranks).items():
            if not (name == "reverse" and k in SAME_REVERSED):
                assert flat(f()) != base[k], (name, k)
    monkeypatch.setattr(D, "fold", FOLD)
    same = SAME_UNSHARDED.get((np.dtype(dt).name, nranks), set())
    for k, f in compositions(fma, dt, nranks, unsharded=True).items():
        if k not in same:
            assert flat(f()) != base[k], ("unsharded", k)


@pytest.mark.parametrize("dt", [f64, f32])
def test_the_ir_cases_reorthogonalise(fma, dt):
    """the near-span data of the worker makes CGSIR and MGSIR run a second pass, and eta = 0.95 makes the IR Lanczos
    steps reorthogonalise: the pass count is then part of what the device must match"""
    out = compositions(fma, dt, 3)
    for alg in (CGSIR, MGSIR):
        assert out[f"orthogonalize {alg} near span"]()[2] >= 2
        assert out[f"vec_orthogonalize {alg} near q"]()[3] >= 2
        assert out[f"lanczos_expand {alg}"]()[4] >= 2
