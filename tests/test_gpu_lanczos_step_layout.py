"""GPU tests of the Lanczos step's Gram-Schmidt sweeps with the three-term prologue taken from the panel ring.

The sweeps of a CGS2 Lanczos step list the basis columns rotated by two, [v_prev, v, q_0, ...], form
w' = (w - beta v_prev) - alpha v per row from the first chunk of each tile in both sweeps (w' is never stored), and
let the producer warps run through the phase boundary.  The column widths below put the rotated chunk boundaries on
every side of v_prev and v (8 columns a chunk in Float64, 16 in Float32, up to a full 12-chunk ring), at row counts
with a ragged last tile, with fewer row tiles than SMs and with CTAs that own two tiles (the chained batch also with
full tiles only and with CTAs that own four).

1. A device-chained batch equals the loop of synchronous steps bit for bit.
2. One synchronous step (fused sweep, split sweeps, and the launch per phase) equals the same step recomputed from
   primitives that stream one vector through the original column order: vec_axpy2 for the prologue, basis_project and
   basis_unproject for the pass.  Not to the bit: the primitives take <v, A v> and the coefficients from other
   reductions.  v is a combination of all the basis columns, so every coefficient is O(|w|) and a wrong column,
   coefficient or operand shows as an O(1) error.
"""
import ctypes as C
import gc
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.factorizations import lanczos as lz
from krylovkit_jl_b200.vectors import handles
from oracle import krylov_oracle as ko

SEED = 20260923
LAM = 8.0
f64, f32 = np.float64, np.float32
# (nx, ny) of the stencil: 5917 rows = 23 full tiles + 29 rows on 24 CTAs; 36503 rows = 142 full tiles + 151 rows,
# so with 132 SMs some CTAs own two tiles
SIZES = [(97, 61), (211, 173)]
SIZE_IDS = ["n5917", "n36503"]
# the chained batch also at 8192 rows = 32 full tiles (no ragged tile) and 105463 rows = 411 full tiles + 247 rows, so
# with 132 SMs the CTA that owns the ragged tile owns four
CHAIN_SIZES = SIZES + [(128, 64), (401, 263)]
CHAIN_SIZE_IDS = SIZE_IDS + ["n8192", "n105463"]


def unit(dtype):
    return 2.0 ** -53 if dtype == f64 else 2.0 ** -24


def run_batch(chain, dtype, nsteps, nx, ny):
    """initialize + one b2k_lanczos_expand_many batch from k = 1; chain False = the loop of synchronous steps"""
    lib = L.load()
    lib.b2k_debug_set_chain(1 if chain else 0)
    try:
        n = nx * ny
        ctx = kk.B200Context(n, nsteps + 8, dtype=dtype)
        op = kk.B200CSR.stencil(ctx, nx, ny)
        x0 = ctx.from_host(ko.splitmix_vector(SEED, n, dtype=dtype))
        it = lz.LanczosIterator(op, x0, kk.cgs2)
        f = lz.initialize(it)
        l0 = ctx.launches
        done = lz.expand_many_(it, f, nsteps, 0.0)
        nl = ctx.launches - l0
        assert done == nsteps
        out = (np.array(f.alphas), np.array(f.betas), np.column_stack([v.to_host() for v in f.V]), f.r.to_host(), nl)
        del f, it, x0
        gc.collect()
        ctx.close()
        return out
    finally:
        lib.b2k_debug_set_chain(1)


@pytest.mark.parametrize("nx,ny", CHAIN_SIZES, ids=CHAIN_SIZE_IDS)
@pytest.mark.parametrize("dtype,K1max", [(f64, 96), (f32, 192)], ids=["float64", "float32"])
def test_chained_batch_equals_stepping(dtype, K1max, nx, ny):
    """A batch from k = 1 to K1 = K1max runs one chained step at every K1 in 2..K1max (among them 2, 3, 8, 9, 10, 16,
    17, 60, 95, 96 in Float64 and 2, 16, 17, 18, 192 in Float32): alpha, beta, V and r equal the stepping loop's."""
    nsteps = K1max - 1
    a1, b1, V1, r1, nl1 = run_batch(True, dtype, nsteps, nx, ny)
    a0, b0, V0, r0, nl0 = run_batch(False, dtype, nsteps, nx, ny)
    assert nl1 <= 2 * nsteps + 2 and nl0 >= 3 * nsteps, (nl1, nl0)     # the batch was chained, the loop was not
    assert np.array_equal(a1, a0) and np.array_equal(b1, b0)
    assert np.array_equal(V1, V0) and np.array_equal(r1, r0)


_Q = {}


def qbasis(n, k):
    if n not in _Q or _Q[n].shape[1] < k:
        _Q[n] = np.linalg.qr(np.random.default_rng(n).standard_normal((n, max(k, 129))))[0]
    return _Q[n][:, :k]


def lanczos_expand(ctx, op, V, r, w, beta_old):
    a, b = C.c_double(), C.c_double()
    ctx.check(ctx.lib.b2k_lanczos_expand(ctx.h, op.h, handles(V + [r]), len(V), r.handle, w.handle, beta_old,
                                         kk.cgs2.tag, kk.cgs2.eta, C.byref(a), C.byref(b)))
    return a.value, b.value


def set_coop(on):
    L.load().b2k_debug_set_coop(1 if on else 0)


STEP_CASES = ([(f64, K1) for K1 in (2, 3, 8, 9, 10, 16, 17, 60, 95, 96, 97, 128)] +
              [(f32, K1) for K1 in (2, 16, 17, 18, 192, 193)])


@pytest.mark.parametrize("nx,ny", SIZES, ids=SIZE_IDS)
@pytest.mark.parametrize("dtype,K1", STEP_CASES, ids=[f"{np.dtype(d).name}-K{K1}" for d, K1 in STEP_CASES])
def test_step_matches_primitives(dtype, K1, nx, ny):
    """b2k_lanczos_expand (CGS2) with K1 = k + 1 basis vectors after push!: the fused sweep up to 96 / 192 columns, the
    split sweeps above.  The cooperative launch and the launch per phase give the same bits; w and alpha agree with
    the step recomputed from primitives to the rounding of the reductions they take from other kernels."""
    n = nx * ny
    u = unit(dtype)
    k = K1 - 1
    Qf = qbasis(n, K1)
    ctx = kk.B200Context(n, K1 + 8, dtype=dtype)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    Vvecs = ctx.empty_range(k)
    for j, q in enumerate(Vvecs):
        q.upload(Qf[:, j].astype(dtype))
    beta_old = 2.5
    c = np.random.default_rng(K1).uniform(0.5, 1.5, K1)
    v = Qf @ c
    rh = (beta_old / np.linalg.norm(v) * v).astype(dtype)
    r = ctx.from_host(rh)
    runs = {}
    try:
        for on in (True, False):
            r.upload(rh)
            w = ctx.empty()
            set_coop(on)
            a, b = lanczos_expand(ctx, op, Vvecs, r, w, beta_old)
            runs[on] = (a, b, w.to_host())
            w.free()
    finally:
        set_coop(True)
    a, b, wd = runs[True]
    assert (a, b) == runs[False][:2] and np.array_equal(wd, runs[False][2])
    # r now holds v = r / beta_old as the step rounded it; recompute the step from primitives
    basis = Vvecs + [r]
    w = ctx.empty()
    op.apply_into(w, r)
    alpha0 = kk.inner(r, w)
    ctx.check(ctx.lib.b2k_vec_axpy2(ctx.h, w.handle, Vvecs[-1].handle, -beta_old, r.handle, -alpha0))
    h = np.zeros(K1)
    kk.project_(h, kk.OrthonormalBasis(basis), w)
    kk.unproject_(w, kk.OrthonormalBasis(basis), h, -1.0, 1.0)
    wr = w.to_host().astype(f64)
    ar = alpha0 + h[-1]
    # |w'| <= |A v| + beta_old + |alpha0| <= 2 |A v| + beta_old; coefficient errors of n-term sums, update errors of
    # K1 + 3 terms
    s = 2 * float(np.linalg.norm(ko.stencil_matrix(nx, ny) @ r.to_host().astype(f64))) + beta_old
    eh = LAM * math.sqrt(n) * u * s
    ew = math.sqrt(K1) * eh + LAM * math.sqrt(K1 + 3) * u * (1 + math.sqrt(K1)) * s
    assert abs(a - ar) <= 2 * eh, (a, ar, eh)
    assert np.linalg.norm(wd.astype(f64) - wr) <= 2 * ew, (np.linalg.norm(wd.astype(f64) - wr), ew)
    assert abs(b - np.linalg.norm(wr)) <= 2 * ew + 2 * eh
    if dtype == f64:
        # the coefficients are O(|w| / sqrt(K1)): a wrong column or coefficient exceeds the bound many times over (in
        # Float32 the bound of the wider cases is of the coefficients' size; the chained test covers those bitwise)
        assert np.median(np.abs(h)) > 1e3 * 2 * ew, (np.median(np.abs(h)), ew)
    ctx.close()
