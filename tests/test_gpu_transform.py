"""GPU tests of the restart GEMM behind basistransform! (b2k_basis_transform, basis.cu) against an fma-order host
restatement, for every kernel its dispatcher can pick, in Float64 and Float32.

Kernels (b2k_debug_transform_kernel ids): k_transform<double|float, U in shared memory|global> (1-4),
k_transform_big<double|float> (5, 6), k_transform_ur<2,18> / <2,36> / <4,18> (7-9), k_transform_f89 (10),
k_transform_f89w (11), k_transform_hyb (12) and k_transform_dmma (13).  Every GPU case asserts the id the derivation
below predicts, and that exactly one TRANSFORM-class launch ran per call.

Rounding contract.  With U rounded to the vector type T first (the Float32 kernels cast the double U), every kernel
gives
    out[:, j] = fold_i fma(Q[:, i], T(U[i, j]), acc),  i = 0 ... m-1 in increasing order, acc = +0 in T,
bit for bit.  The host restates it with the gcc-built fma of test_gpu_blas1.py (Python has no fused multiply-add).
For the DFMA kernels (ids 1-11, and output columns [24, 36) of k_transform_hyb) the code spells this order out.  For
the DMMA outputs (k_transform_dmma, columns [0, 24) of k_transform_hyb) it is what mma.m8n8k4.f64 was measured to do
on an H100 (DESIGN §3.4): each of its four products is added to the accumulator in k order with one rounding per
product, exactly like four chained fma.  Those outputs are also checked exact on small integers (Q and U in [-8, 8]
keep every partial sum below 2^14, so any order gives the same bits), the contract that holds whatever the order.
After every call the columns [keep, m) and every slab column outside the list are bit-identical to before, and a
second call on the same input gives the same bits.

Dispatch (b2k_basis_transform), restated by expected_kernel().  Shared-memory budgets: TR_U_BYTES = 232448 - 12·16384
- 256 = 35 584 bytes for U beside the ring, TD_U_BYTES = 232448 - 12·16896 - 256 = 29 440 beside the DMMA ring.
  Float64: m > 96 (12 ring chunks of 8) -> big; modes 1-3 with keep <= 36 -> ur; mode 7 -> f89w and modes 0 / 5 -> f89
  (keep <= 36); DMMA if m·ceil8(keep)·8 <= 29 440 (and b2k_debug_set_dmma(1)), as hyb under mode 4 when also keep <= 36
  and m·40·8 <= 29 440 (m <= 92); else k_transform with U in shared memory if m·ceil2(keep)·8 <= 35 584.
  Float32: m > 192 -> big; else k_transform, U in shared memory if m·ceil4(keep)·4 <= 35 584.

Row tiles: 256 rows (k_transform, ur, f89, hyb, dmma), 512 (f89w), 64 (big); grid = min(tiles, SMs) (big: SMs times
the CTAs that fit an SM by shared memory, at most 4).  The SM-derived sizes give every CTA one tile, or two and three
tiles on alternate CTAs (f89's two warp sets both busy), with a ragged last tile; m >= 40 makes the ring wrap across
tiles (5+ chunks per tile) and m = 52 wraps f89w's ring inside one tile (13 chunks of 4 columns).

The module's two CPU tests check the dispatch table against the derivation and the restatement itself at tiny sizes.
"""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.vectors import handles
from oracle import krylov_oracle as ko
from test_gpu_blas1 import fma, num_sms  # noqa: F401  (fma: module fixture)
from test_gpu_paths import LAM, TRANSFORM, profiled, unit

gpu = pytest.mark.gpu
f64, f32 = np.float64, np.float32

(K_F64_SMEM, K_F64_GLOBAL, K_F32_SMEM, K_F32_GLOBAL, K_BIG64, K_BIG32, K_UR218, K_UR236, K_UR418, K_F89, K_F89W,
 K_HYB, K_DMMA) = range(1, 14)
NAME = {K_F64_SMEM: "k_transform<double,smem U>", K_F64_GLOBAL: "k_transform<double,global U>",
        K_F32_SMEM: "k_transform<float,smem U>", K_F32_GLOBAL: "k_transform<float,global U>",
        K_BIG64: "k_transform_big<double>", K_BIG32: "k_transform_big<float>", K_UR218: "k_transform_ur<2,18>",
        K_UR236: "k_transform_ur<2,36>", K_UR418: "k_transform_ur<4,18>", K_F89: "k_transform_f89",
        K_F89W: "k_transform_f89w", K_HYB: "k_transform_hyb", K_DMMA: "k_transform_dmma"}
TR_U_BYTES = 232448 - 12 * 16384 - 256
TD_U_BYTES = 232448 - 12 * 16896 - 256
HYB_DF0 = 24                                      # first DFMA output column of k_transform_hyb


def ceil_to(x, q):
    return -(-x // q) * q


def expected_kernel(dt, m, keep, mode=0, dmma=1):
    """the kernel id b2k_basis_transform launches for this shape under b2k_debug_set_transform(mode) and
    b2k_debug_set_dmma(dmma)"""
    if np.dtype(dt) == f32:
        if m > 192:
            return K_BIG32
        return K_F32_SMEM if m * ceil_to(keep, 4) * 4 <= TR_U_BYTES else K_F32_GLOBAL
    if m > 96:
        return K_BIG64
    ur = mode if mode in (1, 2, 3) else 0
    hyb = {0: 2, 4: 1, 5: 2, 7: 3}.get(mode, 0)
    f89_fits = 4 * m * 10 * 8 <= TR_U_BYTES - 64
    dmma_ok = bool(dmma) and m * ceil_to(keep, 8) * 8 <= TD_U_BYTES
    if ur and keep <= 36:
        return {1: K_UR218, 2: K_UR236, 3: K_UR418}[ur]
    if hyb == 3 and keep <= 36 and f89_fits:
        return K_F89W
    if hyb == 2 and keep <= 36 and f89_fits:
        return K_F89
    if dmma_ok and hyb == 1 and keep <= 36 and m * 40 * 8 <= TD_U_BYTES:
        return K_HYB
    if dmma_ok:
        return K_DMMA
    return K_F64_SMEM if m * ceil_to(keep, 2) * 8 <= TR_U_BYTES else K_F64_GLOBAL


def dmma_columns(kid, keep):
    """output columns computed on the FP64 tensor cores (the weaker contract)"""
    if kid == K_DMMA:
        return list(range(keep))
    if kid == K_HYB:
        return list(range(min(HYB_DF0, keep)))
    return []


def restate(Q, U, dt, fma):
    """out[:, j] = fold_i fma(Q[:, i], T(U[i, j]), acc) for i = 0 ... m-1, acc = +0 in T"""
    Qt = np.asarray(Q, dtype=dt)
    Ut = np.asarray(U, dtype=f64).astype(dt)
    acc = np.zeros((Qt.shape[0], Ut.shape[1]), dtype=dt)
    for i in range(Qt.shape[1]):
        acc = fma(Qt[:, i:i + 1], Ut[i:i + 1, :], acc, dt)
    return acc


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == f64 else np.uint32)


def same_bits(a, b):
    return np.array_equal(bits(a), bits(b))


@contextlib.contextmanager
def dispatch(mode=0, dmma=1):
    lib = L.load()
    lib.b2k_debug_set_transform(mode)
    lib.b2k_debug_set_dmma(dmma)
    try:
        yield lib
    finally:
        lib.b2k_debug_set_transform(0)
        lib.b2k_debug_set_dmma(1)


def make_slab(dt, n, m, layout, rng):
    """(context, slab vectors, positions of the m basis columns in the slab).  Every slab column outside the list
    is a sentinel that must come back unchanged."""
    if layout == "contiguous":
        total, idx = m + 2, list(range(1, m + 1))
    elif layout == "strided":                     # every other column
        total, idx = 2 * m + 1, list(range(1, 2 * m, 2))
    elif layout == "reversed":                    # every other column, last first
        total, idx = 2 * m + 1, list(range(2 * m - 1, 0, -2))
    elif layout in ("shuffled", "space2"):        # a seeded permutation with gaps
        total = m + m // 2 + 2
        idx = [int(i) for i in rng.permutation(total)[:m]]
    else:
        raise ValueError(layout)
    if layout == "space2":                        # a second, non-sharded space of another length
        ctx = kk.B200Context(n + 45, 2, dtype=dt)
        sp = ctx.add_space(n, total, sharded=False)
    else:
        ctx = kk.B200Context(n, total, dtype=dt)
        sp = 0
    return ctx, ctx.empty_range(total, sp), idx


def run_case(fma, dt, m, keep, n, mode=0, dmma=1, layout="contiguous", ldu=None, want=None, seed=0):
    """one b2k_basis_transform (twice) on random data against the contract of the kernel that runs; the DMMA
    kernels once more on small integers"""
    kid = expected_kernel(dt, m, keep, mode, dmma)
    if want is not None:
        assert kid == want, f"derivation gives {NAME[kid]}, the table {NAME[want]}"
    ldu = m if ldu is None else ldu
    rng = np.random.default_rng([seed, m, keep, n, mode, dmma, ldu])
    ctx, slab, idx = make_slab(dt, n, m, layout, rng)
    try:
        lib = ctx.lib
        init = rng.standard_normal((len(slab), n)).astype(dt)
        for v, x in zip(slab, init):
            v.upload(x)
        Q = init[idx].T
        U = rng.standard_normal((m, keep))
        Ubuf = np.full((keep, ldu), np.nan)       # column-major ldu x keep; rows [m, ldu) must never be read
        Ubuf[:, :m] = U.T
        hs = handles([slab[i] for i in idx])

        def call(Uc):
            with profiled(ctx) as cnt:
                ctx.check(lib.b2k_basis_transform(ctx.h, hs, m, Uc.ctypes.data_as(C.POINTER(C.c_double)), ldu, keep))
            got = lib.b2k_debug_transform_kernel()
            assert got == kid, f"ran {NAME.get(got, got)}, expected {NAME[kid]}"
            assert cnt[TRANSFORM] == 1
            return np.stack([v.to_host() for v in slab])

        with dispatch(mode, dmma):
            out = call(Ubuf)
            for i in idx[:keep]:
                slab[i].upload(init[i])
            again = call(Ubuf)
        assert same_bits(out, again), "two calls on the same input differ"
        outputs = set(idx[:keep])
        for c in range(len(slab)):
            if c not in outputs:
                assert same_bits(out[c], init[c]), f"slab column {c} (not an output) changed"
        got = out[idx[:keep]].T
        assert not np.isnan(got).any()
        ref = restate(Q, U, dt, fma)
        bad = np.argwhere(bits(got) != bits(ref))
        if len(bad):
            r, j = bad[0]
            on = "DMMA" if j in dmma_columns(kid, keep) else "DFMA"
            raise AssertionError(f"{NAME[kid]}: {len(bad)} outputs differ from the fma fold, first at row {r}, "
                                 f"column {j} ({on}): {got[r, j]!r} != {ref[r, j]!r}")
        if dmma_columns(kid, keep):
            # small integers: exact in every summation order (the contract of DMMA before its order was measured)
            Qi = rng.integers(-8, 9, (n, m)).astype(dt)
            Ui = rng.integers(-8, 9, (m, keep)).astype(f64)
            for j, i in enumerate(idx):
                slab[i].upload(Qi[:, j])
            Ubuf[:, :m] = Ui.T
            with dispatch(mode, dmma):
                outi = call(Ubuf)
            assert same_bits(outi[idx[:keep]].T, (Qi.astype(f64) @ Ui).astype(dt)), f"{NAME[kid]}: inexact on integers"
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ CPU: the tables --------

# (dtype, m, keep, mode, dmma, kernel): both sides of every dispatch boundary and of each kernel's inner passes
BOUNDARIES = [
    # resident ring width: 96 (f64) / 192 (f32) columns, the staged-tile kernel above; 256 is the limit
    (f64, 96, 36, 0, 1, K_F89), (f64, 97, 36, 0, 1, K_BIG64), (f64, 256, 40, 0, 1, K_BIG64),
    (f32, 192, 40, 0, 1, K_F32_SMEM), (f32, 193, 40, 0, 1, K_BIG32), (f32, 256, 40, 0, 1, K_BIG32),
    # U leaves shared memory
    (f64, 96, 46, 0, 1, K_F64_SMEM), (f64, 96, 47, 0, 1, K_F64_GLOBAL),
    (f32, 192, 44, 0, 1, K_F32_SMEM), (f32, 192, 45, 0, 1, K_F32_GLOBAL),
    # DMMA's shared-memory limit m·ceil8(keep) <= 3680
    (f64, 60, 56, 0, 1, K_DMMA), (f64, 60, 57, 0, 1, K_F64_SMEM),
    (f64, 92, 40, 6, 1, K_DMMA), (f64, 92, 41, 6, 1, K_F64_SMEM),
    # the hybrid's limit m <= 92
    (f64, 92, 36, 4, 1, K_HYB), (f64, 93, 36, 4, 1, K_F64_SMEM), (f64, 93, 32, 4, 1, K_DMMA),
    # the keep <= 36 variants at 36 / 37
    (f64, 60, 36, 1, 1, K_UR218), (f64, 60, 37, 1, 1, K_DMMA), (f64, 60, 36, 2, 1, K_UR236),
    (f64, 60, 36, 3, 1, K_UR418), (f64, 96, 36, 3, 1, K_UR418), (f64, 60, 36, 7, 1, K_F89W),
    (f64, 60, 37, 7, 1, K_DMMA), (f64, 60, 36, 5, 1, K_F89), (f64, 60, 37, 0, 1, K_DMMA),
    (f64, 60, 36, 6, 1, K_DMMA), (f64, 60, 36, 6, 0, K_F64_SMEM), (f64, 60, 37, 6, 0, K_F64_SMEM),
    # k_transform: passes of 36 (f64) / 40 (f32) outputs, halves of 18 / 20
    (f64, 40, 18, 6, 0, K_F64_SMEM), (f64, 40, 19, 6, 0, K_F64_SMEM), (f64, 40, 36, 6, 0, K_F64_SMEM),
    (f64, 40, 37, 6, 0, K_F64_SMEM), (f64, 80, 72, 6, 0, K_F64_GLOBAL), (f64, 80, 73, 6, 0, K_F64_GLOBAL),
    (f32, 40, 20, 0, 1, K_F32_SMEM), (f32, 40, 21, 0, 1, K_F32_SMEM), (f32, 100, 40, 0, 1, K_F32_SMEM),
    (f32, 100, 41, 0, 1, K_F32_SMEM), (f32, 100, 80, 0, 1, K_F32_SMEM), (f32, 100, 81, 0, 1, K_F32_SMEM),
    (f32, 120, 20, 0, 1, K_F32_SMEM), (f32, 120, 80, 0, 1, K_F32_GLOBAL), (f32, 120, 81, 0, 1, K_F32_GLOBAL),
    (f32, 192, 21, 0, 1, K_F32_SMEM),
    # k_transform_big: sweeps of 32 outputs, 8 per thread
    (f64, 100, 8, 0, 1, K_BIG64), (f64, 100, 9, 0, 1, K_BIG64), (f64, 100, 32, 0, 1, K_BIG64),
    (f64, 100, 33, 0, 1, K_BIG64), (f32, 193, 8, 0, 1, K_BIG32), (f32, 193, 9, 0, 1, K_BIG32),
    (f32, 193, 32, 0, 1, K_BIG32), (f32, 193, 33, 0, 1, K_BIG32),
    # ur: two output groups of 18
    (f64, 40, 18, 1, 1, K_UR218), (f64, 40, 19, 1, 1, K_UR218), (f64, 40, 18, 3, 1, K_UR418),
    (f64, 40, 19, 3, 1, K_UR418), (f64, 40, 19, 2, 1, K_UR236),
    # f89 / f89w: four groups of 9
    *[(f64, 40, k, md, 1, kid) for md, kid in ((0, K_F89), (7, K_F89W)) for k in (9, 10, 27, 28, 36)],
    # hyb: DMMA columns [0, 24), DFMA [24, 36) in two warp groups of 6
    *[(f64, 40, k, 4, 1, K_HYB) for k in (24, 25, 30, 31)],
    # DMMA passes of 40 columns: streaming (one pass) / resident
    (f64, 60, 40, 6, 1, K_DMMA), (f64, 60, 41, 6, 1, K_DMMA), (f64, 76, 48, 6, 1, K_DMMA),
    # chunk tails (m % 4, % 8, % 16), m = 1, keep = 1
    (f64, 1, 1, 0, 1, K_F89), (f64, 1, 1, 6, 1, K_DMMA), (f64, 1, 1, 6, 0, K_F64_SMEM), (f64, 1, 1, 1, 1, K_UR218),
    (f64, 1, 1, 4, 1, K_HYB), (f64, 1, 1, 7, 1, K_F89W), (f32, 1, 1, 0, 1, K_F32_SMEM),
    (f64, 13, 5, 0, 1, K_F89), (f64, 13, 5, 6, 1, K_DMMA), (f64, 13, 13, 4, 1, K_HYB), (f64, 29, 7, 1, 1, K_UR218),
    (f64, 29, 7, 7, 1, K_F89W), (f64, 29, 1, 6, 0, K_F64_SMEM), (f32, 45, 7, 0, 1, K_F32_SMEM),
    (f32, 17, 1, 0, 1, K_F32_SMEM), (f64, 101, 1, 0, 1, K_BIG64), (f32, 199, 1, 0, 1, K_BIG32),
]

# one configuration per kernel (and both DMMA pass structures), for the row and layout sweeps
KCONF = [  # (id, dtype, m, keep, mode, dmma)
    ("f64-smem", f64, 40, 37, 6, 0), ("f64-global", f64, 96, 47, 0, 1), ("f32-smem", f32, 40, 21, 0, 1),
    ("f32-global", f32, 192, 45, 0, 1), ("big64", f64, 100, 33, 0, 1), ("big32", f32, 193, 9, 0, 1),
    ("ur2x18", f64, 45, 19, 1, 1), ("ur2x36", f64, 45, 19, 2, 1), ("ur4x18", f64, 45, 19, 3, 1),
    ("f89", f64, 45, 28, 0, 1), ("f89w", f64, 52, 28, 7, 1), ("hyb", f64, 45, 31, 4, 1),
    ("dmma-stream", f64, 45, 36, 6, 1), ("dmma-resident", f64, 45, 41, 6, 1),
]
KCONF_IDS = [c[0] for c in KCONF]
ROWS = [1, 2, 3, 255, 256, 257, 511, 512, 513]


def bid(c):
    dt, m, keep, mode, dm, kid = c
    return f"{np.dtype(dt).name}-m{m}-k{keep}-mode{mode}{'' if dm else '-nodmma'}-{NAME[kid]}"


def test_dispatch_table_matches_the_derivation():
    """every table row is what expected_kernel derives, every kernel appears in the tables, and both sides of each
    dispatcher limit are in BOUNDARIES"""
    for c in BOUNDARIES:
        assert expected_kernel(*c[:5]) == c[5], bid(c)
    seen = {c[5] for c in BOUNDARIES} | {expected_kernel(*c[1:]) for c in KCONF}
    assert seen == set(NAME)
    assert {expected_kernel(*c[1:]) for c in KCONF} == set(NAME)
    have = {c[:5] for c in BOUNDARIES}
    for pair in [((f64, 96, 36, 0, 1), (f64, 97, 36, 0, 1)), ((f32, 192, 40, 0, 1), (f32, 193, 40, 0, 1)),
                 ((f64, 96, 46, 0, 1), (f64, 96, 47, 0, 1)), ((f32, 192, 44, 0, 1), (f32, 192, 45, 0, 1)),
                 ((f64, 60, 56, 0, 1), (f64, 60, 57, 0, 1)), ((f64, 92, 36, 4, 1), (f64, 93, 36, 4, 1))]:
        assert set(pair) <= have
        assert expected_kernel(*pair[0]) != expected_kernel(*pair[1])


def test_restatement_at_tiny_sizes(fma):
    """the host fold: exact on small integers, within the float64 product's bound, U rounded to T first, and
    sensitive to the summation order (a reversed fold differs), so the bitwise contract can tell orders apart"""
    rng = np.random.default_rng(3)
    for dt in (f64, f32):
        n, m, keep = 64, 24, 5
        Qi = rng.integers(-8, 9, (n, m)).astype(dt)
        Ui = rng.integers(-8, 9, (m, keep)).astype(f64)
        assert same_bits(restate(Qi, Ui, dt, fma), (Qi.astype(f64) @ Ui).astype(dt))
        Q = rng.standard_normal((n, m)).astype(dt)
        U = rng.standard_normal((m, keep))
        out = restate(Q, U, dt, fma)
        ref = Q.astype(f64) @ U.astype(dt).astype(f64)
        S = np.abs(Q.astype(f64)) @ np.abs(U.astype(dt).astype(f64))
        assert (np.abs(out - ref) <= LAM * math.sqrt(m) * unit(dt) * S).all()
        one = np.zeros(n, dtype=dt)                # one column by scalar steps
        for i in range(m):
            one = fma(Q[:, i], dt(U[i, 2]), one, dt)
        assert same_bits(out[:, 2], one)
        rev = restate(Q[:, ::-1], U[::-1], dt, fma)
        assert not same_bits(out, rev)
    # U is rounded to float32 before the products
    Q = np.ones((1, 1), dtype=f32)
    U = np.array([[1.0 + 2.0 ** -30]])
    assert restate(Q, U, f32, fma)[0, 0] == f32(1.0)


# ------------------------------------------------------------------------------------------ GPU: shapes ------------

@gpu
@pytest.mark.parametrize("case", BOUNDARIES, ids=[bid(c) for c in BOUNDARIES])
def test_dispatch_boundaries(case, fma):
    dt, m, keep, mode, dm, kid = case
    run_case(fma, dt, m, keep, 513, mode, dm, want=kid)


@gpu
@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("conf", KCONF, ids=KCONF_IDS)
def test_rows(conf, n, fma):
    _, dt, m, keep, mode, dm = conf
    run_case(fma, dt, m, keep, n, mode, dm)


def sm_rows(kid, m, dt, which):
    """rows giving every CTA one tile ('one') or two and three tiles on alternate CTAs ('two-three'), the last tile
    ragged"""
    sms = num_sms()
    esize = np.dtype(dt).itemsize
    if kid in (K_BIG64, K_BIG32):
        R, cap = 64, sms * max(1, min(4, (200 * 1024) // (64 * m * esize)))
    else:
        R, cap = (512 if kid == K_F89W else 256), sms
    tiles = cap if which == "one" else 2 * cap + cap // 2
    return tiles * R - 37


@gpu
@pytest.mark.parametrize("which", ["one", "two-three"])
@pytest.mark.parametrize("conf", [c for c in KCONF if "global" not in c[0]],
                         ids=[c[0] for c in KCONF if "global" not in c[0]])
def test_tiles_per_cta(conf, which, fma):
    _, dt, m, keep, mode, dm = conf
    run_case(fma, dt, m, keep, sm_rows(expected_kernel(dt, m, keep, mode, dm), m, dt, which), mode, dm)


@gpu
@pytest.mark.parametrize("layout", ["strided", "reversed", "shuffled", "space2"])
@pytest.mark.parametrize("conf", KCONF, ids=KCONF_IDS)
def test_column_layouts(conf, layout, fma):
    _, dt, m, keep, mode, dm = conf
    run_case(fma, dt, m, keep, 700, mode, dm, layout=layout)


KEEPALL = [("f64-f89", f64, 0, 1), ("f32", f32, 0, 1), ("dmma", f64, 6, 1), ("f64-smem", f64, 6, 0),
           ("ur2x18", f64, 1, 1), ("hyb", f64, 4, 1), ("f89w", f64, 7, 1)]


@gpu
@pytest.mark.parametrize("m", range(1, 9))
@pytest.mark.parametrize("conf", KEEPALL, ids=[c[0] for c in KEEPALL])
def test_keep_equals_m(conf, m, fma):
    """keep == m at tiny m (the BlockLanczos R_new transform)"""
    _, dt, mode, dm = conf
    run_case(fma, dt, m, m, 300, mode, dm, layout="shuffled")


@gpu
@pytest.mark.parametrize("conf", KCONF, ids=KCONF_IDS)
def test_ldu_larger_than_m(conf, fma):
    """U through the C ABI with ldu = m + 3, NaN in rows [m, ldu): the ur path reads U_host with ldu, the others
    pack it first; no NaN may reach an output"""
    _, dt, m, keep, mode, dm = conf
    run_case(fma, dt, m, keep, 300, mode, dm, ldu=m + 3)


# ------------------------------------------------------------------------------------------ refusals ---------------

@gpu
def test_refusals_leave_every_column_untouched(check_kernel=True):
    """m = 0, keep = 0, keep > m, ldu < m and a repeated handle -> EINVAL; m = 257 -> ENOTSUP; columns from two
    spaces -> EDIM.  Each leaves every column bit-identical, and the context works afterwards.  (Also run on the
    host simulator by test_hostsim.py, with check_kernel=False.)"""
    n, m, keep = 300, 6, 3
    ctx = kk.B200Context(n, 262)
    try:
        lib = ctx.lib
        rng = np.random.default_rng(11)
        slab = ctx.empty_range(258)
        other = ctx.from_host(rng.standard_normal(n), ctx.add_space(n, 2))
        for v in slab:
            v.upload(rng.standard_normal(n))
        everything = slab + [other]
        before = np.stack([v.to_host() for v in everything])
        U = np.asfortranarray(rng.standard_normal((257, 257)))
        Up = U.ctypes.data_as(C.POINTER(C.c_double))
        b = slab[:m]
        cases = [("m = 0", b, 0, 1, m, L.EINVAL), ("keep = 0", b, m, 0, m, L.EINVAL),
                 ("keep > m", b, m, m + 1, m, L.EINVAL), ("ldu < m", b, m, keep, m - 1, L.EINVAL),
                 ("m = 257", slab[:257], 257, 4, 257, L.ENOTSUP),
                 ("two spaces", b[:m - 1] + [other], m, keep, m, L.EDIM),
                 ("first and last repeated", b[:m - 1] + [b[0]], m, keep, m, L.EINVAL),
                 ("repeated inside keep", [b[0], b[1], b[1], b[3], b[4], b[5]], m, keep, m, L.EINVAL),
                 ("repeated outside keep", [b[0], b[1], b[2], b[4], b[4], b[5]], m, keep, m, L.EINVAL),
                 ("output repeated as input", [b[0], b[1], b[2], b[3], b[1], b[5]], m, keep, m, L.EINVAL)]
        for what, cols, mm, kp, ldu, code in cases:
            st = lib.b2k_basis_transform(ctx.h, handles(cols), mm, Up, ldu, kp)
            assert st == code, f"{what}: status {st}, expected {code}"
            after = np.stack([v.to_host() for v in everything])
            assert same_bits(after, before), f"{what}: a column changed"
        # the context still works
        kk.basistransform_(kk.OrthonormalBasis(b), U[:m, :keep])
        if check_kernel:
            assert lib.b2k_debug_transform_kernel() == expected_kernel(f64, m, keep)
        np.testing.assert_allclose(np.stack([v.to_host() for v in b[:keep]]).T, before[:m].T @ U[:m, :keep],
                                   rtol=1e-13, atol=1e-13)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------ end to end -------------

DFMA_VARIANTS = [(0, 1), (1, 1), (2, 1), (3, 1), (5, 1), (7, 1), (6, 0)]
DMMA_VARIANTS = [(4, 1), (6, 1)]


@gpu
def test_lanczos_eigsolve_is_bit_identical_under_every_variant():
    """Float64 Lanczos eigsolve with thick restarts (krylovdim 30: every restart transforms m = 30 columns with
    keep <= 30): f89, the three ur layouts, f89w and k_transform give the same Ritz values, vectors and normres bit
    for bit, and so do the hybrid and DMMA kernels, whose tensor-core sums round like the fma fold; all agree with
    the oracle to 1e-10."""
    nx, ny = 125, 80
    n = nx * ny
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(20260923, n)
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=30, maxiter=300, tol=1e-10, verbosity=0)
    ctx = kk.B200Context(n, 48)
    op = kk.B200CSR.stencil(ctx, nx, ny)
    runs = {}
    try:
        for mode, dm in DFMA_VARIANTS + DMMA_VARIANTS:
            with dispatch(mode, dm) as lib:
                with profiled(ctx) as cnt:
                    vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0), 4, "SR", alg)
                assert info.numiter > 1 and cnt[TRANSFORM] >= info.numiter - 1
                assert lib.b2k_debug_transform_kernel() == expected_kernel(f64, 30, 30, mode, dm)
            runs[(mode, dm)] = (np.array(vals[:4]), np.stack([v.to_host() for v in vecs[:4]]),
                                np.array(info.normres[:4]), info.numiter)
            del vecs, info
    finally:
        ctx.close()
    ovals, _, _ = ko.eigsolve_lanczos(A, x0, 4, "SR", krylovdim=30, maxiter=300, tol=1e-10, orth=ko.Orth(ko.CGS2))
    for key in DMMA_VARIANTS + DFMA_VARIANTS[:1]:
        np.testing.assert_allclose(runs[key][0], ovals[:4], rtol=1e-10)
    ref = runs[DFMA_VARIANTS[0]]
    for key in DFMA_VARIANTS[1:] + DMMA_VARIANTS:
        got = runs[key]
        assert got[3] == ref[3], key
        for a, b in zip(got[:3], ref[:3]):
            assert same_bits(a, b), f"mode {key[0]}, dmma {key[1]}: not bit-identical to f89"
