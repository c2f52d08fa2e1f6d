"""The one-pass dense Golub-Kahan-Lanczos step (b2k_op_apply_normal_gram: y = A x and z = A'(A x) from one pass over
A) against oracle/onepass_restate.py, bit for bit: y, and z = T(dres) with dres the grouped sum of the per-CTA Float64
partials.  test_onepass_emulation.py checks that the restatement equals the kernel source on host threads; here the
device is held to it.

The grid depends on the occupancy, which the test cannot compute, so every case reads the launch back through
b2k_debug_onepass_launch ({variant, NZ, grid, ntiles}) and asserts which instance ran.  Variant A:
grid = min(ntiles, k·#SMs) for an integer k >= 1 (k = 3 at n = 512 Float32, DESIGN §6); variant B: min(ntiles, #SMs).

Shapes.  Variant A at every width where the template instance changes (NZ = 1, 2, 4, 7 at n <= 256, 512, 1024, else)
and at the shared-memory limits (1700 Float32, 846 Float64); each instance meets every kind of row count: one row,
31, 32 and 33 rows, a ragged count with fewer tiles than CTAs, and one where every CTA walks at least three tiles.
Variant B (Float32, n <= 512, 64-row tiles) at ld = 0 and 32 mod 64 (the last tile half outside A), with fewer tiles
than SMs and with several tiles per CTA.  Integer data in [-2, 2] makes every partial exact, so y and z are the
exact products whatever the order: the order-independent check.

(The file sorts after test_gpu_zzz_onepass.py for the reason that file gives.)"""
import ctypes as C

import numpy as np
import pytest

import krylovkit_jl_b200 as kk
from krylovkit_jl_b200 import _lib as L
from krylovkit_jl_b200.operators import apply_normal, apply_normal_gram
from oracle import krylov_oracle as ko
from oracle import onepass_restate as rs

pytestmark = pytest.mark.gpu
f64, f32 = np.float64, np.float32
ONEPASS = 8                      # profile class of the one-pass launch
SEED = 20260923
ROW_KINDS = [1, 31, 32, 33, "few", "many"]
WIDTHS = {f32: {1: [1, 6, 255, 256], 2: [257, 511, 512], 4: [513, 1024], 7: [1025, 1700]},
          f64: {1: [1, 2, 255, 256], 2: [257, 512], 4: [513, 846]}}


def _variant_a_cases():
    """(dtype, n, row kind): within an instance, width i of w takes the kinds i, i + w, ...: every instance meets
    every kind"""
    out = []
    for dt, inst in WIDTHS.items():
        for ws in inst.values():
            for i, n in enumerate(ws):
                out += [(dt, n, k) for k in ROW_KINDS[i::len(ws)]]
    return out


_NSM = []


def num_sms():
    if not _NSM:
        import torch
        _NSM.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _NSM[0]


def smem_ctas(n, dt):
    """at most this many variant-A CTAs per SM: threads (8 x 256) and shared memory (228 KB, 1 KB reserved per CTA)"""
    smem = (34 * n + 288) * np.dtype(dt).itemsize
    return max(1, min(8, (228 * 1024) // (smem + 1024)))


def rows_of(kind, n, dt):
    if kind == "few":                            # ragged, fewer tiles than the SMs (hence than the CTAs)
        return 32 * (num_sms() // 3) + 17
    if kind == "many":                           # at least three tiles per CTA whatever the occupancy
        return 32 * 3 * smem_ctas(n, dt) * num_sms() + 5
    return kind


@pytest.fixture(scope="module")
def fma(tmp_path_factory):
    return rs.load_fma(str(tmp_path_factory.mktemp("vfma")))


@pytest.fixture()
def variant_b():
    lib = L.load()
    assert lib.b2k_debug_set_onepass_variant(1) == 0
    yield
    assert lib.b2k_debug_set_onepass_variant(0) == 0


def launch_info():
    out = (C.c_int32 * 4)()
    assert L.load().b2k_debug_onepass_launch(out) == 0
    return tuple(out)


def instance(variant, n):
    """(variant, NZ) the hook reports: variant B has no NZ"""
    return (variant, rs.nz_of(n) if variant == 0 else 0)


def data(dt, m, n, integer=False, seed=0):
    rng = np.random.default_rng(seed + 7 * m + n)
    if integer:
        return rng.integers(-2, 3, (m, n)).astype(dt), rng.integers(-2, 3, n).astype(dt)
    return (rng.random((m, n)) - 0.5).astype(dt), (rng.random(n) - 0.5).astype(dt)


def bits(a):
    a = np.asarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


class Setup:
    """a context with A uploaded, x, and y / z between sentinel columns"""

    def __init__(self, A, x):
        dt = A.dtype.type
        m, n = A.shape
        self.ctx = ctx = kk.B200Context(m, 6, dtype=dt)
        self.sv = ctx.add_space(n, 6, sharded=False)
        self.op = kk.B200Dense.from_host(ctx, A, self.sv)
        self.x = ctx.from_host(x, space=self.sv)
        self.yl, self.y, self.yh = (ctx.from_host(np.full(m, dt(v)), space=0) for v in (7.0, 1e30, -7.0))
        self.zl, self.z, self.zh = (ctx.from_host(np.full(n, dt(v)), space=self.sv) for v in (5.0, 1e30, -5.0))

    def call(self):
        return self.ctx.lib.b2k_op_apply_normal_gram(self.ctx.h, self.op.h, self.x.handle, self.y.handle,
                                                     self.z.handle)

    def run(self):
        self.ctx.check(self.call())
        return self.y.to_host(), self.z.to_host()


def check_against_restatement(A, x, fma, variant, expect_nz):
    s = Setup(A, x)
    y, z = s.run()
    v, nz, grid, ntiles = launch_info()
    m, n = A.shape
    nsm = num_sms()
    assert (v, nz) == (variant, expect_nz)
    assert ntiles == rs.ntiles_of(m, variant)
    if variant == 0:                             # min(ntiles, k·#SMs), k the occupancy
        assert grid == ntiles or (grid < ntiles and grid % nsm == 0), (grid, ntiles, nsm)
    else:
        assert grid == min(ntiles, nsm)
    ry, _, _, rz = rs.apply_normal_gram(A, x, variant, grid, fma)
    assert np.array_equal(bits(y), bits(ry)), np.flatnonzero(bits(y) != bits(ry))[:8]
    assert np.array_equal(bits(z), bits(rz)), np.flatnonzero(bits(z) != bits(rz))[:8]
    s.ctx.close()
    return grid, ntiles


@pytest.mark.parametrize("dt,n,kind", _variant_a_cases(),
                         ids=lambda v: v.__name__ if isinstance(v, type) else str(v))
def test_variant_a(fma, dt, n, kind):
    m = rows_of(kind, n, dt)
    A, x = data(dt, m, n)
    grid, ntiles = check_against_restatement(A, x, fma, 0, rs.nz_of(n))
    if kind == "few":
        assert grid == ntiles < num_sms()
    if kind == "many":
        assert ntiles >= 3 * grid


@pytest.mark.parametrize("ld_mod", [0, 32])
@pytest.mark.parametrize("tiles", ["few", "many"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 300, 512])
def test_variant_b(fma, variant_b, n, tiles, ld_mod):
    nt = num_sms() // 3 if tiles == "few" else 3 * num_sms() + 5       # whole 64-row tiles
    m = 64 * nt - 3 if ld_mod == 0 else 64 * nt + 20                    # ld = 64 nt, or 64 nt + 32
    assert (rs.ld_of(m) % 64) == ld_mod
    A, x = data(f32, m, n)
    grid, ntiles = check_against_restatement(A, x, fma, 1, 0)
    if tiles == "few":
        assert grid == ntiles < num_sms()
    else:
        assert ntiles >= 3 * grid


def test_variant_b_hands_wider_matrices_to_variant_a(fma, variant_b):
    A, x = data(f32, 1000, 513)
    check_against_restatement(A, x, fma, 0, 4)


def test_grid_at_config4_width_is_three_ctas_per_sm(fma):
    """n = 512 Float32: 71 KB of shared memory per CTA, 3 CTAs per SM (DESIGN §6)"""
    m = 32 * 4 * num_sms() + 1
    A, x = data(f32, m, 512)
    grid, ntiles = check_against_restatement(A, x, fma, 0, 2)
    assert grid == 3 * num_sms() < ntiles


@pytest.mark.parametrize("dt,n,kind,variant", [(f32, 1700, "many", 0), (f32, 257, 33, 0), (f32, 6, "many", 0),
                                               (f64, 846, "few", 0), (f64, 1, "many", 0), (f64, 300, 31, 0),
                                               (f32, 512, "many", 1), (f32, 33, "few", 1)])
def test_small_integers_are_exact(dt, n, kind, variant):
    """entries in [-2, 2]: every partial is exact in T, so y = A x and z = T(A'(A x)) exactly, in any order"""
    m = rows_of(kind, n, dt) if variant == 0 else (64 * (3 * num_sms() + 5) + 20 if kind == "many" else 1310)
    A, x = data(dt, m, n, integer=True)
    lib = L.load()
    assert lib.b2k_debug_set_onepass_variant(variant) == 0
    try:
        s = Setup(A, x)
        y, z = s.run()
        assert launch_info()[:2] == instance(variant, n)
    finally:
        assert lib.b2k_debug_set_onepass_variant(0) == 0
    Ai, xi = A.astype(np.int64), x.astype(np.int64)
    yi = Ai @ xi
    np.testing.assert_array_equal(y, yi.astype(dt))
    np.testing.assert_array_equal(z, (Ai.T @ yi).astype(dt))
    s.ctx.close()


@pytest.mark.parametrize("dt,variant", [(f32, 0), (f64, 0), (f32, 1)], ids=["f32-A", "f64-A", "f32-B"])
def test_side_effects(fma, dt, variant):
    """x untouched, the columns next to y and z keep their sentinels, a second call gives the same bits, one launch
    of class 8 with sizeof(T)·(m·n + m + n) algorithmic bytes"""
    m, n = 3001, 300
    A, x = data(dt, m, n)
    lib = L.load()
    assert lib.b2k_debug_set_onepass_variant(variant) == 0
    try:
        s = Setup(A, x)
        ctx = s.ctx
        ctx.check(ctx.lib.b2k_prof_reset(ctx.h))
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 1))
        y, z = s.run()
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 0))
        cnt, ms, nbytes = C.c_int64(), C.c_double(), C.c_double()
        ctx.check(ctx.lib.b2k_prof_read(ctx.h, ONEPASS, C.byref(cnt), C.byref(ms), C.byref(nbytes)))
        assert launch_info()[:2] == instance(variant, n)
        y2, z2 = s.run()
    finally:
        assert lib.b2k_debug_set_onepass_variant(0) == 0
    assert cnt.value == 1
    assert nbytes.value == np.dtype(dt).itemsize * (m * n + m + n)
    assert np.array_equal(bits(s.x.to_host()), bits(x))
    assert np.array_equal(bits(y2), bits(y)) and np.array_equal(bits(z2), bits(z))
    ry, _, _, rz = rs.apply_normal_gram(A, x, variant, launch_info()[2], fma)
    assert np.array_equal(bits(y), bits(ry)) and np.array_equal(bits(z), bits(rz))
    for v, val in ((s.yl, 7.0), (s.yh, -7.0), (s.zl, 5.0), (s.zh, -5.0)):
        assert np.array_equal(v.to_host(), np.full(len(v), dt(val)))
    ctx.close()


@pytest.mark.parametrize("dt,n,ok", [(f64, 846, True), (f64, 847, False), (f64, 1793, False),
                                     (f32, 1700, True), (f32, 1701, False), (f32, 1792, False), (f32, 1793, False)])
def test_width_limits(fma, dt, n, ok):
    """the 32 x n tile must fit the 227 KB of shared memory a CTA may have: (34 n + 288)·sizeof(T) bytes, so 1700
    Float32 / 846 Float64 columns; more than 7 x 256 = 1792 columns is refused before that.  A refused call leaves
    y and z as they were."""
    m = 40
    A, x = data(dt, m, n)
    s = Setup(A, x)
    before = launch_info()
    rc = s.call()
    if ok:
        assert rc == L.OK
        v, nz, grid, _ = launch_info()
        assert (v, nz) == instance(0, n) == (0, 7 if n > 1024 else 4)
        ry, _, _, rz = rs.apply_normal_gram(A, x, 0, grid, fma)
        assert np.array_equal(bits(s.y.to_host()), bits(ry)) and np.array_equal(bits(s.z.to_host()), bits(rz))
    else:
        assert rc == L.ENOTSUP
        msg = s.ctx.lib.b2k_last_error(s.ctx.h).decode()
        assert ("more than 1792 columns" in msg) == (n > 1792), msg
        assert launch_info() == before
        assert np.array_equal(s.y.to_host(), np.full(m, dt(1e30)))
        assert np.array_equal(s.z.to_host(), np.full(n, dt(1e30)))
    s.ctx.close()


def _columns(ctx, op, sv, n, dt):
    """A column by column as apply_normal(e_j): one nonzero product per fma chain, exact"""
    cols = []
    for j in range(n):
        e = np.zeros(n, dtype=dt)
        e[j] = 1
        cols.append(apply_normal(op, ctx.from_host(e, space=sv)).to_host())
    return np.column_stack(cols)


@pytest.mark.parametrize("dt", [f32, f64], ids=["f32", "f64"])
def test_dense_splitmix_equals_the_oracle(dt):
    m, n = 1001, 37
    ctx = kk.B200Context(m, 8, dtype=dt)
    sv = ctx.add_space(n, 8, sharded=False)
    op = kk.B200Dense.splitmix(ctx, m, n, SEED, sv)
    want = ko.dense_splitmix(SEED, m, n, dtype=dt)
    assert np.array_equal(bits(_columns(ctx, op, sv, n, dt)), bits(np.ascontiguousarray(want)))
    ctx.close()


@pytest.mark.parametrize("dt", [f32, f64], ids=["f32", "f64"])
def test_dense_from_host_with_a_leading_dimension(fma, dt):
    """b2k_op_create_dense with ld > m copies rows [0, m) of every column; the padding rows of the host array (NaN
    here) never reach the device"""
    m, n, ld = 77, 40, 77 + 13
    A, x = data(dt, m, n)
    H = np.full((ld, n), np.nan, dtype=dt, order="F")
    H[:m] = A
    ctx = kk.B200Context(m, 8, dtype=dt)
    sv = ctx.add_space(n, 8, sharded=False)
    h = L.c_op()
    ctx.check(ctx.lib.b2k_op_create_dense(ctx.h, C.byref(h), m, n, H.ctypes.data, ld))
    op = kk.B200Dense(ctx, h)
    op.space_in, op.space_out = sv, 0
    assert np.array_equal(bits(_columns(ctx, op, sv, n, dt)), bits(A))
    y, z = apply_normal_gram(op, ctx.from_host(x, space=sv))
    v, nz, grid, _ = launch_info()
    assert (v, nz) == instance(0, n)
    ry, _, _, rz = rs.apply_normal_gram(A, x, 0, grid, fma)
    assert np.array_equal(bits(y.to_host()), bits(ry)) and np.array_equal(bits(z.to_host()), bits(rz))
    ctx.close()
