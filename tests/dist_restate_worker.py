"""Run under torchrun: the row-sharded SpMV kernels, the rank-ordered sums, the sharded Lanczos step and every other
entry point that sums across ranks (groups g1 ... g9 below) against the composed restatement of tests/dist_restate.py,
bit for bit, on every rank (tests/test_gpu_zz_dist_restate.py).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 3 --master-addr 127.0.0.1 \\
        --master-port 29621 tests/dist_restate_worker.py

B2K_ONE_GPU=1: every rank on GPU 0, the library on its NVLink peer window alone (B2K_NO_NCCL=1) and gloo for this
script's own gathers; otherwise one rank per GPU.  With B2K_PEER=0 the library's transport is NCCL: y and the local
partials stay exact, and the cross-rank sums are NCCL's, pinned for two ranks (two addends give the same bits in either
order) and bounded for more.

Every rank records (label, device value, restated value, kind) in the same order; rank 0 gathers the records and
compares them bit for bit (NaNs by position).  kind "global" (cross-rank sums, the Lanczos scalars) must moreover have
the same bits on every rank.  On success rank 0 prints "dist_restate ok".
"""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys
import tempfile
import time

os.environ.setdefault("OPENBLAS_NUM_THREADS", "8")

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import krylovkit_jl_b200 as kk  # noqa: E402
from krylovkit_jl_b200 import _lib as L  # noqa: E402
from krylovkit_jl_b200 import sharding  # noqa: E402
from krylovkit_jl_b200.factorizations import lanczos as lz  # noqa: E402
from krylovkit_jl_b200.vectors import handles  # noqa: E402

import dist_restate as D  # noqa: E402
import tsk_restate as ts  # noqa: E402
from test_gpu_blas1 import _FMA_C  # noqa: E402
from test_gpu_spmv_fused import CALLERS, FEATURES, fused, kernel, launch, device_tiles, same  # noqa: E402

f64, f32 = np.float64, np.float32
KID = {1: "stream", 2: "pipe", 4: "stencil"}
COEFFS = (4.0, -1.4, -0.6, -1.2, -0.8, -0.3, -0.7)


def load_fma(tmp):
    """fma(a, b, c, T) as the fma fixture of test_gpu_blas1.py builds it"""
    src, so = os.path.join(tmp, "vfma.c"), os.path.join(tmp, "libvfma.so")
    with open(src, "w") as fh:
        fh.write(_FMA_C)
    r = subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src, "-lm"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)

    def f(a, b, c, dt):
        a, b, c = (np.ascontiguousarray(t, dtype=dt) for t in np.broadcast_arrays(
            np.asarray(a, dtype=dt), np.asarray(b, dtype=dt), np.asarray(c, dtype=dt)))
        out = np.empty(a.shape, dtype=dt)
        fn = lib.vfma_f64 if dt == f64 else lib.vfma_f32
        fn(C.c_size_t(out.size), C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), C.c_void_p(c.ctypes.data),
           C.c_void_p(out.ctypes.data))
        return out
    return f


class Job:
    def __init__(self):
        self.rank, self.world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        self.local = int(os.environ["LOCAL_RANK"])
        self.one_gpu = os.environ.get("B2K_ONE_GPU", "") == "1"
        if self.one_gpu:
            os.environ["B2K_NO_NCCL"] = "1"
            self.local = 0
            dist.init_process_group("gloo")
        else:
            torch.cuda.set_device(self.local)
            dist.init_process_group("nccl", device_id=torch.device("cuda", self.local))
        self.nccl = os.environ.get("B2K_PEER", "") == "0"
        self.nsm = torch.cuda.get_device_properties(self.local).multi_processor_count
        self.lib = L.load()
        self.records = []

    def gather(self, obj):
        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    def context(self, sizes, dt, ncols=8):
        off = D.offsets(sizes)
        uid = sharding.broadcast_nccl_uid(dist, self.lib)
        return kk.B200Context(sizes[self.rank], ncols, dtype=dt, device=self.local, rank=self.rank, nranks=self.world,
                              nccl_uid=uid, n_global=int(off[-1]), row_offset=int(off[self.rank]))

    def rec(self, label, got, want, kind="local", parts=None):
        """kind local: this rank's bits; global: a cross-rank sum, the same bits on every rank (bounded by the
        partials `parts` where NCCL adds more than two)"""
        self.records.append((label, np.asarray(got), np.asarray(want), kind,
                             None if parts is None else np.asarray(parts, dtype=f64)))

    def finish(self):
        every = self.gather(self.records)
        if self.rank != 0:
            return
        bad, bounded = [], self.nccl and self.world > 2
        for p, recs in enumerate(every):
            assert len(recs) == len(every[0]), (p, len(recs), len(every[0]))
            for i, (label, got, want, kind, parts) in enumerate(recs):
                if kind == "global" and bounded:
                    tol = self.world * 2.0 ** -53 * np.sum(np.abs(parts), axis=0) + 2.0 ** -52 * np.abs(want)
                    ok = bool(np.all(np.abs(got - want) <= tol))
                else:
                    ok = same(got, want)
                    if kind == "global":
                        ok = ok and same(got, every[0][i][1])
                if not ok:
                    bad.append(f"rank {p}: {label}: got {got.ravel()[:4]} want {want.ravel()[:4]}")
        if bad:
            print("\n".join(bad[:40]))
            raise AssertionError(f"dist_restate: {len(bad)} mismatches on {self.world} ranks")
        n = sum(len(r) for r in every)
        print(f"dist_restate ok on {self.world} ranks{' (NCCL)' if self.nccl else ''}: {n} comparisons")


# ----------------------------------------------------------------------------------------------- operators ----

def unequal(world, base, step):
    return [base + step * ((5 * p) % 7) for p in range(world)]


def band(sizes, lo, hi, seed, empty_rank=None, long_row=0):
    """about 5 random, unsorted columns per row in [r - lo, r + hi]; the rows of empty_rank without nonzeros; with
    long_row, the middle row of every shard has that many columns spread over [r0 - lo, r0 + n + hi)"""
    n = sum(sizes)
    off = D.offsets(sizes)
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 9, n)
    if empty_rank is not None:
        lens[off[empty_rank]:off[empty_rank + 1]] = 0
    mids = [int(off[p] + sizes[p] // 2) for p in range(len(sizes))] if long_row else []
    lens[mids] = long_row
    rowptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    cols = np.clip(np.repeat(np.arange(n), lens) + rng.integers(-lo, hi + 1, rowptr[-1]), 0, n - 1)
    for p, r in enumerate(mids):
        c = np.linspace(max(0, off[p] - lo), min(n - 1, off[p + 1] - 1 + hi), long_row).astype(np.int64)
        cols[rowptr[r]:rowptr[r + 1]] = rng.permutation(c)
    return rowptr, cols, rng.standard_normal(rowptr[-1])


def csr_cases(world):
    """(name, shard sizes, global CSR (float64 values))"""
    out = []
    if world in (2, 3):
        sizes, csr, _, _ = D.fold_case(f64, world)
        out.append(("band57-9", sizes, csr))
    else:
        sizes = unequal(world, 1500, 900)
        out.append(("band57-9", sizes, D.band_csr(sum(sizes), 57, 9, 7)))
    # the lower halo of rank p >= 1 is the whole of rank p - 1's shard
    sizes = [300 * 2 ** p for p in range(world - 1)] + [2500]
    rowptr, cols, vals = D.band_csr(sum(sizes), 5, 5, 11)
    off = D.offsets(sizes)
    for p in range(1, world):
        cols[rowptr[off[p]]] = off[p - 1]
    out.append(("whole-shard-halo", sizes, (rowptr, cols, vals)))
    # rank 1 owns rows without nonzeros; its neighbours read its boundary rows
    sizes = unequal(world, 900, 300)
    out.append(("empty-rank", sizes, band(sizes, 30, 30, 12, empty_rank=1)))
    # a row of 2000 nonzeros per shard with columns in both halos
    sizes = unequal(world, 2500, 300)
    out.append(("long-rows", sizes, band(sizes, 40, 40, 13, long_row=2000)))
    return out


def lines(total, world):
    """unequal shards of whole grid lines (or planes)"""
    w = np.arange(1, world + 1, dtype=f64)
    cut = np.r_[0, np.round(np.cumsum(w) / w.sum() * total)].astype(np.int64)
    return list(np.diff(cut))


def stencil_cases(world):
    out = []
    for dims in ((61, 47, 1), (17, 13, 11)):
        unit, count = (dims[0], dims[1]) if dims[2] == 1 else (dims[0] * dims[1], dims[2])
        if 2 * world <= count:
            out.append((dims, [int(unit * m) for m in lines(count, world)]))
    return out


# ----------------------------------------------------------------------------------------------------- SpMV ----

def spmv_launch(job, fma, op, dt, xg, vg, dg, kname, host, label, feats):
    """one b2k_debug_apply_fused launch with `feats` (test_gpu_spmv_fused's feature sets) on this rank's rows"""
    ctx, r0, n = op.ctx, op.ctx.row_offset, op.ctx.n_local
    sl = slice(r0, r0 + n)
    x, v, ds = ctx.from_host(xg[sl]), ctx.from_host(vg[sl]), ctx.from_host(dg[sl])
    y, vout = ctx.empty(), ctx.empty()
    y0 = np.full(n, 7.5, dtype=dt)
    y.upload(y0)
    vout.upload(y0)
    dot, dsub, shift = feats.get("dot"), feats.get("dsub", False), feats.get("shift", False)
    a0, a1 = (0.3, -1.25) if shift else (0.0, 1.0)
    kw = dict(a0=a0, a1=a1, shifted=shift, xscale=feats.get("xscale"), dot_self=dot == "self",
              dsc=-0.45 if dsub else 0.0)
    with kernel(kname):
        st, d = fused(op, x, y, dotv=v if dot == "dotv" else None, vout=vout if feats.get("vout") else None,
                      dsub=ds if dsub else None, l2=feats.get("l2", False), **kw)
        lr = launch()
    job.rec(label + " status", st, L.OK)
    want_k = 4 if kname == "stencil" else (1 if kname == "stream" else 2)
    job.rec(label + " kernel", lr[0], want_k)
    if kname.startswith("pipe"):
        job.rec(label + " variant", lr[1], 1 if kname == "pipe24" else 0)
    src = dict(stencil=host) if kname == "stencil" else dict(csr=host)
    wy, wv, wd = D.spmv(fma, dt, KID.get(lr[0], "pipe"), lr[2], xg, r0, n, dotv=vg if dot == "dotv" else None,
                        dsub=dg if dsub else None, **src, **kw)
    job.rec(label + " y", y.to_host(), wy)
    job.rec(label + " vout", vout.to_host(), wv if feats.get("vout") else y0)
    if dot is not None:
        job.rec(label + " dot partial", np.float64(d), np.float64(wd))
    for t in (x, v, ds, y, vout):
        t.free()


def apply_dot(job, fma, op, dt, xg, vg, kname, host, label):
    """b2k_op_apply_dot: the fold of every rank's restated partial, on every rank"""
    ctx, r0, n = op.ctx, op.ctx.row_offset, op.ctx.n_local
    sl = slice(r0, r0 + n)
    x, v, y = ctx.from_host(xg[sl]), ctx.from_host(vg[sl]), ctx.empty()
    with kernel(kname):
        got = op.apply_dot_into(y, x, v)
        lr = launch()
    src = dict(stencil=host) if kname == "stencil" else dict(csr=host)
    wy, _, wd = D.spmv(fma, dt, KID.get(lr[0], "pipe"), lr[2], xg, r0, n, dotv=vg, **src)
    parts = job.gather(float(wd))
    job.rec(label + " apply_dot y", y.to_host(), wy)
    job.rec(label + " apply_dot", np.float64(got), D.fold(parts), "global", parts)
    for t in (x, v, y):
        t.free()


def operands(n, dt, seed, sizes):
    rng = np.random.default_rng(seed)
    xg = rng.standard_normal(n).astype(dt)
    xg[rng.integers(0, n, n // 50)] = -0.0
    vg = rng.standard_normal(n)
    off = D.offsets(sizes)
    for p in range(len(sizes)):                  # partials of very different sizes: the fold order shows
        vg[off[p]:off[p + 1]] *= (1.0, 2.0 ** -20, -1.0)[p % 3]
    return xg, vg.astype(dt), rng.standard_normal(n).astype(dt)


def spmv_checks(job, fma):
    lib = job.lib
    for dt in (f64, f32):
        for name, sizes, (rowptr, cols, vals) in csr_cases(job.world):
            ctx = job.context(sizes, dt)
            off = D.offsets(sizes)
            loc = D.local_csr(rowptr, cols, vals.astype(dt), off[job.rank], sizes[job.rank])
            op = kk.B200CSR.from_csr_arrays(ctx, sizes[job.rank], int(off[-1]), loc[0], loc[1], loc[2])
            tag = f"{name} {np.dtype(dt).name}"
            job.rec(tag + " csr format", lib.b2k_debug_csr_format(op.h), 0)
            job.rec(tag + " tiles", device_tiles(op), D.R.tiles(loc[0]))
            if name == "band57-9" and job.world in (2, 3):
                _, _, xg, vg = D.fold_case(dt, job.world)
                dg = np.random.default_rng(5).standard_normal(len(xg)).astype(dt)
            else:
                xg, vg, dg = operands(int(off[-1]), dt, 3, sizes)
            for kname in ("stream", "pipe24", "pipe33"):
                for i, feats in enumerate(FEATURES + CALLERS):
                    spmv_launch(job, fma, op, dt, xg, vg, dg, kname, loc, f"{tag} {kname} f{i}", feats)
                apply_dot(job, fma, op, dt, xg, vg, kname, loc, f"{tag} {kname}")
            del op
            ctx.close()
        for dims, sizes in stencil_cases(job.world):
            ctx = job.context(sizes, dt)
            n = int(np.prod(dims))
            xg, vg, dg = operands(n, dt, 4, sizes)
            off = D.offsets(sizes)
            tag = f"stencil{len([d for d in dims if d > 1])}d {np.dtype(dt).name}"
            asm = kk.B200CSR.stencil(ctx, *dims, coeffs=COEFFS)
            loc = D.local_csr(*D.stencil_csr(*dims, COEFFS, dt), off[job.rank], sizes[job.rank])
            job.rec(tag + " assembled csr format", lib.b2k_debug_csr_format(asm.h), 0)
            job.rec(tag + " assembled tiles", device_tiles(asm), D.R.tiles(loc[0]))
            free = kk.B200CSR.stencil_free(ctx, *dims, coeffs=COEFFS)
            for kname in ("stream", "pipe24", "pipe33"):
                for i, feats in enumerate(FEATURES + CALLERS):
                    spmv_launch(job, fma, asm, dt, xg, vg, dg, kname, loc, f"{tag} assembled {kname} f{i}", feats)
                apply_dot(job, fma, asm, dt, xg, vg, kname, loc, f"{tag} assembled {kname}")
            for i, feats in enumerate(FEATURES + CALLERS):
                spmv_launch(job, fma, free, dt, xg, vg, dg, "stencil", (*dims, COEFFS), f"{tag} free f{i}", feats)
            apply_dot(job, fma, free, dt, xg, vg, "stencil", (*dims, COEFFS), f"{tag} free")
            del asm, free
            ctx.close()
    if job.rank == 0:
        print(f"dist_restate: SpMV checks recorded on {job.world} ranks", flush=True)


def refusal_check(job):
    """an operator that couples non-adjacent shards: without NCCL every rank refuses it, from the all-gathered halo
    plan, before any kernel runs"""
    if job.world < 3 or not job.one_gpu:
        return
    sizes = unequal(job.world, 1000, 200)
    rowptr, cols, vals = D.band_csr(sum(sizes), 5, 5, 21)
    off = D.offsets(sizes)
    cols[rowptr[off[2]]] = 0                             # rank 2 reads rank 0
    ctx = job.context(sizes, f64)
    loc = D.local_csr(rowptr, cols, vals, off[job.rank], sizes[job.rank])
    h = L.c_op()
    st = job.lib.b2k_op_create_csr(ctx.h, C.byref(h), sizes[job.rank], int(off[-1]), len(loc[2]),
                                   loc[0].ctypes.data, loc[1].ctypes.data, loc[2].ctypes.data, 8, 0)
    job.rec("non-adjacent refusal", st, L.ENOTSUP)
    x = ctx.from_host(np.ones(sizes[job.rank]))
    job.rec("context usable after the refusal", np.float64(x.inner(x)), np.float64(sum(sizes)), "global",
            [[float(m)] for m in sizes])
    x.free()
    ctx.close()


# ----------------------------------------------------------------------------------------------------- BLAS-1 ----

def blas1_checks(job):
    for dt in (f64, f32):
        if job.world in (2, 3):
            sizes, _, xg, vg = D.fold_case(dt, job.world)
        else:
            sizes = unequal(job.world, 1500, 900)
            xg, vg, _ = operands(sum(sizes), dt, 6, sizes)
        off = D.offsets(sizes)
        sl = slice(off[job.rank], off[job.rank + 1])
        rng = np.random.default_rng(7)
        ig, jg = rng.integers(-8, 9, sum(sizes)).astype(dt), rng.integers(-8, 9, sum(sizes)).astype(dt)
        one = kk.B200Context(sizes[job.rank], 4, dtype=dt, device=job.local)      # this rank's partials
        a, b = one.from_host(xg[sl]), one.from_host(vg[sl])
        p_in, p_nn = a.inner(b), a.inner(a)
        del a, b
        one.close()
        pin, pnn = job.gather(p_in), job.gather(p_nn)
        ctx = job.context(sizes, dt)
        x, v, i, j = (ctx.from_host(t[sl]) for t in (xg, vg, ig, jg))
        tag = np.dtype(dt).name
        job.rec(f"{tag} inner", np.float64(x.inner(v)), D.fold(pin), "global", pin)
        job.rec(f"{tag} norm", np.float64(x.norm()), np.sqrt(D.fold(pnn)), "global", pnn)
        exact = float(ig.astype(f64) @ jg.astype(f64))
        job.rec(f"{tag} inner on integers", np.float64(i.inner(j)), np.float64(exact), "global", [[exact]])
        nn = float(ig.astype(f64) @ ig.astype(f64))
        job.rec(f"{tag} norm on integers", np.float64(i.norm()), np.sqrt(nn), "global", [[nn]])
        del x, v, i, j
        ctx.close()


# ---------------------------------------------------------------------------------------------------- Lanczos ----

def lanczos_checks(job, fma):
    lib = job.lib
    name, sizes, (rowptr, cols, vals) = csr_cases(job.world)[0]
    off = D.offsets(sizes)
    n = int(off[-1])
    sl = slice(off[job.rank], off[job.rank + 1])
    for dt, K1 in ((f64, 9), (f32, 17)):
        k = K1 - 1
        tag = f"lanczos {np.dtype(dt).name}"
        ctx = job.context(sizes, dt, ncols=40)
        loc = D.local_csr(rowptr, cols, vals.astype(dt), off[job.rank], sizes[job.rank])
        op = kk.B200CSR.from_csr_arrays(ctx, sizes[job.rank], n, loc[0], loc[1], loc[2])
        rng = np.random.default_rng([K1, 17])
        V = (rng.standard_normal((n, k)) / math.sqrt(n)).astype(dt)
        r = rng.standard_normal(n)
        rh = (1.7 * r / np.linalg.norm(r)).astype(dt)
        vecs = ctx.empty_range(k + 1)
        for j in range(k):
            vecs[j].upload(V[sl, j])
        vecs[k].upload(rh[sl])
        w = ctx.empty()
        a, b = C.c_double(), C.c_double()
        ctx.check(lib.b2k_lanczos_expand(ctx.h, op.h, handles(vecs), k, vecs[k].handle, w.handle, 1.7, L.CGS2, 0.0,
                                         C.byref(a), C.byref(b)))
        lr = launch()
        grids = job.gather(int(lr[2]))
        job.rec(tag + " SpMV kernel", lr[0], 2)
        if not (job.nccl and job.world > 2):            # NCCL adds the K1 coefficients in its own order
            ws, vg, a0, alpha, beta, n2 = D.lanczos_step(fma, dt, sizes, V, rh, 1.7, (rowptr, cols, vals.astype(dt)),
                                                         "pipe", grids, job.nsm)
            job.rec(tag + " v", vecs[k].to_host(), vg[sl])
            job.rec(tag + " w", w.to_host(), ws[job.rank])
            job.rec(tag + " alpha", np.float64(a.value), np.float64(alpha), "global", [[alpha]])
            job.rec(tag + " beta", np.float64(b.value), np.float64(beta), "global", [[beta]])
        del w, vecs
        # a chained batch equals stepping, on every rank
        x0 = np.random.default_rng(19).standard_normal(n).astype(dt)
        runs = {}
        for chain in (1, 0):
            lib.b2k_debug_set_chain(chain)
            try:
                it = lz.LanczosIterator(op, ctx.from_host(x0[sl]), kk.cgs2)
                f = lz.initialize(it)
                done = lz.expand_many_(it, f, 20, 0.0)
                runs[chain] = (done, np.array(f.alphas), np.array(f.betas),
                               np.column_stack([q.to_host() for q in f.V]), f.r.to_host())
                del f, it
            finally:
                lib.b2k_debug_set_chain(1)
        job.rec(tag + " chained steps", runs[1][0], 20)
        for i, what in ((1, "alphas"), (2, "betas")):
            job.rec(f"{tag} chained {what}", runs[1][i], runs[0][i], "global", np.abs(runs[0][i])[None])
        job.rec(tag + " chained V", runs[1][3], runs[0][3])
        job.rec(tag + " chained r", runs[1][4], runs[0][4])
        del op
        ctx.close()


# ------------------------------------------------------------------------------ the other sharded entry points ----
#
# Groups g1 ... g9 (the labels carry them): g1 b2k_basis_project / unproject, g2 b2k_basis_orthogonalize, g3
# b2k_vec_orthogonalize, g4 b2k_lanczos_expand, g5 the chained MGS2B batch, g6 the CG and BiCGStab steps, g7 the block
# path, g8 the dense adjoint, g9 a replicated space.  The shards are fold_case's, with the last one or two ragged
# (n_p % 256 != 0 and n_p % 4 != 0: a partial last row tile, and a Float32 tail for CTA 0 of that rank), and the
# vectors whose sums cross ranks are scaled by 1, 2^-20 and -1 on consecutive shards.

ETA = 1.0 / math.sqrt(2.0)
SCALES = (1.0, 2.0 ** -20, -1.0)
TINY = {f64: 1e-9, f32: 1e-4}          # well above the rounding of T: IR runs a second pass


def ragged(world):
    if world == 3:
        return [2100, 1303, 2597]
    if world == 2:
        return [3403, 2597]
    return [m + 3 for m in unequal(world, 1500, 900)]


def scaled(sizes, a):
    a = np.array(a, dtype=f64)
    off = D.offsets(sizes)
    for p in range(len(sizes)):
        a[off[p]:off[p + 1]] *= SCALES[p % 3]
    return a


def pd(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def upload(ctx, M, space=0):
    vecs = ctx.empty_range(M.shape[1], space)
    for j, v in enumerate(vecs):
        v.upload(np.ascontiguousarray(M[:, j]))
    return vecs


def exact(job):
    """NCCL adds more than two addends in its own order: the restated compositions hold on the peer window and on
    two ranks"""
    return not (job.nccl and job.world > 2)


def project_checks(job, fma):
    """g1: the fold of the ranks' colsums at k = 8, kcap + 1 (two passes) and 1024 / 1025 (one peer slot, then two
    pieces of the all-reduce); unproject is rank-local"""
    lib = job.lib
    for dt in (f64, f32):
        sizes = ragged(job.world)
        off = D.offsets(sizes)
        sl = slice(off[job.rank], off[job.rank + 1])
        kcap = ts.cfg(dt)[3]
        ks = (8, kcap + 1, 1024, 1025)
        tag = f"g1 {np.dtype(dt).name}"
        ctx = job.context(sizes, dt, ncols=max(ks) + 2)
        rng = np.random.default_rng([31, int(dt == f64)])
        Q = rng.standard_normal((sum(sizes), max(ks))).astype(dt)
        x = scaled(sizes, rng.standard_normal(sum(sizes))).astype(dt)
        vecs = upload(ctx, Q[sl])
        xv, yv = ctx.from_host(x[sl]), ctx.empty()
        for k in ks:
            h = np.zeros(k)
            ctx.check(lib.b2k_basis_project(ctx.h, handles(vecs[:k]), k, xv.handle, 1.0, 0.0, pd(h)))
            parts = job.gather(ts.project(Q[sl, :k], x[sl], job.nsm, fma))
            job.rec(f"{tag} project k={k}", h, D.fold(parts), "global", parts)
        y0 = rng.standard_normal(sum(sizes)).astype(dt)[sl]
        for k in (8, kcap + 1):
            c = rng.standard_normal(k)
            yv.upload(y0)
            ctx.check(lib.b2k_basis_unproject(ctx.h, yv.handle, handles(vecs[:k]), k, pd(c), -0.75, 0.5))
            want = ts.update(Q[sl, :k], y0, ts.coefs(c, -0.75, dt), fma, beta_mode=2, beta=0.5)
            job.rec(f"{tag} unproject k={k}", yv.to_host(), want)
        del vecs, xv, yv
        ctx.close()


def orth_checks(job, fma):
    """g2 b2k_basis_orthogonalize with all seven orthogonalizers (CGSIR / MGSIR also on a vector nearly in span(Q), so
    that they run two passes or more), a classical one past kcap; g3 b2k_vec_orthogonalize with every orthogonalizer"""
    lib = job.lib
    for dt in (f64, f32):
        sizes = ragged(job.world)
        n = sum(sizes)
        off = D.offsets(sizes)
        sl = slice(off[job.rank], off[job.rank + 1])
        kcap = ts.cfg(dt)[3]
        tag = np.dtype(dt).name
        ctx = job.context(sizes, dt, ncols=kcap + 4)
        rng = np.random.default_rng([37, int(dt == f64)])
        Q = np.linalg.qr(rng.standard_normal((n, kcap + 1)))[0].astype(dt)
        v0 = scaled(sizes, rng.standard_normal(n)).astype(dt)
        near = (Q[:, :8] @ rng.standard_normal(8) + TINY[dt] * rng.standard_normal(n)).astype(dt)
        vecs = upload(ctx, Q[sl])
        v = ctx.empty()
        cases = [(alg, 8, v0, 0.0, "") for alg in range(7)]
        cases += [(L.CGSIR, 8, near, ETA, " near span"), (L.MGSIR, 8, near, ETA, " near span"),
                  (L.CGS, kcap + 1, v0, 0.0, ""), (L.CGS2, kcap + 1, v0, 0.0, "")]
        for alg, k, vg, eta, what in cases:
            label = f"g2 {tag} orthogonalize alg={alg} k={k}{what}"
            v.upload(vg[sl])
            h, nrm, passes = np.zeros(k), C.c_double(), C.c_int32()
            ctx.check(lib.b2k_basis_orthogonalize(ctx.h, v.handle, handles(vecs[:k]), k, pd(h), alg, eta,
                                                  C.byref(nrm), C.byref(passes)))
            wh, wn, wp, wv = D.orthogonalize(fma, sizes, Q[:, :k], vg, alg, eta, job.nsm)
            job.rec(label + " h", h, wh, "global", np.abs(wh)[None])
            job.rec(label + " norm", np.float64(nrm.value), np.float64(wn), "global", [[wn]])
            job.rec(label + " passes", np.int32(passes.value), np.int32(wp), "global", [[wp]])
            job.rec(label + " v", v.to_host(), wv[sl])
            if what:
                job.rec(label + " runs two passes or more", wp >= 2, True)
        qg = rng.standard_normal(n)
        qg = (qg / np.linalg.norm(qg)).astype(dt)
        q = ctx.from_host(qg[sl])
        near = (3.0 * qg + TINY[dt] * rng.standard_normal(n)).astype(dt)
        cases = [(alg, v0, 0.0, "") for alg in range(7)] + [(L.CGSIR, near, ETA, " near q"),
                                                              (L.MGSIR, near, ETA, " near q")]
        for alg, vg, eta, what in cases:
            label = f"g3 {tag} vec_orthogonalize alg={alg}{what}"
            v.upload(vg[sl])
            s, nrm = C.c_double(), C.c_double()
            ctx.check(lib.b2k_vec_orthogonalize(ctx.h, v.handle, q.handle, alg, eta, C.byref(s), C.byref(nrm)))
            ws, wn, wv, wp = D.vec_orthogonalize(fma, sizes, qg, vg, alg, eta, job.nsm)
            job.rec(label + " s", np.float64(s.value), np.float64(ws), "global", [[ws]])
            job.rec(label + " norm", np.float64(nrm.value), np.float64(wn), "global", [[wn]])
            job.rec(label + " v", v.to_host(), wv[sl])
            if what:
                job.rec(label + " runs two passes or more", wp >= 2, True)
        del vecs, v, q
        ctx.close()


def expand_checks(job, fma):
    """g4 b2k_lanczos_expand with CGS, CGSIR, MGS, MGS2, MGSIR and MGS2B (the IR variants at eta = 0.95, where this
    step reorthogonalises); g5 the chained MGS2B batch equals stepping, on every rank"""
    lib = job.lib
    _, sizes, (rowptr, cols, vals) = csr_cases(job.world)[0]
    if job.world in (2, 3):
        sizes = ragged(job.world)
    off = D.offsets(sizes)
    n = int(off[-1])
    sl = slice(off[job.rank], off[job.rank + 1])
    K1 = 9
    k = K1 - 1
    for dt in (f64, f32):
        tag = np.dtype(dt).name
        ctx = job.context(sizes, dt, ncols=40)
        csr = (rowptr, cols, vals.astype(dt))
        loc = D.local_csr(*csr, off[job.rank], sizes[job.rank])
        op = kk.B200CSR.from_csr_arrays(ctx, sizes[job.rank], n, loc[0], loc[1], loc[2])
        rng = np.random.default_rng([K1, 23])
        V = (rng.standard_normal((n, k)) / math.sqrt(n)).astype(dt)
        rh = scaled(sizes, rng.standard_normal(n))
        rh = (1.7 * rh / np.linalg.norm(rh)).astype(dt)
        for alg in (L.CGS, L.CGSIR, L.MGS, L.MGS2, L.MGSIR, L.MGS2B):
            eta = 0.95 if alg in (L.CGSIR, L.MGSIR) else 0.0
            label = f"g4 {tag} lanczos_expand alg={alg}"
            vecs = ctx.empty_range(k + 1)
            for j in range(k):
                vecs[j].upload(V[sl, j])
            vecs[k].upload(rh[sl])
            w = ctx.empty()
            a, b = C.c_double(), C.c_double()
            ctx.check(lib.b2k_lanczos_expand(ctx.h, op.h, handles(vecs), k, vecs[k].handle, w.handle, 1.7, alg, eta,
                                             C.byref(a), C.byref(b)))
            lr = launch()
            grids = job.gather(int(lr[2]))
            ww, vg, alpha, beta, passes = D.lanczos_expand(fma, dt, sizes, V, rh, 1.7, csr, KID.get(lr[0], "pipe"),
                                                           grids, job.nsm, alg, eta)
            if eta:
                job.rec(label + " reorthogonalises", passes >= 2, True)
            job.rec(label + " v", vecs[k].to_host(), vg[sl])
            job.rec(label + " w", w.to_host(), ww[sl])
            job.rec(label + " alpha", np.float64(a.value), np.float64(alpha), "global", [[alpha]])
            job.rec(label + " beta", np.float64(b.value), np.float64(beta), "global", [[beta]])
            del vecs, w
        x0 = np.random.default_rng(29).standard_normal(n).astype(dt)
        runs = {}
        for chain in (1, 0):
            lib.b2k_debug_set_chain(chain)
            try:
                it = lz.LanczosIterator(op, ctx.from_host(x0[sl]), kk.mgs2b)
                f = lz.initialize(it)
                done = lz.expand_many_(it, f, 20, 0.0)
                runs[chain] = (done, np.array(f.alphas), np.array(f.betas),
                               np.column_stack([q.to_host() for q in f.V]), f.r.to_host())
                del f, it
            finally:
                lib.b2k_debug_set_chain(1)
        job.rec(f"g5 {tag} mgs2b chained steps", runs[1][0], 20)
        for i, what in ((1, "alphas"), (2, "betas")):
            job.rec(f"g5 {tag} mgs2b chained {what}", runs[1][i], runs[0][i], "global", np.abs(runs[0][i])[None])
        job.rec(f"g5 {tag} mgs2b chained V", runs[1][3], runs[0][3])
        job.rec(f"g5 {tag} mgs2b chained r", runs[1][4], runs[0][4])
        del op
        ctx.close()


def solver_step_checks(job, fma):
    """g6 b2k_cg_step (beta = 0 and not; a shifted and an unshifted operator) and b2k_bicgstab_half (first = 1, 0)
    followed by b2k_bicgstab_full: the local vectors, and the dots and norms as global records"""
    lib = job.lib
    _, sizes, (rowptr, cols, vals) = csr_cases(job.world)[0]
    if job.world in (2, 3):
        sizes = ragged(job.world)
    off = D.offsets(sizes)
    n = int(off[-1])
    sl = slice(off[job.rank], off[job.rank + 1])
    for dt in (f64, f32):
        tag = np.dtype(dt).name
        ctx = job.context(sizes, dt, ncols=16)
        csr = (rowptr, cols, vals.astype(dt))
        loc = D.local_csr(*csr, off[job.rank], sizes[job.rank])
        op = kk.B200CSR.from_csr_arrays(ctx, sizes[job.rank], n, loc[0], loc[1], loc[2])
        rng = np.random.default_rng([41, int(dt == f64)])

        def rnd():
            return scaled(sizes, rng.standard_normal(n)).astype(dt)

        def spmv_of():
            lr = launch()
            return KID.get(lr[0], "pipe"), job.gather(int(lr[2]))

        for a0, a1 in ((0.0, 1.0), (0.3, 1.5)):
            for beta in (0.0, 0.6):
                label = f"g6 {tag} cg_step a0={a0} beta={beta}"
                xh, rh, ph = rnd(), rnd(), rnd()
                x, r, p, q = (ctx.from_host(t[sl]) for t in (xh, rh, ph, np.zeros(n, dt)))
                pq, nr = C.c_double(), C.c_double()
                ctx.check(lib.b2k_cg_step(ctx.h, op.h, x.handle, r.handle, p.handle, q.handle, a0, a1, beta, 1.3,
                                          C.byref(pq), C.byref(nr)))
                kname, grids = spmv_of()
                xn, rn, pn, qn, wpq, wnr, dpq, drr = D.cg_step(fma, dt, sizes, xh, rh, ph, csr, kname, grids, job.nsm,
                                                               a0, a1, beta, 1.3)
                for name, got, want in (("p", p, pn), ("q", q, qn), ("x", x, xn), ("r", r, rn)):
                    job.rec(f"{label} {name}", got.to_host(), want[sl])
                job.rec(label + " <p,q>", np.float64(pq.value), np.float64(wpq), "global", dpq)
                job.rec(label + " ||r||", np.float64(nr.value), np.float64(wnr), "global", drr)
                del x, r, p, q
            for first in (1, 0):
                label = f"g6 {tag} bicgstab a0={a0} first={first}"
                rsh, rh, ph, vh, xh = rnd(), rnd(), rnd(), rnd(), rnd()
                rs, r, p, v, s, x, t = (ctx.from_host(a[sl]) for a in (rsh, rh, ph, vh, np.zeros(n, dt), xh,
                                                                         np.zeros(n, dt)))
                sg, ns = C.c_double(), C.c_double()
                ctx.check(lib.b2k_bicgstab_half(ctx.h, op.h, rs.handle, r.handle, p.handle, v.handle, s.handle, a0, a1,
                                                0.9, 0.45, 1.1, first, C.byref(sg), C.byref(ns)))
                kname, grids = spmv_of()
                pn, vn, sn, wsg, wns, dsg, dss = D.bicgstab_half(fma, dt, sizes, rsh, rh, ph, vh, csr, kname, grids,
                                                                 job.nsm, a0, a1, 0.9, 0.45, 1.1, first)
                for name, got, want in (("p", p, pn), ("v", v, vn), ("s", s, sn)):
                    job.rec(f"{label} half {name}", got.to_host(), want[sl])
                job.rec(label + " half sigma", np.float64(sg.value), np.float64(wsg), "global", dsg)
                job.rec(label + " half ||s||", np.float64(ns.value), np.float64(wns), "global", dss)
                alpha = 1.1 / wsg
                om, nr, rho = C.c_double(), C.c_double(), C.c_double()
                ctx.check(lib.b2k_bicgstab_full(ctx.h, op.h, x.handle, r.handle, rs.handle, p.handle, s.handle,
                                                t.handle, a0, a1, alpha, C.byref(om), C.byref(nr), C.byref(rho)))
                kname, grids = spmv_of()
                xn, rn, tn, wom, wnr, wrho, parts = D.bicgstab_full(fma, dt, sizes, xh, rsh, pn, sn, csr, kname, grids,
                                                                    job.nsm, a0, a1, alpha)
                for name, got, want in (("t", t, tn), ("x", x, xn), ("r", r, rn)):
                    job.rec(f"{label} full {name}", got.to_host(), want[sl])
                job.rec(label + " full omega", np.float64(om.value), np.float64(wom), "global", [[wom]])
                job.rec(label + " full ||r||", np.float64(nr.value), np.float64(wnr), "global", parts[2])
                job.rec(label + " full rho", np.float64(rho.value), np.float64(wrho), "global", parts[3])
                del rs, r, p, v, s, x, t
        del op
        ctx.close()


class Block:
    """the block entry points on a context's vectors (column-major host matrices)"""

    def __init__(self, ctx):
        self.ctx, self.lib = ctx, ctx.lib

    def inner(self, X, Y):
        M = np.zeros(len(X) * len(Y))
        self.ctx.check(self.lib.b2k_block_inner(self.ctx.h, handles(X), len(X), handles(Y), len(Y), pd(M)))
        return M

    def axpy(self, Y, X, M):
        M = np.ascontiguousarray(M, dtype=f64)
        self.ctx.check(self.lib.b2k_block_axpy(self.ctx.h, handles(Y), len(Y), handles(X), len(X), pd(M), len(X)))

    def orthogonalize(self, Rb, V, passes):
        k, p = len(V), len(Rb)
        H, G = np.zeros(max(1, k * p)), np.zeros(p * p)
        self.ctx.check(self.lib.b2k_block_orthogonalize(self.ctx.h, handles(Rb), p, handles(V) if k else None, k,
                                                        passes, pd(H), pd(G)))
        return H[:k * p], G

    def gram(self, Rb):
        return self.orthogonalize(Rb, [], 1)[1]

    def cholqr(self, X, G0=None):
        R, ok = np.zeros(len(X) ** 2), C.c_int32()
        self.ctx.check(self.lib.b2k_block_cholqr(self.ctx.h, handles(X), len(X), 1e-12,
                                                 None if G0 is None else pd(G0), pd(R), C.byref(ok)))
        return R, ok.value


def block_checks(job, composed=True):
    """g7: rank p's partial is the same entry point on a one-rank context over the rank's slices (the same local
    length, so the same grid); block_inner at p q > 1024 (two pieces of the all-reduce), block_axpy, block_orthogonalize
    passes 1 / 2 fused (p <= 4, k <= 48) and unfused (p > 4, k > 48), k = 0 with the Gram matrix, and block_cholqr.
    composed = False (NCCL beyond two ranks, which adds in its own order): block_inner (bounded), block_axpy with the
    same host coefficients and the k = 0 Gram matrix (bounded) only"""
    for dt in (f64, f32):
        tag = f"g7 {np.dtype(dt).name}"
        sizes = ragged(job.world)
        n = sum(sizes)
        off = D.offsets(sizes)
        sl = slice(off[job.rank], off[job.rank + 1])
        rng = np.random.default_rng([43, int(dt == f64)])
        ctx = job.context(sizes, dt, ncols=160)
        one = kk.B200Context(sizes[job.rank], 160, dtype=dt, device=job.local)
        B, B1 = Block(ctx), Block(one)
        # block_inner / block_axpy: 130 x 8
        Xg = rng.standard_normal((n, 130)).astype(dt)
        Yg = np.column_stack([scaled(sizes, rng.standard_normal(n)) for _ in range(8)]).astype(dt)
        X, Y, X1, Y1 = upload(ctx, Xg[sl]), upload(ctx, Yg[sl]), upload(one, Xg[sl]), upload(one, Yg[sl])
        parts = job.gather(B1.inner(X1, Y1))
        M = D.fold(parts)
        job.rec(f"{tag} block_inner 130x8", B.inner(X, Y), M, "global", parts)
        B.axpy(Y, X, M)
        B1.axpy(Y1, X1, M)
        job.rec(f"{tag} block_axpy 130x8", np.column_stack([y.to_host() for y in Y]),
                np.column_stack([y.to_host() for y in Y1]))
        del X, Y, X1, Y1
        # block_orthogonalize
        for p, k, passes in () if not composed else ((3, 20, 1), (3, 20, 2), (4, 48, 2), (6, 20, 2), (3, 60, 2)):
            label = f"{tag} block_orthogonalize p={p} k={k} passes={passes}"
            Vg = np.linalg.qr(rng.standard_normal((n, k)))[0].astype(dt)
            Rg = np.column_stack([scaled(sizes, rng.standard_normal(n)) for _ in range(p)]).astype(dt)
            # the composition on one GPU: project (block_inner), update (block_axpy), Gram (k = 0)
            V1, R1 = upload(one, Vg[sl]), upload(one, Rg[sl])
            H1, G1 = B1.orthogonalize(R1, V1, passes)
            got1 = np.column_stack([c.to_host() for c in R1])
            for c, j in zip(R1, range(p)):
                c.upload(Rg[sl, j])
            Hs = []
            for _ in range(passes):
                Hs.append(B1.inner(V1, R1))
                B1.axpy(R1, V1, Hs[-1])
            job.rec(label + " one-GPU H", H1, Hs[0] + (Hs[1] if passes == 2 else 0.0))
            job.rec(label + " one-GPU R", got1, np.column_stack([c.to_host() for c in R1]))
            job.rec(label + " one-GPU G", G1, B1.gram(R1))
            # the sharded call against the fold of the one-rank partials
            V, Rb = upload(ctx, Vg[sl]), upload(ctx, Rg[sl])
            H, G = B.orthogonalize(Rb, V, passes)
            for c, j in zip(R1, range(p)):
                c.upload(Rg[sl, j])
            Hw = []
            for _ in range(passes):
                parts = job.gather(B1.inner(V1, R1))
                Hw.append(D.fold(parts))
                B1.axpy(R1, V1, Hw[-1])
            gparts = job.gather(B1.gram(R1))
            job.rec(label + " H", H, Hw[0] + (Hw[1] if passes == 2 else 0.0), "global", np.abs(H)[None])
            job.rec(label + " R", np.column_stack([c.to_host() for c in Rb]),
                    np.column_stack([c.to_host() for c in R1]))
            job.rec(label + " G", G, D.fold(gparts), "global", gparts)
            del V1, R1, V, Rb
        # k = 0: the Gram matrix alone; block_cholqr starts from the same fold
        Xg = np.column_stack([scaled(sizes, rng.standard_normal(n)) for _ in range(4)]).astype(dt)
        X, X1 = upload(ctx, Xg[sl]), upload(one, Xg[sl])
        gparts = job.gather(B1.gram(X1))
        G0 = D.fold(gparts)
        job.rec(f"{tag} block_orthogonalize k=0 G", B.gram(X), G0, "global", gparts)
        if not composed:
            del X, X1
            one.close()
            ctx.close()
            continue
        Ra, oka = B.cholqr(X)
        Xa = np.column_stack([c.to_host() for c in X])
        for c, j in zip(X, range(4)):
            c.upload(Xg[sl, j])
        Rb_, okb = B.cholqr(X, G0)
        job.rec(f"{tag} block_cholqr ok", np.int32(oka), np.int32(1), "global", [[1]])
        job.rec(f"{tag} block_cholqr R from the folded Gram", Ra, Rb_, "global", np.abs(Rb_)[None])
        job.rec(f"{tag} block_cholqr ok from the folded Gram", np.int32(okb), np.int32(1), "global", [[1]])
        job.rec(f"{tag} block_cholqr X", Xa, np.column_stack([c.to_host() for c in X]))
        del X, X1
        one.close()
        ctx.close()


def dense_adjoint_checks(job, fma):
    """g8: y = A' x of a row-sharded dense A is T(fold of the ranks' project colsums), the same on every rank (n = 40:
    one pass; kcap + 5: two)"""
    for dt in (f64, f32):
        tag = f"g8 {np.dtype(dt).name}"
        sizes = ragged(job.world)
        m = sum(sizes)
        off = D.offsets(sizes)
        sl = slice(off[job.rank], off[job.rank + 1])
        rng = np.random.default_rng([47, int(dt == f64)])
        ctx = job.context(sizes, dt, ncols=4)
        x = scaled(sizes, rng.standard_normal(m)).astype(dt)
        xv = ctx.from_host(x[sl])
        for ncol in (40, ts.cfg(dt)[3] + 5):
            A = rng.standard_normal((m, ncol)).astype(dt)
            sv = ctx.add_space(ncol, 2, sharded=False)
            op = kk.B200Dense.from_host(ctx, A[sl], sv)
            y = ctx.empty(sv)
            op.apply_adjoint_into(y, xv)
            parts = job.gather(ts.project(A[sl], x[sl], job.nsm, fma))
            job.rec(f"{tag} dense adjoint n={ncol}", y.to_host(), D.fold(parts).astype(dt), "global", parts)
            del op, y
        del xv
        ctx.close()


def replicated_checks(job, fma):
    """g9: a space created with sharded = 0 on the multi-rank context holds the same full vectors on every rank and
    is summed on none: orthogonalize (CGS2: the fused sweep, MGS) and project give the one-rank restatement"""
    lib = job.lib
    for dt in (f64, f32):
        tag = f"g9 {np.dtype(dt).name}"
        sizes = ragged(job.world)
        nrep = 3001
        rng = np.random.default_rng([53, int(dt == f64)])
        ctx = job.context(sizes, dt, ncols=4)
        sv = ctx.add_space(nrep, 12, sharded=False)
        Q = np.linalg.qr(rng.standard_normal((nrep, 8)))[0].astype(dt)
        vg = rng.standard_normal(nrep).astype(dt)
        vecs = upload(ctx, Q, sv)
        v = ctx.empty(sv)
        v.upload(vg)
        h = np.zeros(8)
        ctx.check(lib.b2k_basis_project(ctx.h, handles(vecs), 8, v.handle, 1.0, 0.0, pd(h)))
        want = D.project(fma, [nrep], Q, vg, job.nsm)
        job.rec(f"{tag} replicated project", h, want, "global", np.abs(want)[None])
        for alg in (L.CGS2, L.MGS):
            v.upload(vg)
            h, nrm, passes = np.zeros(8), C.c_double(), C.c_int32()
            ctx.check(lib.b2k_basis_orthogonalize(ctx.h, v.handle, handles(vecs), 8, pd(h), alg, 0.0, C.byref(nrm),
                                                  C.byref(passes)))
            wh, wn, _, wv = D.orthogonalize(fma, [nrep], Q, vg, alg, 0.0, job.nsm)
            job.rec(f"{tag} replicated orthogonalize alg={alg} h", h, wh, "global", np.abs(wh)[None])
            job.rec(f"{tag} replicated orthogonalize alg={alg} norm", np.float64(nrm.value), np.float64(wn), "global",
                    [[wn]])
            job.rec(f"{tag} replicated orthogonalize alg={alg} v", v.to_host(), wv, "global", np.abs(wv)[None])
        del vecs, v
        ctx.close()


def section(job, name, fn, *args):
    t0 = time.perf_counter()
    fn(job, *args)
    if job.rank == 0:
        print(f"dist_restate: {name} recorded on {job.world} ranks in {time.perf_counter() - t0:.1f} s", flush=True)


def main():
    t0 = time.perf_counter()
    job = Job()
    tmp = tempfile.mkdtemp(prefix="dist_restate_fma_")
    try:
        fma = load_fma(tmp)
        refusal_check(job)
        blas1_checks(job)
        lanczos_checks(job, fma)
        spmv_checks(job, fma)
        # every group runs on every transport; where NCCL adds more than two ranks' partials in its own order, the
        # groups whose later values depend on those bits (g2 - g6, the composed block orthogonalization) are left out
        # and the global records of the others are bounded
        section(job, "g1 project", project_checks, fma)
        if exact(job):
            section(job, "g2 g3 orthogonalize", orth_checks, fma)
            section(job, "g4 g5 lanczos_expand", expand_checks, fma)
            section(job, "g6 CG / BiCGStab steps", solver_step_checks, fma)
        section(job, "g8 dense adjoint", dense_adjoint_checks, fma)
        section(job, "g9 replicated space", replicated_checks, fma)
        section(job, "g7 block path", block_checks, exact(job))
        job.finish()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    dist.barrier()
    dist.destroy_process_group()
    if job.rank == 0:
        print(f"dist_restate: worker wall time {time.perf_counter() - t0:.1f} s on {job.world} ranks", flush=True)


if __name__ == "__main__":
    main()
