"""Run under torchrun: the row-sharded SpMV kernels, the rank-ordered sums and the sharded Lanczos step against the
composed restatement of tests/dist_restate.py, bit for bit, on every rank (tests/test_gpu_zz_dist_restate.py).

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


def main():
    job = Job()
    tmp = tempfile.mkdtemp(prefix="dist_restate_fma_")
    try:
        fma = load_fma(tmp)
        refusal_check(job)
        blas1_checks(job)
        lanczos_checks(job, fma)
        spmv_checks(job, fma)
        job.finish()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
