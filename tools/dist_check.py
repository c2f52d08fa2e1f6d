"""Run under torchrun (one rank per GPU): row-sharded eigsolve / primitives vs the CPU oracle.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29611 tools/dist_check.py

B2K_ONE_GPU=1: all ranks share GPU 0 (torch.distributed over gloo, library transport = NVLink peer window only,
B2K_NO_NCCL=1 — NCCL refuses two ranks on one device).  Same checks; this is how a single-GPU box exercises the
sharded path, including the in-kernel cross-rank reductions (the ranks' kernels then alternate by time slicing).
"""
import os
import sys

os.environ.setdefault("OPENBLAS_NUM_THREADS", "8")   # small oracle problems: a 128-thread pool only adds latency

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import krylovkit_jl_b200 as kk  # noqa: E402
from krylovkit_jl_b200 import sharding  # noqa: E402
from oracle import krylov_oracle as ko  # noqa: E402


def watchdog_check(rank, world, local):
    """DIST_CHECK_WATCHDOG=1: a rank that leaves the SPMD call order must not leave its peers spinning on the GPU.
    Rank 0 calls one all-reduce more than the others; its in-kernel wait for the missing flags gives up after
    B2K_PEER_TIMEOUT_S and the call returns B2K_ENCCL (csrc/common.cuh: peer_spin, csrc/dist.cu: b2k_stream_sync)."""
    import time
    os.environ["B2K_PEER_TIMEOUT_S"] = "2"
    uid = sharding.broadcast_nccl_uid(dist, kk._lib.load())
    n_loc = 4096
    ctx = kk.B200Context(n_loc, 8, device=local, rank=rank, nranks=world, nccl_uid=uid,
                         n_global=n_loc * world, row_offset=n_loc * rank)
    x = ctx.splitmix(7)
    nrm = x.norm()                                  # every rank takes part: works
    assert nrm > 0.0
    dist.barrier()
    if rank == 0:
        t0 = time.time()
        try:
            x.norm()                                # nobody else comes
        except kk.B200Error as e:
            assert "timed out" in str(e), str(e)
            dt = time.time() - t0
            assert 1.0 < dt < 150.0, dt             # the 2 s the test allows, plus scheduling
            print(f"dist_check ok on {world} ranks (watchdog): B2K_ENCCL after {dt:.1f} s")
        else:
            raise AssertionError("the lone all-reduce returned without an error")
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


def onepass_check(shard, n_global, rank, world, local, dev, use_nccl):
    """b2k_op_apply_normal_gram on a row-sharded splitmix matrix (oracle/onepass_restate.py states the order), on a
    context of its own per type: Float64 with 300 columns, Float32 with 1100 (two 1024-column pieces of the peer
    all-reduce when NCCL is off; more than the 846 columns a Float64 tile may have).  Each rank's y is its own rows'
    restatement with the grid that rank launched; z, on every rank, is the rank-ordered sum from 0.0 of the ranks'
    restated Float64 sums, rounded to T.  With NCCL, more than 1024 columns go through ncclAllReduce, whose order is
    NCCL's: with three or more ranks only the Float64 bound is asserted there (two addends give the same bits in
    either order)."""
    import ctypes
    import shutil
    import tempfile
    from krylovkit_jl_b200.operators import apply_normal_gram
    from oracle import onepass_restate as rs
    tmp = tempfile.mkdtemp(prefix="onepass_fma_")
    try:
        fma = rs.load_fma(tmp)
        lib = kk._lib.load()
        for dt, ncols, seed in ((np.float64, 300, 41), (np.float32, 1100, 43)):
            uid = sharding.broadcast_nccl_uid(dist, lib)
            ctx = kk.B200Context(shard.n_local, 4, dtype=dt, device=local, rank=rank, nranks=world, nccl_uid=uid,
                                 n_global=n_global, row_offset=shard.row_offset)
            sv = ctx.add_space(ncols, 4, sharded=False)
            op = kk.B200Dense.splitmix(ctx, shard.n_local, ncols, seed, sv)
            A = ko.dense_splitmix(seed, shard.n_local, ncols, dtype=dt, row0=shard.row_offset, m_global=n_global)
            x = (ko.splitmix_vector(seed + 1, ncols) - 0.5).astype(dt)
            y, z = apply_normal_gram(op, ctx.from_host(x, space=sv))
            info = (ctypes.c_int32 * 4)()
            assert lib.b2k_debug_onepass_launch(info) == 0 and info[0] == 0, list(info)
            ry, _, dres, _ = rs.apply_normal_gram(A, x, 0, info[2], fma)
            u = np.uint64 if dt == np.float64 else np.uint32
            assert np.array_equal(y.to_host().view(u), ry.view(u)), (rank, ncols)
            parts = [torch.zeros(ncols, dtype=torch.float64, device=dev) for _ in range(world)]
            dist.all_gather(parts, torch.from_numpy(dres).to(dev))
            per_rank = [p.cpu().numpy() for p in parts]
            want = rs.rank_sum(per_rank)
            zh = z.to_host()
            if use_nccl and ncols > 1024 and world > 2:
                bound = world * 2.0 ** -53 * np.sum(np.abs(per_rank), axis=0) + np.abs(want) * np.finfo(dt).eps
                assert np.all(np.abs(zh - want) <= bound), (rank, ncols)
            else:
                assert np.array_equal(zh.view(u), want.astype(dt).view(u)), (rank, ncols)
            del y, z, op
            ctx.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if rank == 0:
        print(f"dist_check: one-pass GKL step bit-equal to the restatement on {world} ranks")


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    one_gpu = os.environ.get("B2K_ONE_GPU", "") == "1"
    if one_gpu:
        os.environ["B2K_NO_NCCL"] = "1"
        local = 0
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = "cpu" if one_gpu else "cuda"
    if os.environ.get("DIST_CHECK_WATCHDOG", "") == "1":
        return watchdog_check(rank, world, local)
    uid = sharding.broadcast_nccl_uid(dist, kk._lib.load())
    nx, ny = 200, 151
    n = nx * ny
    shard = sharding.shard_grid_lines(nx, ny, rank, world)
    ctx = kk.B200Context(shard.n_local, 64, device=local, rank=rank, nranks=world, nccl_uid=uid,
                         n_global=n, row_offset=shard.row_offset)
    A = ko.stencil_matrix(nx, ny)
    x0 = ko.splitmix_vector(20260923, n)
    sl = slice(shard.row_offset, shard.row_offset + shard.n_local)
    sizes = [sharding.shard_grid_lines(nx, ny, r, world).n_local for r in range(world)]

    def gather(vec):
        """the global vector from its row shards (padded to equal length: gloo's all_gather wants that)"""
        loc = torch.zeros(max(sizes), dtype=torch.float64, device=dev)
        loc[:shard.n_local] = torch.from_numpy(vec.to_host()).to(dev)
        parts = [torch.zeros(max(sizes), dtype=torch.float64, device=dev) for _ in range(world)]
        dist.all_gather(parts, loc)
        return torch.cat([p[:m] for p, m in zip(parts, sizes)]).cpu().numpy()
    # 1. device-side start vector is the global splitmix sequence
    xd = ctx.splitmix(20260923)
    assert np.array_equal(xd.to_host(), x0[sl])
    # 2. sharded SpMV (halo exchange) for the stencil and for an uploaded CSR with global columns
    ref = A @ x0
    op = kk.B200CSR.stencil(ctx, nx, ny)
    y = kk.apply(op, xd)
    assert np.allclose(y.to_host(), ref[sl], rtol=1e-14, atol=1e-14)
    Aloc = A[sl].tocsr()
    op2 = kk.B200CSR.from_csr_arrays(ctx, shard.n_local, n, Aloc.indptr.astype(np.int64),
                                     Aloc.indices.astype(np.int64), Aloc.data)
    y2 = kk.apply(op2, xd)
    assert np.array_equal(y2.to_host(), y.to_host())
    # 2b. the matrix-free stencil operator: the same bits as the assembled one (halo = one grid line per neighbour)
    opf = kk.B200CSR.stencil_free(ctx, nx, ny)
    assert np.array_equal(kk.apply(opf, xd).to_host(), y.to_host())
    # 3. global reductions
    assert abs(xd.inner(y) - x0 @ ref) < 1e-9 * abs(x0 @ ref)
    assert abs(xd.norm() - np.linalg.norm(x0)) < 1e-12 * np.linalg.norm(x0)
    # 4. eigsolve, converged and fixed-cycle, vs the serial oracle
    for orth, oorth in ((kk.cgs2, ko.Orth(ko.CGS2)), (kk.mgs2, ko.Orth(ko.MGS2))):
        alg = kk.Lanczos(orth=orth, krylovdim=30, maxiter=200, tol=1e-10, verbosity=0)
        vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0[sl]), 3, "SR", alg)
        ovals, ovecs, oinfo = ko.eigsolve_lanczos(A, x0, 3, "SR", krylovdim=30, maxiter=200, tol=1e-10,
                                                  orth=oorth)
        assert info.converged >= 3 and info.numops == oinfo["numops"], (info.numops, oinfo["numops"])
        assert np.allclose(vals[:3], ovals[:3], rtol=1e-10)
        lam = ko.laplace_eigenvalues(nx, ny)
        assert np.allclose(vals[:3], lam[:3], rtol=1e-10)
        # gather one Ritz vector and check the residual globally
        v = gather(vecs[0])
        assert np.linalg.norm(A @ v - vals[0] * v) < 1e-8
        del vecs
    # 4b. the benchmark regime (fixed restart cycles, tol = 0) through the device-chained steps — in-kernel
    #     cross-rank reductions and halo rows pushed by the Gram-Schmidt launch — vs the serial oracle, and vs the
    #     same job with one synchronous step at a time (NCCL / peer all-reduce launches between the sweeps)
    alg = kk.Lanczos(orth=kk.cgs2, krylovdim=40, maxiter=4, tol=0.0, verbosity=0)
    lib = kk._lib.load()
    res = {}
    for chain in (1, 0):
        lib.b2k_debug_set_chain(chain)
        vals, vecs, info = kk.eigsolve(op, ctx.from_host(x0[sl]), 4, "SR", alg)
        res[chain] = (np.array(vals[:4]), info.numops, np.array(info.normres[:4]))
        del vecs
    lib.b2k_debug_set_chain(1)
    ovals, _, oinfo = ko.eigsolve_lanczos(A, x0, 4, "SR", krylovdim=40, maxiter=4, tol=0.0, orth=ko.Orth(ko.CGS2))
    assert res[1][1] == res[0][1] == oinfo["numops"]
    assert np.allclose(res[1][0], ovals[:4], rtol=1e-10) and np.allclose(res[0][0], ovals[:4], rtol=1e-10)
    assert np.allclose(res[1][0], res[0][0], rtol=1e-12), (res[1][0], res[0][0])
    assert np.allclose(res[1][2], oinfo["normres"][:4], rtol=1e-6)
    if os.environ.get("DIST_CHECK_SHORT", "") == "1":
        if rank == 0:
            print(f"dist_check ok on {world} ranks (short): Ritz values {res[1][0][:3]}")
        dist.barrier()
        ctx.close()
        onepass_check(shard, n, rank, world, local, dev, use_nccl=not one_gpu)
        dist.destroy_process_group()
        return
    # 5. widened drivers (SURVEY §8f) on the sharded context: every scalar they see is all-reduced inside
    #    the library, so the host logic is rank-replicated; results = the serial oracle's

    import importlib
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    cdc = (5.0, -1.4, -0.6, -1.2, -0.8, 0.0, 0.0)
    Acd = ko.stencil_matrix(nx, ny, 1, cdc)
    opcd = kk.B200CSR.stencil(ctx, nx, ny, 1, cdc)
    bh = ko.splitmix_vector(7, n)
    ox, oinfo = ko.linsolve_bicgstab(Acd, bh, maxiter=200, tol=1e-10)
    for fused in (True, False):
        ls.USE_FUSED_BICGSTAB = fused
        x, info = kk.linsolve(opcd, ctx.from_host(bh[sl]), None, kk.BiCGStab(maxiter=200, tol=1e-10, verbosity=0))
        assert info.converged == 1 and abs(info.numiter - oinfo["numiter"]) <= 1, (info.numiter, oinfo["numiter"])
        xg = gather(x)
        assert np.linalg.norm(Acd @ xg - bh) < 1e-9 and np.allclose(xg, ox, rtol=1e-7, atol=1e-9)
    ls.USE_FUSED_BICGSTAB = True
    spd = (5.0, -1.0, -1.0, -1.0, -1.0, 0.0, 0.0)
    Aspd, opspd = ko.stencil_matrix(nx, ny, 1, spd), kk.B200CSR.stencil(ctx, nx, ny, 1, spd)
    x, info = kk.linsolve(opspd, ctx.from_host(bh[sl]), None, kk.CG(maxiter=500, tol=1e-9, verbosity=0))
    ox, oinfo = ko.linsolve_cg(Aspd, bh, maxiter=500, tol=1e-9)
    assert info.converged == 1 and abs(info.numiter - oinfo["numiter"]) <= 1
    assert np.linalg.norm(Aspd @ gather(x) - bh) < 1e-8
    # fixed number of restart cycles (tol = 0): same Krylov spaces as the serial oracle, same Ritz values
    alg = kk.Arnoldi(orth=kk.cgs2, krylovdim=30, maxiter=4, tol=0.0, verbosity=0)
    vals, vecs, info = kk.eigsolve(opcd, ctx.from_host(x0[sl]), 2, "LR", alg)
    ovals, _, oinfo = ko.eigsolve_arnoldi(Acd, x0, 2, "LR", krylovdim=30, maxiter=4, tol=0.0, orth=ko.Orth(ko.CGS2))
    assert info.numops == oinfo["numops"] and np.allclose(vals[:2], ovals[:2], rtol=1e-7), (vals[:2], ovals[:2])
    vg = gather(vecs[0].re) + 1j * gather(vecs[0].im)
    rg = gather(info.residual[0].re) + 1j * gather(info.residual[0].im)
    assert np.linalg.norm(Acd @ vg - vals[0] * vg - rg) < 1e-9
    del vecs, info
    X0 = [ko.splitmix_vector(100 + i, n) for i in range(3)]
    alg = kk.BlockLanczos(krylovdim=30, maxiter=4, tol=0.0, verbosity=0)
    vals, vecs, info = kk.eigsolve(op, kk.Block([ctx.from_host(x[sl]) for x in X0]), 3, "SR", alg)
    ovals, _, oinfo = ko.eigsolve_blocklanczos(A, X0, 3, "SR", krylovdim=30, maxiter=4, tol=0.0)
    assert info.numops == oinfo["numops"] and np.allclose(vals[:3], ovals[:3], rtol=1e-7), (vals[:3], ovals[:3])
    del vecs, info
    w, info = kk.exponentiate(op, -0.3, ctx.from_host(x0[sl]), kk.Lanczos(orth=kk.cgs2, krylovdim=25, tol=1e-10, verbosity=0))
    ow, _ = ko.expintegrator(A, -0.3, (x0,), "lanczos", ko.Orth(ko.CGS2), krylovdim=25, tol=1e-10)
    assert info.converged == 1 and np.allclose(gather(w), ow, rtol=1e-9, atol=1e-11)
    if rank == 0:
        print(f"dist_check ok on {world} ranks: Ritz values {vals[:3]}")
    dist.barrier()
    ctx.close()
    # the one-pass dense GKL step on the row shards: y and the per-rank sums against the restatement
    onepass_check(shard, n, rank, world, local, dev, use_nccl=not one_gpu)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
