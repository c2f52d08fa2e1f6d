"""Measure the pencil product of geneigsolve on the GPU and print one JSON line.

    python tools/geneig_measure.py [--nx 4000 --ny 2500] [--reps 20] [--cycles 3]

Pencil: K the 5-point Dirichlet Laplacian on an nx x ny grid, M = I + K/8 assembled with K's pattern (n = 1e7 by
default).  For Float64 and Float32:
  * the fused b2k_pencil_apply (w = A x - ρ B x - β vprev, bx = B x) against the same result composed of existing calls
    (two b2k_op_apply, two b2k_vec_axpby), timed with CUDA events over `reps` warmed-up repetitions, as algorithmic
    GB/s and as a share of the H100 SXM's 3.35 TB/s.  Bytes: fused 2 (T + 2) nnz + 4 (n + 1) + 4 T n (x, vprev read,
    w, bx written); composed 2 [(T + 4) nnz + 4 (n + 1) + 2 T n] + 2 * 3 T n.
  * seconds per restart cycle of geneigsolve(:LR, krylovdim = 30) on the pencil, with the share of the cross Gram
    sweeps (b2k_prof class 9).
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import krylovkit_jl_b200 as kk  # noqa: E402

HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception as e:          # the measurement still stands, the card is reported as unknown
        return f"unknown ({e})", "unknown"


def timed(ctx, fn, reps):
    for _ in range(3):
        fn()
    ctx.sync()
    ms = C.c_double()
    ctx.check(ctx.lib.b2k_timer_start(ctx.h))
    for _ in range(reps):
        fn()
    ctx.check(ctx.lib.b2k_timer_stop(ctx.h, C.byref(ms)))
    return ms.value / 1e3 / reps


def measure(dt, nx, ny, reps, cycles):
    n = nx * ny
    es = np.dtype(dt).itemsize
    ctx = kk.B200Context(n, 4 * 31 + 3, dtype=dt)
    try:
        K = kk.B200CSR.stencil(ctx, nx, ny)
        M = kk.B200CSR.stencil(ctx, nx, ny, coeffs=(1.5, -0.125, -0.125, -0.125, -0.125, 0.0, 0.0))
        nnz = K.nnz
        P = kk.B200Pencil(K, M)
        x, vp = ctx.splitmix(1), ctx.splitmix(2)
        w, bx = ctx.empty(), ctx.empty()
        rho, beta = 0.37, 0.61

        def fused():
            P.apply_into(x, w, bx, rho, vp, beta)

        def composed():
            K.apply_into(w, x)
            M.apply_into(bx, x)
            w.add_(bx, -rho)
            w.add_(vp, -beta)

        fused()
        ref_w, ref_bx = w.to_host(), bx.to_host()
        composed()
        same = bool(np.array_equal(w.to_host(), ref_w) and np.array_equal(bx.to_host(), ref_bx))
        b_fused = 2 * (es + 2) * nnz + 4 * (n + 1) + 4 * es * n
        b_comp = 2 * ((es + 4) * nnz + 4 * (n + 1) + 2 * es * n) + 2 * 3 * es * n
        t_f, t_c = [], []
        for _ in range(3):                    # alternate the two so drift hits both
            t_f.append(timed(ctx, fused, reps))
            t_c.append(timed(ctx, composed, reps))
        tf, tc = min(t_f), min(t_c)
        res = dict(dtype=np.dtype(dt).name, n=n, nnz=nnz, bitwise_equal=same,
                   fused_ms=tf * 1e3, composed_ms=tc * 1e3,
                   fused_GBps=b_fused / tf / 1e9, composed_GBps=b_comp / tc / 1e9,
                   fused_share_of_hbm=b_fused / tf / HBM, composed_share_of_hbm=b_comp / tc / HBM,
                   speedup=tc / tf)
        # seconds per restart cycle of geneigsolve(:LR, krylovdim = 30)
        alg = kk.GolubYe(krylovdim=30, maxiter=cycles, tol=1e-14, verbosity=0)
        x0 = ctx.splitmix(3)
        kk.geneigsolve(P, x0, 1, "LR", kk.GolubYe(krylovdim=30, maxiter=1, tol=1e-14, verbosity=0))   # warm-up
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 1))
        ctx.check(ctx.lib.b2k_prof_reset(ctx.h))
        ctx.sync()
        t0 = time.perf_counter()
        _, _, info = kk.geneigsolve(P, x0, 1, "LR", alg)
        ctx.sync()
        dt_solve = time.perf_counter() - t0
        cnt, ms, nb = C.c_int64(), C.c_double(), C.c_double()
        ctx.check(ctx.lib.b2k_prof_read(ctx.h, 9, C.byref(cnt), C.byref(ms), C.byref(nb)))
        ctx.check(ctx.lib.b2k_prof_enable(ctx.h, 0))
        res.update(cycle_s=dt_solve / info.numiter, cycles=info.numiter, numops=info.numops,
                   cross_gram_share=ms.value / 1e3 / dt_solve, cross_gram_calls=cnt.value)
        P.free()
        return res
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nx", type=int, default=4000)
    ap.add_argument("--ny", type=int, default=2500)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cycles", type=int, default=3)
    a = ap.parse_args()
    name, pl = card()
    out = dict(card=name, power_limit=pl, results=[measure(dt, a.nx, a.ny, a.reps, a.cycles)
                                                   for dt in (np.float64, np.float32)])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
