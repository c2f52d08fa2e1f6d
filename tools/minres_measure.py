"""Measure MINRES on the GPU and print one JSON line.

    python tools/minres_measure.py [--nx 4000 --ny 2500] [--iters 256] [--rounds 3] [--gmres-cycles 20]

System: (A − σI) x = b with A the 5-point Dirichlet Laplacian on an nx x ny grid (n = 1e7 by default), σ in the middle
of the widest gap between neighbouring closed-form eigenvalues in the lower third of the spectrum (indefinite and
nonsingular), Float64, b from the splitmix generator.
  * b2k_minres_chain: CUDA-event time per iteration over `iters` iterations (calls of 32) after a warm-up call, as
    algorithmic GB/s and as a share of the H100 SXM's 3.35 TB/s.  Bytes per iteration: one SpMV in the operator's active
    layout (values and column indices as streamed, row pointers, x read, y written) + 9 W for k_minres_step
    (W = 8 n).  The flush launch that ends each call (6 W per 32 iterations) is in the time and not in the bytes.
  * the same solve three ways, to the tolerance the chain reached after `iters` iterations: linsolve(MINRES) chained,
    linsolve(MINRES) literal, linsolve(GMRES(krylovdim = 40)) bounded at `gmres-cycles` restart cycles — iterations,
    operator applications, wall time to solution; the three are alternated `rounds` times and the best time kept.
The card's name and power limit are read in the same run.  Needs a GPU; there is no fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import krylovkit_jl_b200 as kk  # noqa: E402

HBM = 3.35e12
CALL = 32
F32V, I16, RP16 = 1, 2, 4          # b2k_debug_csr_format bits


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception as e:          # the measurement still stands, the card is reported as unknown
        return f"unknown ({e})", "unknown"


def laplace_shift(nx, ny):
    """the middle of the widest gap between neighbouring eigenvalues in the lower third of the spectrum (past the
    first 50), from the closed form λ = 4 − 2cos(iπ/(nx+1)) − 2cos(jπ/(ny+1))"""
    lx = 2 - 2 * np.cos(np.arange(1, nx + 1) * np.pi / (nx + 1))
    ly = 2 - 2 * np.cos(np.arange(1, ny + 1) * np.pi / (ny + 1))
    lam = np.unique(np.round((lx[:, None] + ly[None, :]).ravel(), 12))
    g = np.diff(lam[:len(lam) // 3])
    j = int(np.argmax(g[50:])) + 50
    return float(0.5 * (lam[j] + lam[j + 1])), float(g[j])


def spmv_bytes(n, nnz, es, fmt):
    """bytes one CSR SpMV streams in the layout `fmt` (b2k_debug_csr_format): matrix + x + y"""
    return nnz * ((4 if fmt & F32V else es) + (2 if fmt & I16 else 4)) + (n + 1) * (2 if fmt & RP16 else 4) + 2 * es * n


def iteration_bytes(n, nnz, es, fmt):
    return spmv_bytes(n, nnz, es, fmt) + 9 * es * n


def measure(nx, ny, iters, rounds, gmres_cycles):
    ls = importlib.import_module("krylovkit_jl_b200.linsolve")
    n, es = nx * ny, 8
    sigma, gap = laplace_shift(nx, ny)
    ctx = kk.B200Context(n, 56)
    try:
        op = kk.B200CSR.stencil(ctx, nx, ny)
        fmt = int(ctx.lib.b2k_debug_csr_format(op.h))
        b = ctx.splitmix(20260923)
        beta1 = b.norm()
        names = ("x", "p_prev", "p_cur", "q", "d1", "d2")
        v = {k: ctx.zeros() for k in names}

        def chain_run(calls):
            for k in names:
                v[k].zerovector_()
            v["p_cur"].scale_(1.0, b)
            st, phibar = [beta1, 1.0 / beta1, 0.0, -1.0, 0.0, 0.0, 0.0, beta1], beta1
            for _ in range(calls):
                rec, done = np.zeros((CALL, 8)), C.c_int32()
                sin, sout = (C.c_double * 8)(*st), (C.c_double * 8)()
                ctx.check(ctx.lib.b2k_minres_chain(ctx.h, op.h, *[v[k].handle for k in names], -sigma, 1.0, sin, 0.0,
                                                   CALL, rec.ctypes.data_as(C.POINTER(C.c_double)), sout, C.byref(done)))
                assert done.value == CALL
                st, phibar = list(sout), rec[-1, 4]
            return phibar

        calls = -(-iters // CALL)
        chain_run(1)
        ctx.sync()
        ms = C.c_double()
        ctx.check(ctx.lib.b2k_timer_start(ctx.h))
        phibar = chain_run(calls)
        ctx.check(ctx.lib.b2k_timer_stop(ctx.h, C.byref(ms)))
        t_it = ms.value / 1e3 / (calls * CALL)
        nbytes = iteration_bytes(n, op.nnz, es, fmt)
        res = dict(n=n, nnz=op.nnz, sigma=sigma, gap=gap, csr_format=fmt, chain_iterations=calls * CALL,
                   chain_ms_per_iteration=t_it * 1e3, bytes_per_iteration=nbytes, chain_GBps=nbytes / t_it / 1e9,
                   chain_share_of_hbm=nbytes / t_it / HBM, phibar_over_beta1=phibar / beta1)
        for k in names:
            v[k].free()
        tol = phibar * 1.0001
        arms = {
            "minres_chained": (True, kk.MINRES(maxiter=4 * calls * CALL, tol=tol, verbosity=0)),
            "minres_literal": (False, kk.MINRES(maxiter=4 * calls * CALL, tol=tol, verbosity=0)),
            "gmres40": (True, kk.GMRES(krylovdim=40, maxiter=gmres_cycles, tol=tol, verbosity=0)),
        }
        best = {}
        for _ in range(rounds):                    # alternate the arms so drift hits all of them
            for name, (chain, alg) in arms.items():
                ls.USE_MINRES_CHAIN = chain
                ctx.sync()
                t0 = time.perf_counter()
                x, info = kk.linsolve(op, b, None, alg, -sigma, 1.0)
                ctx.sync()
                dt = time.perf_counter() - t0
                if name not in best or dt < best[name]["seconds"]:
                    best[name] = dict(seconds=dt, converged=info.converged, numiter=info.numiter, numops=info.numops,
                                      normres_over_beta1=info.normres / beta1)
                del x, info
        ls.USE_MINRES_CHAIN = True
        res["tol_over_beta1"] = tol / beta1
        res["solves"] = best
        return res
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--nx", type=int, default=4000)
    ap.add_argument("--ny", type=int, default=2500)
    ap.add_argument("--iters", type=int, default=256, help="iterations timed through b2k_minres_chain (>= 200)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gmres-cycles", type=int, default=20)
    a = ap.parse_args()
    if a.iters < 200:
        ap.error("--iters must be at least 200")
    name, pl = card()
    print(json.dumps(dict(card=name, power_limit=pl, result=measure(a.nx, a.ny, a.iters, a.rounds, a.gmres_cycles))))


if __name__ == "__main__":
    main()
