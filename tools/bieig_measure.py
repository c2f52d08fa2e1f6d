"""Measurements of bieigsolve (BiArnoldi) on one GPU, written as one JSON file.

    python tools/bieig_measure.py --out DIR [--n 10000000] [--reps 20] [--maxiter 3]

1. b2k_basis_cross_inner at n rows, p = q in {16, 31, 61}, Float64 and Float32: the sweep kernel's time (CUDA events
   of the profile class, over `reps` calls after warm-up) and the whole call's time (events around the calls, each
   of which ends in a host synchronisation).  Algorithmic bytes and flops from shapes, achieved bytes/s, and which
   bound (HBM at 3.35 TB/s, or the FMA rate of the type) limits the kernel.  In the same run, alternating with it,
   the border of one restart cycle formed the reference's way (biarnoldi.jl:285-288, 354-358) through existing
   calls: per expansion step two b2k_basis_project calls and one inner product, plus the two projections of the
   process step.
2. bieigsolve on a non-symmetric convection-diffusion stencil assembled on the device (B200CSR.stencil with unequal
   west / east and south / north coefficients, 4000 x 2500 grid), krylovdim 30, a fixed maxiter: time per restart
   cycle, numops, the share of the time spent in the cross Gram sweeps, and one check of every returned pair:
   ||A x - lambda x - r|| / ||A||_inf ||x|| (one SpMV per real / imaginary part).
The card's name, power limit and maximum SM clock are read in the same run.  Nothing is written into the tree.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# centre, west, east, south, north (down / up unused in 2-D): upwinded convection to the east and north
COEFFS = (4.0, -1.3, -0.7, -1.2, -0.8, 0.0, 0.0)
HBM = 3.35e12                                   # H100 SXM data sheet, bytes/s
FMA_RATE = {"float64": 33.5e12, "float32": 66.9e12}     # H100 SXM data sheet, non-tensor FP64 / FP32 flop/s
CROSS = 9                                       # profile class of the cross Gram sweep


def convdiff_eigenvalues(nx, ny, c=COEFFS, top=None):
    """Eigenvalues of the Dirichlet 5-point stencil c on an nx x ny grid: a Kronecker sum of two tridiagonal Toeplitz
    matrices, c0 + 2 sqrt(cw ce) cos(i pi / (nx + 1)) + 2 sqrt(cs cn) cos(j pi / (ny + 1)) (real when cw ce > 0 and
    cs cn > 0).  `top`: only the `top` largest, in decreasing order."""
    ax = 2.0 * np.sqrt(c[1] * c[2]) * np.cos(np.arange(1, nx + 1) * np.pi / (nx + 1))
    ay = 2.0 * np.sqrt(c[3] * c[4]) * np.cos(np.arange(1, ny + 1) * np.pi / (ny + 1))
    if top is None:
        return (c[0] + ax[:, None] + ay[None, :]).ravel()
    ax, ay = np.sort(ax)[::-1][:top], np.sort(ay)[::-1][:top]
    return np.sort((c[0] + ax[:, None] + ay[None, :]).ravel())[::-1][:top]


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("nvidia-smi failed: this measurement needs the GPU")
    name, power, clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def prof_ms(ctx, cls):
    cnt, ms = C.c_int64(), C.c_double()
    ctx.check(ctx.lib.b2k_prof_read(ctx.h, cls, C.byref(cnt), C.byref(ms), None))
    return cnt.value, ms.value


def timed(ctx, fn, reps):
    """(call ms, sweep-kernel ms) per call"""
    lib = ctx.lib
    ctx.check(lib.b2k_prof_reset(ctx.h))
    ctx.check(lib.b2k_prof_enable(ctx.h, 1))
    ctx.check(lib.b2k_timer_start(ctx.h))
    for _ in range(reps):
        fn()
    ms = C.c_double()
    ctx.check(lib.b2k_timer_stop(ctx.h, C.byref(ms)))
    ctx.check(lib.b2k_prof_enable(ctx.h, 0))
    _, kms = prof_ms(ctx, CROSS)
    return ms.value / reps, kms / reps


def kernel_section(kk, n, reps):
    from krylovkit_jl_b200.vectors import handles
    rows = []
    for dt in (np.float64, np.float32):
        es = np.dtype(dt).itemsize
        pmax = 61
        ctx = kk.B200Context(n, 2 * pmax + 6, dtype=dt)
        W = [ctx.splitmix(100 + i) for i in range(pmax)]
        V = [ctx.splitmix(300 + i) for i in range(pmax)]
        lib = ctx.lib
        for p in (16, 31, 61):
            kd = p - 1                                   # X = [W_1 .. W_kd, r_W]: krylovdim + 1 columns
            keep = (3 * kd) // 5
            X, Y = W[:p], V[:p]
            hx, hy = handles(X), handles(Y)
            G = np.zeros((p, p), order="F")
            Gp = G.ctypes.data_as(C.POINTER(C.c_double))
            h = np.zeros(p)
            hp = h.ctypes.data_as(C.POINTER(C.c_double))
            d = C.c_double()

            def cross(skip):
                ctx.check(lib.b2k_basis_cross_inner(ctx.h, hx, p, hy, p, skip, skip, Gp, p))

            def reference_way():
                # expansions keep+1 .. kd: the border of M, then the two projections of the process step
                for j in range(keep, kd):
                    ctx.check(lib.b2k_basis_project(ctx.h, hx, j, Y[j].handle, 1.0, 0.0, hp))
                    ctx.check(lib.b2k_basis_project(ctx.h, hy, j, X[j].handle, 1.0, 0.0, hp))
                    ctx.check(lib.b2k_vec_inner(ctx.h, X[j].handle, Y[j].handle, C.byref(d)))
                ctx.check(lib.b2k_basis_project(ctx.h, hx, kd, Y[kd].handle, 1.0, 0.0, hp))
                ctx.check(lib.b2k_basis_project(ctx.h, hy, kd, X[kd].handle, 1.0, 0.0, hp))

            for _ in range(2):                           # warm-up of every shape
                cross(0)
                cross(keep)
                reference_way()
            res = {"full": [], "cycle": [], "ref_call": []}
            for _ in range(3):                           # alternate the two ways
                res["full"].append(timed(ctx, lambda: cross(0), reps))
                res["cycle"].append(timed(ctx, lambda: cross(keep), reps))
                ms = C.c_double()
                ctx.check(lib.b2k_timer_start(ctx.h))
                for _ in range(max(1, reps // 4)):
                    reference_way()
                ctx.check(lib.b2k_timer_stop(ctx.h, C.byref(ms)))
                res["ref_call"].append(ms.value / max(1, reps // 4))
            bytes_cross = 2.0 * p * n * es
            flops_full = 2.0 * n * p * p
            flops_cycle = 2.0 * n * (p * p - keep * keep)
            ref_bytes = sum(2 * (j + 1) * n * es + 2 * n * es for j in range(keep, kd)) + 2 * (kd + 1) * n * es
            call_full = min(c for c, _ in res["full"])
            k_full = min(k for _, k in res["full"])
            call_cycle = min(c for c, _ in res["cycle"])
            k_cycle = min(k for _, k in res["cycle"])
            t_hbm, t_fma = bytes_cross / HBM, flops_full / FMA_RATE[np.dtype(dt).name]
            rows.append({
                "dtype": np.dtype(dt).name, "n": n, "p": p, "q": p, "keep": keep,
                "bytes": bytes_cross, "flops_full": flops_full, "flops_cycle": flops_cycle,
                "kernel_ms_full": k_full, "call_ms_full": call_full,
                "kernel_ms_cycle": k_cycle, "call_ms_cycle": call_cycle,
                "achieved_bytes_per_s_full": bytes_cross / (k_full * 1e-3),
                "bound": "HBM" if t_hbm >= t_fma else "FMA",
                "share_of_bound_full": max(t_hbm, t_fma) / (k_full * 1e-3),
                "reference_way_ms": min(res["ref_call"]), "reference_way_bytes": ref_bytes,
                "runs": res,
            })
        ctx.close()
    return rows


def e2e_section(kk, maxiter, nx=4000, ny=2500, krylovdim=30, howmany=4):
    n = nx * ny
    ctx = kk.B200Context(n, 2 * krylovdim + 24 + 8 * (howmany + 1), dtype=np.float64)
    A = kk.B200CSR.stencil(ctx, nx, ny, 1, COEFFS)
    v0, w0 = ctx.splitmix(11), ctx.splitmix(12)
    lib = ctx.lib
    kk.bieigsolve(A, v0, w0, howmany, "LR", krylovdim=krylovdim, maxiter=1, verbosity=0)     # warm-up
    ctx.check(lib.b2k_prof_reset(ctx.h))
    ctx.check(lib.b2k_prof_enable(ctx.h, 1))
    ctx.sync()
    t0 = time.perf_counter()
    vals, (V, W), (iV, iW) = kk.bieigsolve(A, v0, w0, howmany, "LR", krylovdim=krylovdim, maxiter=maxiter,
                                           verbosity=0)
    ctx.sync()
    wall = time.perf_counter() - t0
    ctx.check(lib.b2k_prof_enable(ctx.h, 0))
    ncross, cross_ms = prof_ms(ctx, CROSS)
    normA = abs(COEFFS[0]) + sum(abs(c) for c in COEFFS[1:5])
    checks = []
    for lam, x, r in zip(vals, V, iV.residual):
        worst = 0.0
        # A x - λ x - r = (A re - a re + b im - r_re) + i (A im - a im - b re - r_im), λ = a + i b
        for part, other, sign, rp in ((x.re, x.im, 1.0, r.re), (x.im, x.re, -1.0, r.im)):
            y = kk.apply(A, part)
            y.add_(part, -lam.real)
            y.add_(other, sign * lam.imag)
            y.add_(rp, -1.0)
            worst = max(worst, y.norm())
        checks.append(worst / (normA * x.norm()))
    out = {"nx": nx, "ny": ny, "n": n, "krylovdim": krylovdim, "howmany": howmany, "maxiter": maxiter,
           "numiter": iV.numiter, "numops": iV.numops, "converged": iV.converged, "wall_s": wall,
           "s_per_cycle": wall / iV.numiter, "cross_calls": ncross, "cross_kernel_ms": cross_ms,
           "cross_share": cross_ms * 1e-3 / wall, "values": [[v.real, v.imag] for v in vals],
           "analytic_top": convdiff_eigenvalues(nx, ny, COEFFS, top=howmany).tolist(),
           "normres": list(map(float, iV.normres)), "relation_check": checks}
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--maxiter", type=int, default=3)
    args = ap.parse_args()
    import krylovkit_jl_b200 as kk
    os.makedirs(args.out, exist_ok=True)
    result = {"card": card(), "kernel": kernel_section(kk, args.n, args.reps),
              "bieigsolve": e2e_section(kk, args.maxiter)}
    result["card_after"] = card()
    path = os.path.join(args.out, "bieig_measure.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(path)


if __name__ == "__main__":
    main()
