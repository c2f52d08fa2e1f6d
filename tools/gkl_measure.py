"""Time the device-chained GKL step (b2k_gkl_expand_many) against the literal (A, At) tuple path on the H100.

    python tools/gkl_measure.py [--grids 3000x3000,700x700] [--steps 20] [--rounds 3] [--out DIR]

Workload: the Dirichlet forward-difference gradient G of an nx x ny grid ((nx+1) ny + nx (ny+1) rows, nx ny columns,
four nonzeros a column), Float64, ClassicalGramSchmidt2.  For each grid:
  * per GKL step: the same `--steps` expansions from the same start, chained (one call) and literal (one expansion per
    iteration, about four host round trips each), alternated in one process, best of `--rounds` after a warm-up;
    CUDA events on the context stream (b2k_timer_start / stop) around the expansions;
  * algorithmic bytes per step from the shapes: two CSR streams (12 B per nonzero, 4 B per row pointer), the gathered
    operand, y, the previous vector read and stored by each epilogue, and the U sweep's (2K + 3) m words at the
    batch's mean basis size K; TB/s = bytes / time;
  * a whole fixed-work svdsolve (tol = 0, fixed maxiter, howmany = 1), chained B200CSR entry against the tuple path.
Prints one JSON line per grid with the card name, power limit and clocks read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import ctypes as C  # noqa: E402

import krylovkit_jl_b200 as kk  # noqa: E402
from krylovkit_jl_b200.factorizations import gkl  # noqa: E402
from oracle import krylov_oracle as ko  # noqa: E402


def gradient(nx, ny):
    def d1(k):
        return sp.diags([np.ones(k), -np.ones(k)], [0, -1], shape=(k + 1, k), format="csr")
    return sp.vstack([sp.kron(sp.identity(ny, format="csr"), d1(nx), format="csr"),
                      sp.kron(d1(ny), sp.identity(nx, format="csr"), format="csr")], format="csr")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(ctx, fn):
    ctx.check(ctx.lib.b2k_timer_start(ctx.h))
    fn()
    ms = C.c_double()
    ctx.check(ctx.lib.b2k_timer_stop(ctx.h, C.byref(ms)))
    return ms.value


def expansions(ctx, op, opt, u0, steps, chained):
    """initialize a GKL factorization (not timed), then time `steps` expansions"""
    pair = (op, opt)
    it = gkl.GKLIterator(pair, u0, kk.cgs2, pair=pair if chained else None)
    f = gkl.initialize(it)
    ctx.sync()
    if chained:
        ms = timed(ctx, lambda: gkl.expand_many_(it, f, steps, 0.0))
    else:
        ms = timed(ctx, lambda: [gkl.expand_(it, f) for _ in range(steps)])
    assert len(f) == steps + 1
    alphas = list(f.alphas)
    del f, it
    return ms, alphas


def measure(nx, ny, steps, rounds, maxiter):
    t0 = time.time()
    A = gradient(nx, ny)
    m, n = A.shape
    build_s = time.time() - t0
    kd = steps + 2
    ctx = kk.B200Context(m, 3 * kd + 14)
    try:
        sv = ctx.add_space(n, 2 * kd + 14, sharded=False)
        op = kk.B200CSR.from_scipy(ctx, A).with_spaces(sv, 0)
        opt = op.transpose()
        u0 = ctx.from_host(ko.splitmix_vector(20261018, m))
        for chained in (True, False):                     # warm-up: every kernel and shape of the timed window
            expansions(ctx, op, opt, u0, steps, chained)
        best = {True: float("inf"), False: float("inf")}
        alph = {}
        for _ in range(rounds):
            for chained in (True, False):
                ms, al = expansions(ctx, op, opt, u0, steps, chained)
                best[chained] = min(best[chained], ms)
                alph[chained] = al
        kmean = 1 + (steps + 1) / 2.0
        nnz = A.nnz
        step_bytes = (2 * 12.0 * nnz + 4.0 * (m + n + 2) + 8.0 * (4 * n + 4 * m) + (2 * kmean + 3) * 8.0 * m)
        per = {c: best[c] / steps for c in best}
        # whole fixed-work svdsolve
        alg = kk.GKL(orth=kk.cgs2, krylovdim=kd, maxiter=maxiter, tol=0.0, verbosity=0)
        whole = {}
        for label, target in (("chained", op), ("tuple", (op, opt))):
            kk.svdsolve(target, u0, 1, "LR", alg)            # warm-up
            ts = []
            for _ in range(rounds):
                ctx.sync()
                t = time.perf_counter()
                S, _, _, info = kk.svdsolve(target, u0, 1, "LR", alg)
                ctx.sync()
                ts.append(time.perf_counter() - t)
            whole[label] = dict(s=min(ts), sigma=float(S[0]), numops=info.numops)
        rel = float(np.max(np.abs(np.array(alph[True]) - np.array(alph[False])) / np.abs(np.array(alph[False]))))
        return dict(grid=f"{nx}x{ny}", rows=m, cols=n, nnz=nnz, steps=steps, host_build_s=round(build_s, 1),
                    chained_ms_per_step=per[True], literal_ms_per_step=per[False],
                    speedup=per[False] / per[True], bytes_per_step=step_bytes,
                    chained_tb_s=step_bytes / (per[True] * 1e-3) / 1e12,
                    literal_tb_s=step_bytes / (per[False] * 1e-3) / 1e12,
                    alpha_max_rel_diff=rel, svdsolve=whole, card=card())
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="3000x3000,700x700")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--maxiter", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []
    for g in a.grids.split(","):
        nx, ny = (int(v) for v in g.split("x"))
        r = measure(nx, ny, a.steps, a.rounds, a.maxiter)
        line = json.dumps(r)
        print(line, flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "gkl_measure.jsonl"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
