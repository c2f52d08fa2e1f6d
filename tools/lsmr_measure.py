"""Time lssolve(LSMR) on a device CSR matrix, chained (b2k_lsmr_chain) against the literal loop over (A, Aᵀ); print
one JSON line.

    python tools/lsmr_measure.py [--iters 16 80] [--rounds 3] [--small]

Problems: the 8e6 x 4e6 [L; I] of tools/run_configs.py::widened (L the 5-point Laplacian of a 2000 x 2000 grid) and the
forward-difference gradient of a 3000 x 3000 grid (17.99e6 x 9e6).  For each problem, Float64 and Float32, and
krylovdim 1 (no reorthogonalisation), 8 with ModifiedGramSchmidt and 8 with ClassicalGramSchmidt2, both paths run a
fixed number of iterations (tol = 0) twice, at iters[0] and iters[1]; the time per iteration is the difference over the
iteration difference, so the set-up (the device transpose of the chained entry, the first Aᵀ b) drops out.  A call is
timed with CUDA events on the context stream (b2k_timer_start / b2k_timer_stop) around the whole lssolve; the two paths
are alternated `rounds` times after a warm-up of each, and the best time is kept.  Both paths' x after iters[1]
iterations must agree to 1e-10 (Float64) / 1e-4 (Float32) relative in the 2-norm; the script fails otherwise.  The
card's name and power limit are read in the same run.  Needs a GPU; there is no fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import krylovkit_jl_b200 as kk  # noqa: E402
from oracle import krylov_oracle as ko  # noqa: E402  (host-side test matrices only)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, pl = [s.strip() for s in out.split(",")]
    return name, pl


def grad2d(nx, ny):
    dx = sp.diags([-np.ones(nx - 1), np.ones(nx - 1)], [0, 1], shape=(nx - 1, nx), format="csr")
    dy = sp.diags([-np.ones(ny - 1), np.ones(ny - 1)], [0, 1], shape=(ny - 1, ny), format="csr")
    return sp.vstack([sp.kron(sp.identity(ny, format="csr"), dx), sp.kron(dy, sp.identity(nx, format="csr"))]).tocsr()


def l_on_i(nx, ny):
    n = nx * ny
    return sp.vstack([ko.stencil_matrix(nx, ny), sp.identity(n, format="csr")]).tocsr()


def run_problem(name, Ah, dtype, iters, rounds):
    m, n = Ah.shape
    ctx = kk.B200Context(m, 12, dtype=dtype)
    res = []
    try:
        sv = ctx.add_space(n, 24, sharded=False)
        A = kk.B200CSR.from_scipy(ctx, Ah.astype(dtype)).with_spaces(sv, 0)
        At = kk.B200CSR.from_scipy(ctx, Ah.T.tocsr().astype(dtype)).with_spaces(0, sv)
        b = ctx.splitmix(1234)
        for orth, K in (("mgs", 1), ("mgs", 8), ("cgs2", 8)):
            def run(op, N):
                alg = kk.LSMR(orth=getattr(kk, orth), maxiter=N, krylovdim=K, tol=0.0, verbosity=0)
                ms = C.c_double()
                ctx.check(ctx.lib.b2k_timer_start(ctx.h))
                x, info = kk.lssolve(op, b, alg)
                ctx.check(ctx.lib.b2k_timer_stop(ctx.h, C.byref(ms)))
                t = ms.value * 1e-3
                assert info.numiter == N
                return t, x
            best = {"chain": [np.inf, np.inf], "literal": [np.inf, np.inf]}
            ops = {"chain": A, "literal": (A, At)}
            for p in ops:                                   # warm-up
                run(ops[p], iters[0])
            xs = {}
            for _ in range(rounds):
                for p in ("chain", "literal"):
                    for j, N in enumerate(iters):
                        t, x = run(ops[p], N)
                        best[p][j] = min(best[p][j], t)
                        if j == 1:
                            xs[p] = x.to_host().astype(np.float64)
            per = {p: (best[p][1] - best[p][0]) / (iters[1] - iters[0]) for p in best}
            dx = float(np.linalg.norm(xs["chain"] - xs["literal"]) / np.linalg.norm(xs["literal"]))
            if not dx <= (1e-10 if dtype == np.float64 else 1e-4):
                raise SystemExit(f"{name} {np.dtype(dtype).name} {orth} K={K}: chained and literal x differ by {dx}")
            res.append({"problem": name, "m": m, "n": n, "nnz": int(Ah.nnz), "dtype": np.dtype(dtype).name,
                        "orth": orth, "krylovdim": K, "chain_ms_per_iter": per["chain"] * 1e3,
                        "literal_ms_per_iter": per["literal"] * 1e3,
                        "speedup": per["literal"] / per["chain"], "x_rel_diff": dx})
            print(json.dumps(res[-1]), file=sys.stderr, flush=True)
    finally:
        ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, nargs=2, default=[16, 80])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--small", action="store_true", help="small grids, for a quick check of the script")
    a = ap.parse_args()
    name, pl = card()
    probs = [("L_on_I_2000", lambda: l_on_i(2000, 2000)), ("grad_3000", lambda: grad2d(3000, 3000))]
    if a.small:
        probs = [("L_on_I_200", lambda: l_on_i(200, 200)), ("grad_300", lambda: grad2d(300, 300))]
    out = []
    for pname, make in probs:
        Ah = make()
        for dt in (np.float64, np.float32):
            out += run_problem(pname, Ah, dt, a.iters, a.rounds)
        del Ah
    print(json.dumps({"card": name, "power_limit": pl, "iters": a.iters, "rounds": a.rounds, "results": out}))


if __name__ == "__main__":
    main()
