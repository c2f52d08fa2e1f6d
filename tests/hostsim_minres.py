"""TEST INFRASTRUCTURE ONLY — the numpy stand-in of tests/hostsim_geneig.py extended by the entry point MINRES adds to
the C-ABI, b2k_minres_chain, with the library's refusals and handle-role contract (the roles of p_prev / p_cur and
d1 / d2 rotate once per completed iteration).  `installed()` routes `_lib.load()` to it like `hostsim.installed()`.
`minres_lie = (count, factor)` makes the next `count` convergence tests see factor·|φ̄| (the false-convergence branch
of the driver).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L

import hostsim_geneig
import minres_oracle as mo
from hostsim import _key, _set, _view


class MinresHostSimLib(hostsim_geneig.GenHostSimLib):
    def __init__(self):
        super().__init__()
        self.minres_calls = 0           # calls of b2k_minres_chain that got through the refusals
        self.minres_lie = (0, 1.0)

    def b2k_minres_chain(self, h, op, x, p_prev, p_cur, q, d1, d2, a0, a1, state_in, tol, nsteps, rec_out, state_out,
                         done):
        ctx = self._c(h)
        if op is None or state_in is None or rec_out is None or state_out is None or done is None or nsteps < 1:
            return self._fail(ctx, L.EINVAL, "minres_chain: null pointer / nsteps < 1")
        vecs = []
        for v in (x, p_prev, p_cur, q, d1, d2):
            v = int(v)
            if v < 0 or (v >> 20) >= len(ctx.spaces) or (v & 0xFFFFF) not in ctx.spaces[v >> 20].cols:
                return self._fail(ctx, L.EINVAL, f"invalid vector handle {v:#x}")
            vecs.append(self._vec(ctx, v))
        A = self.ops[_key(op)]
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "minres_chain: single-GPU contexts only")
        if not sp.issparse(A):
            return self._fail(ctx, L.ENOTSUP, "minres_chain: CSR / stencil operators only")
        n = len(vecs[0])
        if any(len(v) != n for v in vecs) or A.shape != (n, n):
            return self._fail(ctx, L.EDIM, "minres_chain: length mismatch")
        for i in range(6):
            for j in range(i):
                if vecs[i] is vecs[j]:
                    return self._fail(ctx, L.EINVAL, f"minres_chain: vectors {j} and {i} are the same")
        self.minres_calls += 1
        nsteps = min(nsteps, 511)
        xv, pp, pc, qv, da, db = vecs
        dt = ctx.dtype
        st = [float(s) for s in _view(state_in, 8, C.c_double)]
        rec = _view(rec_out, 8 * nsteps, C.c_double).reshape(nsteps, 8)
        d = 0
        for i in range(nsteps):
            ctx.launches += 2
            vk, vp = pc * dt(st[1]), pp * dt(st[2])
            qv[:] = self._shifted(ctx, op, vk, a0, a1)
            alpha = float(np.dot(vk.astype(np.float64), qv.astype(np.float64)))
            pp[:] = (qv + dt(-alpha) * vk) + dt(-st[0]) * vp
            bn = float(np.sqrt(np.dot(pp.astype(np.float64), pp.astype(np.float64))))
            al, bn, gamma, phi, phibar, sing, delta, eps = mo.givens_step(st, alpha, bn)
            # the library applies this update one launch late (it needs γ_k, hence β_{k+1}); the result is the same
            db[:] = 0 if sing else ((vk + dt(-delta) * da) + dt(-eps) * db) * dt(1.0 / gamma)
            xv[:] = xv + dt(phi) * db
            pp, pc, da, db = pc, pp, db, da
            code = 2.0 if sing else (1.0 if phibar < tol else (3.0 if bn == 0.0 else 0.0))
            cnt, fac = self.minres_lie
            if code == 0.0 and cnt > 0 and fac * phibar < tol:
                self.minres_lie = (cnt - 1, fac)
                phibar, code = fac * phibar, 1.0
            rec[i] = (al, bn, gamma, phi, phibar, code, delta, eps)
            d = i + 1
            if code != 0.0:
                break
        ctx.launches += 1
        _view(state_out, 8, C.c_double)[:] = st
        _set(done, d)
        return L.OK


class installed(hostsim_geneig.installed):
    """hostsim_geneig.installed, with the stand-in that also simulates b2k_minres_chain."""

    def __enter__(self):
        super().__enter__()
        L._lib = MinresHostSimLib()
        return L._lib
