"""TEST INFRASTRUCTURE ONLY — the numpy stand-in of tests/hostsim_gkl.py (which simulates the device transpose)
extended by the entry point the chained lssolve adds to the C-ABI, b2k_lsmr_chain, with the library's refusals and its
role contract: u and v normalised on entry and on return, v_{iter0+1} in ring slot iter0 % max(K, 1), and after a stop
code 2 / 3 the reference's v in its old slot / in the spare column.  The vectors are rounded as numpy rounds the
literal loop (not fma for fma); the scalars as the device recurrence.  `installed()` routes `_lib.load()` to it.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L

import hostsim_gkl
from hostsim import _key, _set, _view
from lsmr_restate import lsmr_scalars

MAX_CHAIN = 512
MAX_RING = 128
PANEL_COLS = {np.float64: 96, np.float32: 192}      # the cooperative sweep's panel ring


class LsmrHostSimLib(hostsim_gkl.GklHostSimLib):
    def __init__(self):
        super().__init__()
        self.lsmr_calls = 0         # calls of b2k_lsmr_chain that got through the refusals
        self.lsmr_iters = 0         # iterations those calls completed
        self.lsmr_codes = []        # stop code of every call's last iteration
        self.lsmr_enotsup = 0       # calls refused with B2K_ENOTSUP

    def b2k_lsmr_chain(self, hc, A, At, x, h, hbar, r, Ah, Ahbar, u, av, ring, K, spare, alg, iter0, state_in, tol,
                       nsteps, rec_out, state_out, done):
        ctx = self._c(hc)
        if A is None or At is None or ring is None or state_in is None or rec_out is None or state_out is None:
            return self._fail(ctx, L.EINVAL, "lsmr_chain: null pointer")
        if nsteps < 1 or nsteps > MAX_CHAIN - 1 or iter0 < 0:
            return self._fail(ctx, L.EINVAL, "lsmr_chain: need 1 <= nsteps <= 511 and iter0 >= 0")
        R = max(int(K), 1)
        if R > MAX_RING:
            return self._fail(ctx, L.ENOTSUP, "lsmr_chain: krylovdim > 128")
        mh = [int(v) for v in (r, Ah, Ahbar, u, av)]
        nh = [int(v) for v in (x, h, hbar, spare)]
        rh = [int(ring[i]) for i in range(R)]
        for v in mh + nh + rh:
            if v < 0 or (v >> 20) >= len(ctx.spaces) or (v & 0xFFFFF) not in ctx.spaces[v >> 20].cols:
                return self._fail(ctx, L.EINVAL, f"invalid vector handle {v:#x}")
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "lsmr_chain: row-sharded contexts are not supported")
        M, Mt = self.ops[_key(A)], self.ops[_key(At)]
        if not (sp.issparse(M) and sp.issparse(Mt)) or _key(A) in self.free_ops or _key(At) in self.free_ops:
            return self._fail(ctx, L.ENOTSUP, "lsmr_chain: A and A' must be stored CSR matrices")
        if K > 1 and int(alg) not in (L.MGS, L.MGS2, L.CGS2, L.MGS2B):
            self.lsmr_enotsup += 1
            return self._fail(ctx, L.ENOTSUP, f"lsmr_chain: orthogonalizer {alg} does not chain with krylovdim > 1")
        if K > 1 and int(alg) in (L.CGS2, L.MGS2B) and R > PANEL_COLS[ctx.dtype]:
            self.lsmr_enotsup += 1
            return self._fail(ctx, L.ENOTSUP, "lsmr_chain: the ring does not fit the sweep's panel ring")
        m, n = M.shape
        if Mt.shape != (n, m):
            return self._fail(ctx, L.EDIM, "lsmr_chain: A' is not A's shape transposed")
        if any(len(self._vec(ctx, v)) != m or (v >> 20) != (mh[0] >> 20) for v in mh) or \
                any(len(self._vec(ctx, v)) != n or (v >> 20) != (nh[3] >> 20) for v in nh + rh):
            return self._fail(ctx, L.EDIM, "lsmr_chain: a vector has the wrong length or space")
        allh = mh + nh + rh
        if len(set(allh)) != len(allh):
            return self._fail(ctx, L.EINVAL, "lsmr_chain: two handles of one vector")
        self.lsmr_calls += 1
        T = ctx.dtype
        xv, hv, hbv, sv = (self._vec(ctx, v).copy() for v in nh)
        rv, ahv, ahbv, uv, _ = (self._vec(ctx, v).copy() for v in mh)
        rg = [self._vec(ctx, v).copy() for v in rh]
        st = [float(s) for s in _view(state_in, 10, np.ctypeslib.ctypes.c_double)]
        recs = _view(rec_out, 16 * nsteps, np.ctypeslib.ctypes.c_double).reshape(nsteps, 16)
        d = 0
        v = rg[iter0 % R]
        code = 0.0
        f64 = lambda a: a.astype(np.float64)  # noqa: E731
        for i in range(nsteps):
            k = iter0 + 1 + i
            ctx.launches += 4 + (0 if K <= 1 else 2)
            alpha, beta = st[0], st[1]
            tr = -st[7] / st[3]
            Avv = (M @ v).astype(T)
            ahv = Avv if tr == 0.0 else Avv + T(tr) * ahv
            ut = Avv + T(-alpha) * uv
            beta = float(np.sqrt(f64(ut) @ f64(ut)))
            bskip = not beta > tol
            if not bskip:
                uv = ut * T(1 / beta)
                vt = (Mt @ uv).astype(T) + T(-beta) * v
                if K > 1:
                    basis = rg[:min(int(K), k)]
                    passes = 2 if int(alg) != L.MGS else 1
                    for _ in range(passes):
                        if int(alg) in (L.MGS, L.MGS2):
                            for q in basis:
                                vt = vt - T(float(f64(q) @ f64(vt))) * q
                        else:
                            cs = [float(f64(q) @ f64(vt)) for q in basis]
                            for q, c in zip(basis, cs):
                                vt = vt - T(c) * q
                alpha = float(np.sqrt(f64(vt) @ f64(vt)))
                if alpha > tol:
                    v = vt * T(1 / alpha)
                    rg[k % R] = v
                else:
                    v = vt
                    sv = vt
            else:
                uv = ut
            st[1] = beta
            st, rec = lsmr_scalars(st, alpha, beta, bskip, tol)
            g, cz = rec[12], rec[13]
            hbv = hv if g == 0.0 else hv + T(g) * hbv
            ahbv = ahv if g == 0.0 else ahv + T(g) * ahbv
            xv = xv + T(cz) * hbv
            rv = rv + T(-cz) * ahbv
            tr = -st[7] / st[3]
            hv = v if tr == 0.0 else v + T(tr) * hv
            recs[i] = rec
            d = i + 1
            code = rec[7]
            if code != 0.0:
                break
        ctx.launches += 2
        self.lsmr_iters += d
        self.lsmr_codes.append(code)
        for hnd, arr in zip(nh, (xv, hv, hbv, sv)):
            self._setvec(ctx, hnd, arr)
        for hnd, arr in zip(mh[:4], (rv, ahv, ahbv, uv)):
            self._setvec(ctx, hnd, arr)
        for hnd, arr in zip(rh, rg):
            self._setvec(ctx, hnd, arr)
        _view(state_out, 10, np.ctypeslib.ctypes.c_double)[:] = st
        _set(done, d)
        return L.OK


class installed(hostsim_gkl.installed):
    """hostsim_gkl.installed, with the stand-in that also simulates b2k_lsmr_chain."""

    def __enter__(self):
        super().__enter__()
        L._lib = LsmrHostSimLib()
        return L._lib
