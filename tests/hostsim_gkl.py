"""TEST INFRASTRUCTURE ONLY — the numpy stand-in of tests/hostsim_bieig.py extended by the entry point the sparse
svdsolve adds to the C-ABI, b2k_gkl_expand_many, with the library's refusals and handle contract (new U / V columns
allocated by the library, the residual passed in released once a step is committed).  Matrix-free stencils are
marked as such (b2k_op_info reports kind 2, b2k_op_create_transpose refuses them), so the front end's refusal of
them can be exercised.  `installed()` routes `_lib.load()` to it like `hostsim.installed()`.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko

import hostsim_bieig
from hostsim import _key, _set

MAX_CHAIN = 512
CHAIN_COLS = {np.float64: 96, np.float32: 192}      # the sweep's panel ring (include/b200krylov.h)


class GklHostSimLib(hostsim_bieig.BiHostSimLib):
    def __init__(self):
        super().__init__()
        self.gkl_calls = 0          # calls of b2k_gkl_expand_many that got through the refusals
        self.gkl_steps = 0          # steps those calls committed
        self.free_ops: set[int] = set()

    def b2k_op_create_stencil_free(self, h, out, nx, ny, nz, c):
        st = self.b2k_op_create_stencil(h, out, nx, ny, nz, c)
        self.free_ops.add(_key(out._obj if hasattr(out, "_obj") else out))
        return st

    def b2k_op_info(self, op, nr, nc, nnz, kind):
        st = super().b2k_op_info(op, nr, nc, nnz, kind)
        if _key(op) in self.free_ops:
            _set(kind, 2)
        return st

    def b2k_op_create_transpose(self, h, out, op):
        if _key(op) in self.free_ops:
            return self._fail(self._c(h), L.ENOTSUP, "op_create_transpose: a matrix-free stencil has no transpose")
        return super().b2k_op_create_transpose(h, out, op)

    def _space_of(self, ctx, handles_, n):
        """The one space all handles live in, if it has length n and every handle is live; else None."""
        spaces = set()
        for v in handles_:
            v = int(v)
            s = v >> 20
            if v < 0 or s >= len(ctx.spaces) or (v & 0xFFFFF) not in ctx.spaces[s].cols:
                return None
            spaces.add(s)
        if len(spaces) != 1:
            return None
        s = spaces.pop()
        return s if ctx.spaces[s].n == n else None

    def b2k_gkl_expand_many(self, h, A, At, ucols, vcols, k, nsteps, beta_old, tol, alg, alphas, betas, done, r_out):
        ctx = self._c(h)
        if A is None or At is None or ucols is None or vcols is None or alphas is None or betas is None:
            return self._fail(ctx, L.EINVAL, "gkl_expand_many: null pointer")
        if k < 1 or nsteps < 1 or nsteps > MAX_CHAIN:
            return self._fail(ctx, L.EINVAL, "gkl_expand_many: need k >= 1 and 1 <= nsteps <= 512")
        if not (beta_old > 0.0) or not math.isfinite(beta_old):
            return self._fail(ctx, L.EINVAL, "gkl_expand_many: beta_old must be positive and finite")
        if int(alg) not in (L.CGS2, L.MGS2B):
            return self._fail(ctx, L.ENOTSUP, "gkl_expand_many: ClassicalGramSchmidt2 / ModifiedGramSchmidt2Blocked only")
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "gkl_expand_many: row-sharded contexts are not supported")
        M, Mt = self.ops[_key(A)], self.ops[_key(At)]
        if not (sp.issparse(M) and sp.issparse(Mt)) or _key(A) in self.free_ops or _key(At) in self.free_ops:
            return self._fail(ctx, L.ENOTSUP, "gkl_expand_many: A and A' must be stored CSR matrices")
        m, n = M.shape
        if Mt.shape != (n, m):
            return self._fail(ctx, L.EDIM, "gkl_expand_many: A' is not A's shape transposed")
        su = self._space_of(ctx, list(ucols)[:k + 1], m)
        sv = self._space_of(ctx, list(vcols)[:k], n)
        if su is None or sv is None:
            return self._fail(ctx, L.EDIM, "gkl_expand_many: U, r (length m) and V (length n) must each be columns "
                                           "of one space")
        if k + nsteps > CHAIN_COLS[ctx.dtype]:
            return self._fail(ctx, L.ENOTSUP, "gkl_expand_many: too many columns for the sweep's panel ring")
        self.gkl_calls += 1
        T = ctx.dtype
        U = [self._vec(ctx, c) for c in list(ucols)[:k]]
        V = [self._vec(ctx, c) for c in list(vcols)[:k]]
        r0 = int(ucols[k])
        r = self._vec(ctx, r0)
        beta = float(beta_old)
        d = 0
        out_r = r0
        err = L.OK
        for i in range(nsteps):
            ctx.launches += 4 if int(alg) == L.MGS2B else 3
            uc, vc, wc = self._alloc(ctx, su), self._alloc(ctx, sv), self._alloc(ctx, su)
            if uc is None or vc is None or wc is None:
                for c in (uc, vc, wc):
                    if c is not None:
                        self.b2k_vec_free(h, c)
                err = self._fail(ctx, L.ENOMEM, "gkl_expand_many: no free column left")
                break
            # gklrecurrence (gkl.jl:308-323) as the oracle rounds it, with the chain's orthogonalisation
            u = r * T(1 / beta)
            v = Mt @ u
            v = v - T(beta) * V[-1]
            if int(alg) == L.MGS2B:
                v, _ = ko._cgs_pass(v, V, np.empty(len(V)))
            alpha = ko.norm(v)
            v = v * T(1 / alpha)
            rn = M @ v
            rn = rn - T(alpha) * u
            rn, _ = ko._cgs_pass(rn, U + [u], np.empty(len(U) + 1))
            beta = ko.norm(rn)
            self._setvec(ctx, uc, u)
            self._setvec(ctx, vc, v)
            self._setvec(ctx, wc, rn)
            U.append(self._vec(ctx, uc))
            V.append(self._vec(ctx, vc))
            ucols[k + i], vcols[k + i], ucols[k + i + 1] = uc, vc, wc
            if i > 0:
                self.b2k_vec_free(h, out_r)               # the previous residual's column goes back to the slab
            out_r, r = wc, self._vec(ctx, wc)
            alphas[i] = alpha
            betas[i] = beta if math.isfinite(alpha) else math.nan
            d = i + 1
            if not (math.isfinite(alpha) and math.isfinite(beta)) or beta <= tol:
                break
        ctx.launches += 1                                  # the flush
        if d > 0:
            self.b2k_vec_free(h, r0)
            self.gkl_steps += d
        _set(done, d)
        _set(r_out, out_r)
        return err

    def _alloc(self, ctx, space):
        c0 = ctx.spaces[space].alloc(1, ctx.dtype)
        return None if c0 < 0 else (space << 20) | c0


class installed(hostsim_bieig.installed):
    """hostsim_bieig.installed, with the stand-in that also simulates b2k_gkl_expand_many."""

    def __enter__(self):
        super().__enter__()
        L._lib = GklHostSimLib()
        return L._lib

