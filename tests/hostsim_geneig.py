"""TEST INFRASTRUCTURE ONLY — the numpy stand-in of tests/hostsim_bieig.py extended by the pencil entry points geneigsolve
adds to the C-ABI (b2k_pencil_create / _destroy / _apply / _rayleigh) with the library's refusals, and the path hook
b2k_debug_pencil_path.  `installed()` routes `_lib.load()` to it like `hostsim_bieig.installed()` does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L

import hostsim_bieig
from hostsim import _key, _set


class GenHostSimLib(hostsim_bieig.BiHostSimLib):
    def __init__(self):
        super().__init__()
        self.pencils: dict[int, dict] = {}
        self.pencil_path = 0
        self.pencil_calls = {0: 0, 1: 0}       # pencil calls that passed their checks, by path

    def b2k_debug_pencil_path(self):
        return self.pencil_path

    def b2k_pencil_create(self, h, out, A, B):
        ctx = self._c(h)
        if out is None or A is None or B is None:
            return self._fail(ctx, L.EINVAL, "pencil_create: null pointer")
        ka, kb = _key(A), _key(B)
        if ka == kb:
            return self._fail(ctx, L.EINVAL, "pencil_create: A and B are the same operator")
        if ka not in self.ops or kb not in self.ops:
            return self._fail(ctx, L.EINVAL, "pencil_create: an operator of another context")
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "pencil_create: row-sharded contexts are not supported")
        Am, Bm = self.ops[ka], self.ops[kb]
        n = Am.shape[0]
        if Am.shape != (n, n) or Bm.shape != (n, n):
            return self._fail(ctx, L.EDIM, "pencil_create: A and B must be square of one size")
        fused = (sp.issparse(Am) and sp.issparse(Bm) and n > 0 and np.array_equal(Am.indptr, Bm.indptr)
                 and np.array_equal(Am.indices, Bm.indices))
        self.next_id += 1
        self.pencils[self.next_id] = dict(ctx=_key(h), A=ka, B=kb, n=n, fused=int(fused))
        _set(out, self.next_id)
        return L.OK

    def b2k_pencil_destroy(self, h, P):
        ctx = self._c(h)
        p = self.pencils.get(_key(P))
        if p is None or p["ctx"] != _key(h):
            return self._fail(ctx, L.EINVAL, "pencil_destroy: the pencil belongs to another context")
        del self.pencils[_key(P)]
        return L.OK

    def _check(self, h, P, vecs, who):
        """the library's checks, in its order; returns (status, pencil, arrays)"""
        ctx = self._c(h)
        p = self.pencils.get(_key(P)) if P is not None else None
        if p is None:
            return L.EINVAL, None, None
        if p["ctx"] != _key(h):
            return self._fail(ctx, L.EINVAL, f"{who}: the pencil belongs to another context"), None, None
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, f"{who}: row-sharded contexts are not supported"), None, None
        arrs = []
        for i, v in enumerate(vecs):
            if v is None:
                arrs.append(None)
                continue
            v = int(v)
            sp_, col = v >> 20, v & 0xFFFFF
            if v < 0 or sp_ >= len(ctx.spaces) or col not in ctx.spaces[sp_].cols:
                return self._fail(ctx, L.EINVAL, f"invalid vector handle {v:#x}"), None, None
            a = ctx.spaces[sp_].cols[col]
            if len(a) != p["n"]:
                return self._fail(ctx, L.EDIM, f"{who}: vector {i} has {len(a)} entries"), None, None
            for j, b in enumerate(arrs):
                if b is a:
                    return self._fail(ctx, L.EINVAL, f"{who}: vectors {j} and {i} are the same"), None, None
            arrs.append(a)
        return L.OK, p, arrs

    def b2k_pencil_apply(self, h, P, x, w, bx, rho, vprev, beta, dot):
        st, p, (a) = self._check(h, P, [x, w, bx, None if int(vprev) < 0 else vprev], "pencil_apply")
        if st != L.OK:
            return st
        ctx = self._c(h)
        xv, wv, bxv, vp = a
        self.pencil_path = p["fused"]
        self.pencil_calls[p["fused"]] += 1
        ctx.launches += 1 if p["fused"] else (3 + (vp is not None) + (dot is not None))
        dt = ctx.dtype
        Bx = (self.ops[p["B"]] @ xv).astype(dt)
        W = (self.ops[p["A"]] @ xv).astype(dt) + dt(-rho) * Bx
        if vp is not None:
            W = W + dt(-beta) * vp
        bxv[:] = Bx
        wv[:] = W
        if dot is not None:
            _set(dot, float(np.dot(xv.astype(np.float64), wv.astype(np.float64))))
        return L.OK

    def b2k_pencil_rayleigh(self, h, P, x, ax, bx, xax, xbx):
        st, p, a = self._check(h, P, [x, ax, bx], "pencil_rayleigh")
        if st != L.OK:
            return st
        ctx = self._c(h)
        xv, axv, bxv = a
        self.pencil_path = p["fused"]
        self.pencil_calls[p["fused"]] += 1
        ctx.launches += 1 if p["fused"] else (2 + (xax is not None) + (xbx is not None))
        axv[:] = self.ops[p["A"]] @ xv
        bxv[:] = self.ops[p["B"]] @ xv
        x64 = xv.astype(np.float64)
        if xax is not None:
            _set(xax, float(np.dot(x64, axv.astype(np.float64))))
        if xbx is not None:
            _set(xbx, float(np.dot(x64, bxv.astype(np.float64))))
        return L.OK


class installed(hostsim_bieig.installed):
    """hostsim_bieig.installed, with the stand-in that also simulates the pencil entry points."""

    def __enter__(self):
        super().__enter__()
        L._lib = GenHostSimLib()
        return L._lib
