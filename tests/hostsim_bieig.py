"""TEST INFRASTRUCTURE ONLY — the numpy stand-in of tests/hostsim.py extended by the two entry points bieigsolve adds to
the C-ABI: b2k_basis_cross_inner (the cross Gram matrix of two column lists) and b2k_op_create_transpose (CSR of A' on
the device), with the library's refusals.  `installed()` routes `_lib.load()` to it like `hostsim.installed()` does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L

import hostsim
from hostsim import _key, _view


class BiHostSimLib(hostsim.HostSimLib):
    def __init__(self):
        super().__init__()
        self.cross_calls = 0        # calls of b2k_basis_cross_inner that got through the refusals

    def b2k_basis_cross_inner(self, h, X, p, Y, q, p0, q0, G, ldg):
        """G[i, j] = <X[i], Y[j]> outside the leading p0 x q0 block, float64 products here; nothing is written when a
        call is refused."""
        ctx = self._c(h)
        if X is None or Y is None or G is None:
            return self._fail(ctx, L.EINVAL, "basis_cross_inner: null pointer")
        if not (1 <= p <= 256 and 1 <= q <= 256 and 0 <= p0 <= p and 0 <= q0 <= q and ldg >= p):
            return self._fail(ctx, L.EINVAL, "basis_cross_inner: bad sizes")
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "basis_cross_inner: row-sharded contexts are not supported")
        Xs, Ys = self._cols(ctx, X, p), self._cols(ctx, Y, q)
        if len({len(v) for v in Xs + Ys}) != 1:
            return self._fail(ctx, L.EDIM, "basis_cross_inner: columns of different lengths")
        self.cross_calls += 1
        Gv = _view(G, ldg * (q - 1) + p, C.c_double)
        M = np.column_stack([x.astype(np.float64) for x in Xs]).T @ np.column_stack([y.astype(np.float64) for y in Ys])
        for j in range(q):
            for i in range(p):
                if not (i < p0 and j < q0):
                    Gv[j * ldg + i] = M[i, j]
        return L.OK

    def b2k_op_create_transpose(self, h, out, op):
        """A' of a CSR operator with sorted indices.  The stand-in stores a matrix-free stencil like the assembled one,
        so that refusal is not simulated."""
        ctx = self._c(h)
        A = self.ops[_key(op)]
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "op_create_transpose: row-sharded contexts are not supported")
        if not sp.issparse(A):
            return self._fail(ctx, L.ENOTSUP, "op_create_transpose: dense operator; use apply_adjoint")
        if not any(s.n == A.shape[1] for s in ctx.spaces):
            return self._fail(ctx, L.EDIM, "op_create_transpose: no vector space has the length of A' rows")
        T = A.T.tocsr()
        T.sort_indices()
        return self._newop(out, T)


class installed(hostsim.installed):
    """hostsim.installed, with the stand-in that also simulates the bieigsolve entry points."""

    def __enter__(self):
        super().__enter__()
        L._lib = BiHostSimLib()
        return L._lib
