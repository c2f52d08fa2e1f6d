"""TEST INFRASTRUCTURE ONLY — a numpy stand-in for libb200krylov's C-ABI, so the host-side driver
logic of krylovkit.jl_b200 (restart bookkeeping, Schur reordering, step-size control, handle
lifetimes, column budgets) can be exercised by `pytest -m "not gpu"` in a container without a GPU.

It is never importable from the package, ships nothing, and measures nothing: the product still
loads the CUDA library or raises.  `install()` swaps the object `_lib.load()` returns for the
duration of a test; semantics follow include/b200krylov.h entry by entry, the arithmetic is the
oracle's (tests may use the oracle).  The fused entry points (b2k_lanczos_expand[_many],
b2k_cg_step, b2k_bicgstab_half/_full) are simulated as well; `installed(fused=False)` switches the
drivers to their literal VectorInterface paths, `installed(fused=True)` exercises the fused branches'
host-side bookkeeping (handle accounting of expand_many, the two-call BiCGStab flow).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from krylovkit_jl_b200 import _lib as L
from oracle import krylov_oracle as ko


def _set(ref, val):
    obj = getattr(ref, "_obj", ref)
    if hasattr(obj, "value"):
        obj.value = val
    else:
        obj[0] = val


def _view(ptr, n, ctype):
    """numpy view (writes go through) of n elements behind an address / ctypes pointer / array."""
    if n == 0:
        return np.zeros(0, dtype=np.ctypeslib.as_array((ctype * 1)()).dtype)
    if isinstance(ptr, (int, np.integer)):
        return np.ctypeslib.as_array((ctype * n).from_address(int(ptr)))
    if isinstance(ptr, C.Array):
        return np.ctypeslib.as_array(ptr)[:n]
    if hasattr(ptr, "contents"):
        return np.ctypeslib.as_array(ptr, shape=(n,))
    obj = getattr(ptr, "_obj", None)
    if obj is not None:
        return _view(C.addressof(obj), n, ctype)
    raise TypeError(f"hostsim: cannot view {type(ptr)}")


def _key(h):
    return h.value if hasattr(h, "value") else h


class _Space:
    def __init__(self, n, ncols):
        self.n, self.ncols = int(n), int(ncols)
        self.cols: dict[int, np.ndarray] = {}

    def alloc(self, count, dtype):
        for c0 in range(self.ncols - count + 1):
            if all((c0 + i) not in self.cols for i in range(count)):
                for i in range(count):
                    self.cols[c0 + i] = np.zeros(self.n, dtype=dtype)
                return c0
        return -1


class _Ctx:
    def __init__(self, n, ncols, dtype, dist=None):
        self.dtype = np.float64 if dtype == L.F64 else np.float32
        self.ctype = C.c_double if dtype == L.F64 else C.c_float
        self.spaces = [_Space(n, ncols)]
        self.sharded = [True]
        self.err = b""
        self.launches = 0
        self.dist = dist            # None, or dict(rank, nranks, n_global, row_offset): rows sharded over ranks

    def allsum(self, v, sharded=True):
        """The library's all-reduce of scalars / coefficient vectors (NCCL there, gloo here)."""
        a = np.atleast_1d(np.asarray(v, dtype=np.float64)).copy()
        if self.dist is not None and sharded:
            import torch
            import torch.distributed as tdist
            t = torch.from_numpy(a)
            tdist.all_reduce(t)
            a = t.numpy()
        return a

    def gather_rows(self, x):
        """x over all ranks, in rank order (what the halo exchange provides to the local rows)."""
        if self.dist is None:
            return x
        import torch.distributed as tdist
        parts = [None] * self.dist["nranks"]
        tdist.all_gather_object(parts, np.asarray(x))
        return np.concatenate(parts)


class _global_reductions:
    """While active, the oracle's inner / norm see GLOBAL sums — so that its orthogonalisation and block
    routines, run on the local rows by every rank, behave like the library's sharded kernels."""

    def __init__(self, ctx: _Ctx, sharded=True):
        self.ctx, self.on = ctx, ctx.dist is not None and sharded

    def __enter__(self):
        if self.on:
            self.saved = (ko.inner, ko.norm)
            ctx = self.ctx
            ko.inner = lambda x, y: float(ctx.allsum(np.dot(np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)))[0])
            ko.norm = lambda x: float(np.sqrt(ctx.allsum(np.dot(np.asarray(x, dtype=np.float64), np.asarray(x, dtype=np.float64)))[0]))
        return self

    def __exit__(self, *exc):
        if self.on:
            ko.inner, ko.norm = self.saved
        return False


class HostSimLib:
    def __init__(self):
        self.ctxs: dict[int, _Ctx] = {}
        self.ops: dict[int, object] = {}
        self.next_id = 1000
        self.err = b""
        self.chain = True          # b2k_lanczos_expand_many follows the device-chained handle contract (CGS2)

    def b2k_debug_used_columns(self, h, space):
        return len(self._c(h).spaces[space].cols)

    def b2k_debug_set_onepass_variant(self, v):
        return L.OK if v in (0, 1) else L.EINVAL            # one numpy product stands for both kernels

    def b2k_debug_set_transform(self, mode):
        return L.OK

    def b2k_debug_set_chain(self, on):
        self.chain = bool(on)
        return L.OK

    # ---- plumbing ---------------------------------------------------------------------------
    def _fail(self, ctx, code, msg):
        (ctx if ctx is not None else self).err = msg.encode()
        return code

    def _c(self, h) -> _Ctx:
        return self.ctxs[_key(h)]

    def _vec(self, ctx: _Ctx, v) -> np.ndarray:
        v = int(v)
        return ctx.spaces[v >> 20].cols[v & 0xFFFFF]

    def _setvec(self, ctx: _Ctx, v, arr):
        v = int(v)
        ctx.spaces[v >> 20].cols[v & 0xFFFFF][:] = arr

    def _sh(self, ctx, v):
        return ctx.sharded[int(v) >> 20]

    def _cols(self, ctx, cols, k):
        return [self._vec(ctx, c) for c in list(cols)[:k]]

    def b2k_abi_version(self):
        return 1

    def b2k_last_error(self, h):
        k = _key(h) if h is not None else None
        return (self.ctxs[k].err if k in self.ctxs else self.err) or b""

    def b2k_ctx_create(self, out, device, n_local, ncols, dtype):
        if n_local < 1 or ncols < 1:
            return self._fail(None, L.EINVAL, "ctx_create: bad shape")
        self.next_id += 1
        self.ctxs[self.next_id] = _Ctx(n_local, ncols, dtype)
        _set(out, self.next_id)
        return L.OK

    def b2k_nccl_unique_id(self, buf):
        return L.OK

    def b2k_ctx_create_dist(self, out, device, n_local, ncols, dtype, rank, nranks, uid, n_global, row_offset):
        self.next_id += 1
        self.ctxs[self.next_id] = _Ctx(n_local, ncols, dtype, dict(rank=int(rank), nranks=int(nranks),
                                                                   n_global=int(n_global), row_offset=int(row_offset)))
        _set(out, self.next_id)
        return L.OK

    def b2k_ctx_destroy(self, h):
        self.ctxs.pop(_key(h), None)
        return L.OK

    def b2k_space_create(self, h, n_local, ncols, sharded, out):
        ctx = self._c(h)
        ctx.spaces.append(_Space(n_local, ncols))
        ctx.sharded.append(bool(sharded))
        _set(out, len(ctx.spaces) - 1)
        return L.OK

    def b2k_ctx_sync(self, h):
        return L.OK

    def b2k_ctx_launch_count(self, h):
        return self._c(h).launches

    def b2k_ctx_stream(self, h):
        return None

    def b2k_device_sync(self):
        return L.OK

    # "pinned" host buffers: plain host memory, kept alive until freed
    def b2k_pinned_alloc(self, nbytes, out):
        buf = (C.c_byte * max(1, int(nbytes)))()
        if not hasattr(self, "_pinned"):
            self._pinned = {}
        self._pinned[C.addressof(buf)] = buf
        _set(out, C.addressof(buf))
        return L.OK

    def b2k_pinned_free(self, p):
        getattr(self, "_pinned", {}).pop(_key(p), None)
        return L.OK

    def b2k_cache_release(self):
        return L.OK

    def b2k_timer_start(self, h):
        import time
        self._c(h).t0 = time.perf_counter()
        return L.OK

    def b2k_timer_stop(self, h, ms):
        import time
        _set(ms, (time.perf_counter() - self._c(h).t0) * 1e3)
        return L.OK

    # the per-kernel event profile has no meaning here: accepted, always empty
    def b2k_prof_enable(self, h, on):
        return L.OK

    def b2k_prof_reset(self, h):
        return L.OK

    def b2k_prof_read(self, h, cls, count, ms, nbytes):
        _set(count, 0)
        _set(ms, 0.0)
        _set(nbytes, 0.0)
        return L.OK

    # ---- vectors ------------------------------------------------------------------------------
    def b2k_vec_alloc(self, h, space, out):
        return self.b2k_vec_alloc_range(h, space, 1, out)

    def b2k_vec_alloc_range(self, h, space, count, out):
        ctx = self._c(h)
        c0 = ctx.spaces[space].alloc(count, ctx.dtype)
        if c0 < 0:
            return self._fail(ctx, L.ENOMEM, f"vec_alloc: no {count} free column(s) left in space {space} "
                                              f"({ctx.spaces[space].ncols} columns)")
        _set(out, (space << 20) | c0)
        return L.OK

    def b2k_vec_free(self, h, v):
        ctx = self.ctxs.get(_key(h))
        if ctx is not None:
            ctx.spaces[int(v) >> 20].cols.pop(int(v) & 0xFFFFF, None)
        return L.OK

    def b2k_vec_upload(self, h, v, host):
        ctx = self._c(h)
        x = self._vec(ctx, v)
        x[:] = _view(host, len(x), ctx.ctype)
        return L.OK

    def b2k_vec_download(self, h, v, host):
        ctx = self._c(h)
        x = self._vec(ctx, v)
        _view(host, len(x), ctx.ctype)[:] = x
        return L.OK

    def b2k_vec_copy(self, h, dst, src):
        ctx = self._c(h)
        if len(self._vec(ctx, dst)) != len(self._vec(ctx, src)):
            return self._fail(ctx, L.EDIM, "vec_copy: length mismatch")
        self._setvec(ctx, dst, self._vec(ctx, src))
        return L.OK

    def b2k_vec_zero(self, h, v):
        self._setvec(self._c(h), v, 0.0)
        return L.OK

    def b2k_vec_fill(self, h, v, value):
        self._setvec(self._c(h), v, value)
        return L.OK

    def b2k_vec_fill_splitmix(self, h, v, seed):
        ctx = self._c(h)
        off = ctx.dist["row_offset"] if (ctx.dist and self._sh(ctx, v)) else 0
        self._setvec(ctx, v, ko.splitmix_vector(int(seed), len(self._vec(ctx, v)), offset=off))
        return L.OK

    def b2k_vec_inner(self, h, x, y, out):
        ctx = self._c(h)
        a, b = self._vec(ctx, x), self._vec(ctx, y)
        if len(a) != len(b):
            return self._fail(ctx, L.EDIM, "inner: length mismatch")
        _set(out, float(ctx.allsum(np.dot(a.astype(np.float64), b.astype(np.float64)), self._sh(ctx, x))[0]))
        return L.OK

    def b2k_vec_norm(self, h, x, out):
        ctx = self._c(h)
        a = self._vec(ctx, x).astype(np.float64)
        _set(out, float(np.sqrt(ctx.allsum(np.dot(a, a), self._sh(ctx, x))[0])))
        return L.OK

    def b2k_vec_axpby(self, h, y, x, alpha, beta):
        ctx = self._c(h)
        a, b = self._vec(ctx, y), self._vec(ctx, x)
        if len(a) != len(b):
            return self._fail(ctx, L.EDIM, "axpby: length mismatch")
        self._setvec(ctx, y, (beta * a if beta != 0 else 0.0) + alpha * b)
        return L.OK

    def b2k_vec_scale(self, h, y, x, alpha):
        ctx = self._c(h)
        self._setvec(ctx, y, alpha * self._vec(ctx, x))
        return L.OK

    def b2k_vec_axpy2(self, h, y, x1, a1, x2, a2):
        ctx = self._c(h)
        self._setvec(ctx, y, self._vec(ctx, y) + a1 * self._vec(ctx, x1) + a2 * self._vec(ctx, x2))
        return L.OK

    # ---- operators ----------------------------------------------------------------------------
    def _newop(self, out, obj):
        self.next_id += 1
        self.ops[self.next_id] = obj
        _set(out, self.next_id)
        return L.OK

    def _index_shape(self, ctx, who, idx_bytes, index_base, n_rows, n_cols, nnz):
        """the library's refusals of an index-array operator, in its order, before any array is read"""
        if idx_bytes not in (4, 8) or index_base not in (0, 1):
            return self._fail(ctx, L.EINVAL, f"{who}: idx_bytes must be 4/8, index_base 0/1")
        if min(n_rows, n_cols, nnz) < 0:
            return self._fail(ctx, L.EINVAL, f"{who}: negative size")
        if max(n_rows, nnz) >= 1 << 31:
            return self._fail(ctx, L.ENOTSUP, f"{who}: rows and nnz per GPU must be < 2^31")
        if ctx.dist is None and n_cols >= 1 << 31:        # a row shard's n_cols is the global column count
            return self._fail(ctx, L.ENOTSUP, f"{who}: columns on one GPU must be < 2^31")
        if n_rows != ctx.spaces[0].n and (ctx.dist is not None or not any(s.n == n_rows for s in ctx.spaces)):
            return self._fail(ctx, L.EDIM, f"{who}: {n_rows} local rows but space 0 holds {ctx.spaces[0].n}")
        return L.OK

    @staticmethod
    def _ptr_ok(p, count):
        """p (int64, base removed) runs from 0 to count, never decreasing"""
        return p[0] == 0 and p[-1] == count and bool(np.all(np.diff(p) >= 0))

    def b2k_op_create_csr(self, h, out, n_rows, n_cols, nnz, rowptr, colidx, vals, idx_bytes, index_base):
        ctx = self._c(h)
        st = self._index_shape(ctx, "op_create_csr", idx_bytes, index_base, n_rows, n_cols, nnz)
        if st != L.OK:
            return st
        it = C.c_int64 if idx_bytes == 8 else C.c_int32
        rp = np.array(_view(rowptr, n_rows + 1, it), dtype=np.int64) - index_base
        if not self._ptr_ok(rp, nnz):
            return self._fail(ctx, L.EINVAL, "op_create_csr: rowptr does not rise from 0 to nnz")
        ci = np.array(_view(colidx, nnz, it), dtype=np.int64) - index_base
        if ctx.dist is not None:                      # local rows, GLOBAL column indices
            n_cols = ctx.dist["n_global"]
        if nnz > 0 and (ci.min() < 0 or ci.max() >= n_cols):
            return self._fail(ctx, L.EINVAL, f"op_create_csr: column index out of range [0, {n_cols})")
        va = np.array(_view(vals, nnz, ctx.ctype))
        return self._newop(out, sp.csr_matrix((va, ci, rp), shape=(n_rows, n_cols)))

    def b2k_op_create_csc(self, h, out, n_rows, n_cols, nnz, colptr, rowval, nzval, idx_bytes, index_base):
        ctx = self._c(h)
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "op_create_csc: single-GPU contexts only")
        st = self._index_shape(ctx, "op_create_csc", idx_bytes, index_base, n_rows, n_cols, nnz)
        if st != L.OK:
            return st
        it = C.c_int64 if idx_bytes == 8 else C.c_int32
        cp = np.array(_view(colptr, n_cols + 1, it), dtype=np.int64) - index_base
        if not self._ptr_ok(cp, nnz):
            return self._fail(ctx, L.EINVAL, "op_create_csc: colptr does not rise from 0 to nnz")
        rv = np.array(_view(rowval, nnz, it), dtype=np.int64) - index_base
        if nnz > 0 and (rv.min() < 0 or rv.max() >= n_rows):
            return self._fail(ctx, L.EINVAL, "op_create_csc: row index out of range")
        nz = np.array(_view(nzval, nnz, ctx.ctype))
        return self._newop(out, sp.csc_matrix((nz, rv, cp), shape=(n_rows, n_cols)).tocsr())

    def b2k_op_create_stencil(self, h, out, nx, ny, nz, c):
        ctx = self._c(h)
        if min(nx, ny, nz) < 1:
            return self._fail(ctx, L.EINVAL, "stencil: bad grid")
        nglob = ctx.dist["n_global"] if ctx.dist is not None else ctx.spaces[0].n
        if nx * ny * nz != nglob:
            return self._fail(ctx, L.EDIM, f"stencil: grid has {nx * ny * nz} points, the operator needs {nglob}")
        A = ko.stencil_matrix(nx, ny, nz, tuple(float(c[i]) for i in range(7)), dtype=ctx.dtype)
        if ctx.dist is not None:                      # this rank's rows of the global operator
            r0 = ctx.dist["row_offset"]
            A = A[r0:r0 + ctx.spaces[0].n].tocsr()
        return self._newop(out, A)

    def b2k_op_create_dense(self, h, out, m, n, host, ld):
        ctx = self._c(h)
        if ld < m or m < 1 or n < 1:
            return self._fail(ctx, L.EINVAL, "dense: bad shape")
        if m != ctx.spaces[0].n:
            return self._fail(ctx, L.EDIM, f"dense: {m} local rows but space 0 holds {ctx.spaces[0].n}")
        A = np.array(_view(host, ld * n, ctx.ctype)).reshape(n, ld).T[:m, :]
        return self._newop(out, np.array(A))

    def b2k_op_create_dense_splitmix(self, h, out, m, n, seed):
        ctx = self._c(h)
        return self._newop(out, ko.dense_splitmix(int(seed), m, n, dtype=ctx.dtype))

    def b2k_op_destroy(self, h, op):
        self.ops.pop(_key(op), None)
        return L.OK

    def b2k_op_info(self, op, nr, nc, nnz, kind):
        A = self.ops[_key(op)]
        _set(nr, A.shape[0])
        _set(nc, A.shape[1])
        _set(nnz, A.nnz if sp.issparse(A) else A.size)
        _set(kind, 0 if sp.issparse(A) else 1)
        return L.OK

    def b2k_op_csr_download(self, h, op, rowptr, colidx, vals):
        ctx = self._c(h)
        A = self.ops[_key(op)]
        _view(rowptr, A.shape[0] + 1, C.c_int32)[:] = A.indptr
        _view(colidx, A.nnz, C.c_int32)[:] = A.indices
        _view(vals, A.nnz, ctx.ctype)[:] = A.data
        return L.OK

    def _apply(self, ctx, op, x, y, a0=0.0, a1=1.0, adjoint=False):
        A = self.ops[_key(op)]
        xv, yv = self._vec(ctx, x), self._vec(ctx, y)
        M = A.T if adjoint else A
        if ctx.dist is not None:
            if not sp.issparse(A) or adjoint:
                return self._fail(ctx, L.ENOTSUP, "hostsim: only sharded CSR operators are simulated")
            xg = ctx.gather_rows(xv)                  # stands for the halo exchange
            if M.shape[1] != len(xg) or M.shape[0] != len(yv):
                return self._fail(ctx, L.EDIM, "apply: shard / operator mismatch")
            ctx.launches += 1
            r = M @ xg
            self._setvec(ctx, y, a1 * r + a0 * xv if (a0 != 0 or a1 != 1) else r)
            return L.OK
        if M.shape[1] != len(xv) or M.shape[0] != len(yv):
            return self._fail(ctx, L.EDIM, f"apply: x has {len(xv)} entries, operator wants {M.shape[1]}")
        ctx.launches += 1
        r = M @ xv
        self._setvec(ctx, y, a1 * r + a0 * xv if (a0 != 0 or a1 != 1) else r)
        return L.OK

    def b2k_op_apply(self, h, op, x, y):
        return self._apply(self._c(h), op, x, y)

    def b2k_op_apply_shifted(self, h, op, x, y, a0, a1):
        return self._apply(self._c(h), op, x, y, a0, a1)

    def b2k_op_apply_adjoint(self, h, op, x, y):
        ctx = self._c(h)
        if sp.issparse(self.ops[_key(op)]):
            return self._fail(ctx, L.ENOTSUP, "apply_adjoint on a CSR operator")
        return self._apply(ctx, op, x, y, adjoint=True)

    def b2k_op_apply_normal_gram(self, h, op, x, y, z):
        """y = A x and z = A'(A x): one pass over a dense A on the device, two numpy products here (working
        precision, like the kernel's per-tile sums)."""
        ctx = self._c(h)
        A = self.ops[_key(op)]
        if sp.issparse(A):
            return self._fail(ctx, L.ENOTSUP, "apply_normal_gram: dense operators only")
        if ctx.dist is not None:
            return self._fail(ctx, L.ENOTSUP, "hostsim: only sharded CSR operators are simulated")
        xv, yv, zv = self._vec(ctx, x), self._vec(ctx, y), self._vec(ctx, z)
        if A.shape[1] != len(xv) or A.shape[1] != len(zv) or A.shape[0] != len(yv):
            return self._fail(ctx, L.EDIM, "apply_normal_gram: length mismatch")
        if len({_key(x), _key(y), _key(z)}) < 3:
            return self._fail(ctx, L.EINVAL, "apply_normal_gram: x, y and z must be three different vectors")
        ctx.launches += 2
        r = A @ xv
        self._setvec(ctx, y, r)
        self._setvec(ctx, z, A.T @ r)
        return L.OK

    def b2k_op_apply_dot(self, h, op, x, y, v, out):
        ctx = self._c(h)
        st = self._apply(ctx, op, x, y)
        if st == L.OK:
            d = np.dot(self._vec(ctx, v).astype(np.float64), self._vec(ctx, y).astype(np.float64))
            _set(out, float(ctx.allsum(d, self._sh(ctx, y))[0]))
        return st

    # ---- basis ----------------------------------------------------------------------------------
    def b2k_basis_project(self, h, cols, k, x, alpha, beta, hptr):
        ctx = self._c(h)
        hv = _view(hptr, k, C.c_double)
        xv = self._vec(ctx, x).astype(np.float64)
        dots = np.zeros(k)
        for j, q in enumerate(self._cols(ctx, cols, k)):
            if len(q) != len(xv):
                return self._fail(ctx, L.EDIM, "project: length mismatch")
            dots[j] = float(np.dot(q.astype(np.float64), xv))
        dots = ctx.allsum(dots, self._sh(ctx, x))
        for j in range(k):
            hv[j] = (beta * hv[j] if beta != 0 else 0.0) + alpha * dots[j]
        ctx.launches += 1
        return L.OK

    def b2k_basis_unproject(self, h, y, cols, k, c, alpha, beta):
        ctx = self._c(h)
        cv = _view(c, k, C.c_double)
        yv = self._vec(ctx, y)
        acc = beta * yv.astype(np.float64) if beta != 0 else np.zeros(len(yv))
        for j, q in enumerate(self._cols(ctx, cols, k)):
            if len(q) != len(yv):
                return self._fail(ctx, L.EDIM, "unproject: length mismatch")
            acc = acc + (alpha * cv[j]) * q
        self._setvec(ctx, y, acc)
        ctx.launches += 1
        return L.OK

    def b2k_basis_orthogonalize(self, h, v, cols, k, hptr, alg, eta, nrm, passes):
        ctx = self._c(h)
        hv = _view(hptr, k, C.c_double)
        b = [q.astype(np.float64) for q in self._cols(ctx, cols, k)]
        x = np.zeros(k)
        oalg = ko.CGS2 if int(alg) == L.MGS2B else int(alg)        # blocked MGS2: both sweeps classical
        with _global_reductions(ctx, self._sh(ctx, v)):
            w, x = ko.orthogonalize(self._vec(ctx, v).astype(np.float64), b, x, ko.Orth(oalg, float(eta)))
            nw = ko.norm(w)
        self._setvec(ctx, v, w)
        hv[:] = x
        _set(nrm, float(nw))
        if passes is not None:
            _set(passes, 1)
        ctx.launches += 1
        return L.OK

    def b2k_vec_orthogonalize(self, h, v, q, alg, eta, s, nrm):
        ctx = self._c(h)
        oalg = ko.MGS2 if int(alg) == L.MGS2B else int(alg)
        with _global_reductions(ctx, self._sh(ctx, v)):
            w, sv = ko.orthogonalize_vec(self._vec(ctx, v).astype(np.float64), self._vec(ctx, q).astype(np.float64),
                                         ko.Orth(oalg, float(eta)), eps=float(np.finfo(ctx.dtype).eps))
            nw = ko.norm(w)
        self._setvec(ctx, v, w)
        _set(s, float(sv))
        _set(nrm, float(nw))
        return L.OK

    def b2k_basis_transform(self, h, cols, m, U, ldu, keep):
        ctx = self._c(h)
        if m < 1 or keep < 1 or keep > m or ldu < m:
            return L.EINVAL
        hs = [int(c) for c in list(cols)[:m]]
        for c in hs:
            if c < 0 or (c >> 20) >= len(ctx.spaces) or (c & 0xFFFFF) not in ctx.spaces[c >> 20].cols:
                return self._fail(ctx, L.EINVAL, f"invalid vector handle {c:#x}")
        if len({c >> 20 for c in hs}) > 1:
            return self._fail(ctx, L.EDIM, "basis vectors live in different spaces")
        if len(set(hs)) < m:
            return self._fail(ctx, L.EINVAL, "basis_transform: a column is listed twice")
        if m > 256:
            return self._fail(ctx, L.ENOTSUP, "basis_transform: m exceeds the supported basis width (256)")
        Um = np.array(_view(U, ldu * keep, C.c_double)).reshape(keep, ldu).T[:m, :]
        Q = np.column_stack([q.astype(np.float64) for q in self._cols(ctx, cols, m)])
        R = Q @ Um
        for j in range(keep):
            self._setvec(ctx, list(cols)[j], R[:, j])
        ctx.launches += 1
        return L.OK

    def b2k_basis_rank1update(self, h, cols, k, y, x, alpha, beta):
        ctx = self._c(h)
        xv = _view(x, k, C.c_double)
        yv = self._vec(ctx, y).astype(np.float64)
        for i, c in enumerate(list(cols)[:k]):
            self._setvec(ctx, c, beta * self._vec(ctx, c) + (alpha * xv[i]) * yv)
        return L.OK

    def b2k_basis_givens(self, h, q1, q2, c, s):
        ctx = self._c(h)
        a, b = self._vec(ctx, q1).copy(), self._vec(ctx, q2).copy()
        self._setvec(ctx, q1, c * a - s * b)
        self._setvec(ctx, q2, s * a + c * b)
        return L.OK

    def b2k_basis_householder(self, h, cols, k, v, beta, work):
        ctx = self._c(h)
        vv = _view(v, k, C.c_double)
        qs = self._cols(ctx, cols, k)
        w = sum(vv[i] * qs[i].astype(np.float64) for i in range(k))
        for i, c in enumerate(list(cols)[:k]):
            self._setvec(ctx, c, self._vec(ctx, c) - (beta * vv[i]) * w)
        return L.OK

    # ---- fused steps: same arithmetic as the literal sequences, one call -------------------------------
    class _OpView:
        """The operator as the oracle's `apply` sees it: local rows times the gathered vector."""

        def __init__(self, ctx, A):
            self.ctx, self.A = ctx, A

        def __matmul__(self, x):
            return self.A @ self.ctx.gather_rows(x)

    def b2k_lanczos_expand(self, h, op, cols, k, r, w, beta_old, alg, eta, alpha_out, beta_out):
        ctx = self._c(h)
        cl = list(cols)[:k + 1]
        if int(cl[k]) != int(r):
            return self._fail(ctx, L.EINVAL, "lanczos_expand: cols[k] must be r")
        if beta_old == 0.0:
            return self._fail(ctx, L.EINVAL, "lanczos_expand: beta_old == 0")
        self._setvec(ctx, r, self._vec(ctx, r) * (1.0 / beta_old))      # lanczos.jl:257
        V = [self._vec(ctx, c).astype(np.float64) for c in cl]
        with _global_reductions(ctx, self._sh(ctx, r)):
            if int(alg) == L.MGS2B:
                # the reference's MGS2 recurrence (lanczos.jl:325-338) with the second sweep as one classical pass
                A_ = self._OpView(ctx, self.ops[_key(op)])
                wn = ko.apply(A_, V[-1])
                wn = wn - float(beta_old) * V[-2]
                alpha = ko.inner(V[-1], wn)
                wn = wn - alpha * V[-1]
                wn, sx = ko.orthogonalize(wn, V, np.zeros(len(V)), ko.Orth(ko.CGS))
                alpha += sx[-1]
                beta = ko.norm(wn)
            else:
                wn, alpha, beta = ko.lanczos_recurrence(self._OpView(ctx, self.ops[_key(op)]), V, float(beta_old),
                                                        ko.Orth(int(alg), float(eta)))
        self._setvec(ctx, w, wn)
        _set(alpha_out, float(alpha))
        _set(beta_out, float(beta))
        ctx.launches += 3
        return L.OK

    def b2k_lanczos_expand_many(self, h, op, cols, k, nsteps, beta_old, tol, alg, eta, alphas, betas, done, r_out):
        ctx = self._c(h)
        r = int(cols[k])
        _set(done, 0)
        _set(r_out, r)
        beta = float(beta_old)
        for i in range(nsteps):
            wref = C.c_int32()
            st = self.b2k_vec_alloc(h, r >> 20, wref)
            if st != L.OK:
                return st
            a, b = C.c_double(), C.c_double()
            st = self.b2k_lanczos_expand(h, op, cols, k, r, wref.value, beta, alg, eta, a, b)
            if st != L.OK:
                self.b2k_vec_free(h, wref.value)
                return st
            alphas[i], betas[i] = a.value, b.value
            if self.chain and alg in (L.CGS2, L.MGS2B):
                # the device-chained contract: the normalised vector lives in a column of its own and the old
                # residual's column goes back to the slab (it may be handed out again right away)
                vref = C.c_int32()
                st = self.b2k_vec_alloc(h, r >> 20, vref)
                if st != L.OK:
                    return st
                self.b2k_vec_copy(h, vref.value, r)
                self.b2k_vec_free(h, r)
                cols[k] = vref.value
            k += 1
            cols[k] = wref.value
            r, beta = wref.value, b.value
            _set(done, i + 1)
            _set(r_out, r)
            if beta <= tol:
                break
        return L.OK

    def _shifted(self, ctx, op, x, a0, a1):
        y = self.ops[_key(op)] @ ctx.gather_rows(x)
        return a1 * y + a0 * x if (a0 != 0 or a1 != 1) else y

    def b2k_cg_step(self, h, op, x, r, p, q, a0, a1, beta, rho, pq_out, normr_out):
        ctx = self._c(h)
        sh = self._sh(ctx, r)
        rv = self._vec(ctx, r).astype(np.float64)
        pv = beta * self._vec(ctx, p) + rv if beta != 0 else rv.copy()
        qv = self._shifted(ctx, op, pv, a0, a1)
        pq = float(ctx.allsum(np.dot(pv, qv), sh)[0])
        alpha = rho / pq
        self._setvec(ctx, p, pv)
        self._setvec(ctx, q, qv)
        self._setvec(ctx, x, self._vec(ctx, x) + alpha * pv)
        rn = rv - alpha * qv
        self._setvec(ctx, r, rn)
        _set(pq_out, pq)
        _set(normr_out, float(np.sqrt(ctx.allsum(np.dot(rn, rn), sh)[0])))
        return L.OK

    def b2k_cg_chain(self, h, op, x, r, p, q, a0, a1, beta, rho, tol, nsteps, pq_out, normr_out, done):
        hs = [int(v) for v in (x, r, p, q)]
        for i in range(4):
            for j in range(i):
                if hs[i] == hs[j]:
                    return self._fail(self._c(h), L.EINVAL, f"cg_chain: vectors {j} and {i} are the same")
        d = 0
        for i in range(nsteps):
            pq, nr = C.c_double(), C.c_double()
            st = self.b2k_cg_step(h, op, x, r, p, q, a0, a1, beta, rho, pq, nr)
            if st != L.OK:
                return st
            pq_out[i], normr_out[i] = pq.value, nr.value
            d = i + 1
            if nr.value < tol:
                break
            rho_old = rho
            rho = nr.value * nr.value
            beta = rho / rho_old
        _set(done, d)
        return L.OK

    def b2k_bicgstab_half(self, h, op, rs, r, p, v, s, a0, a1, beta, omega, rho, first, sigma_out, norms_out):
        ctx = self._c(h)
        sh = self._sh(ctx, r)
        rv = self._vec(ctx, r).astype(np.float64)
        pv = rv.copy() if first else rv + beta * (self._vec(ctx, p) - omega * self._vec(ctx, v))
        vv = self._shifted(ctx, op, pv, a0, a1)
        sigma = float(ctx.allsum(np.dot(self._vec(ctx, rs).astype(np.float64), vv), sh)[0])
        sv = rv - (rho / sigma) * vv
        self._setvec(ctx, p, pv)
        self._setvec(ctx, v, vv)
        self._setvec(ctx, s, sv)
        _set(sigma_out, sigma)
        _set(norms_out, float(np.sqrt(ctx.allsum(np.dot(sv, sv), sh)[0])))
        return L.OK

    def b2k_bicgstab_full(self, h, op, x, r, rs, p, s, t, a0, a1, alpha, omega_out, normr_out, rho_out):
        ctx = self._c(h)
        sh = self._sh(ctx, r)
        sv = self._vec(ctx, s).astype(np.float64)
        tv = self._shifted(ctx, op, sv, a0, a1)
        ts, tt = ctx.allsum([np.dot(tv, sv), np.dot(tv, tv)], sh)
        omega = ts / tt
        self._setvec(ctx, t, tv)
        self._setvec(ctx, x, (self._vec(ctx, x) + alpha * self._vec(ctx, p)) + omega * sv)
        rn = sv - omega * tv
        self._setvec(ctx, r, rn)
        nr, rho = ctx.allsum([np.dot(rn, rn), np.dot(self._vec(ctx, rs).astype(np.float64), rn)], sh)
        _set(omega_out, float(omega))
        _set(normr_out, float(np.sqrt(nr)))
        _set(rho_out, float(rho))
        return L.OK

    def b2k_bicgstab_chain(self, h, op, x, r, rs, p, v, s, t, a0, a1, rho, rho_old, alpha, omega, tol, nsteps,
                           rec_out, done):
        hs = [int(w) for w in (x, r, rs, p, v, s, t)]
        for i in range(7):
            for j in range(i):
                if hs[i] == hs[j]:
                    return self._fail(self._c(h), L.EINVAL, f"bicgstab_chain: vectors {j} and {i} are the same")
        d = 0
        for i in range(nsteps):
            beta = (rho / rho_old) * (alpha / omega)
            sg, ns = C.c_double(), C.c_double()
            st = self.b2k_bicgstab_half(h, op, rs, r, p, v, s, a0, a1, beta, omega, rho, 0, sg, ns)
            if st != L.OK:
                return st
            alpha = rho / sg.value
            rec = [rho, sg.value, alpha, ns.value, 0.0, 0.0, 0.0, 0.0]
            d = i + 1
            if ns.value < tol:
                rec[7] = 1.0
            else:
                om, nr, rn = C.c_double(), C.c_double(), C.c_double()
                st = self.b2k_bicgstab_full(h, op, x, r, rs, p, s, t, a0, a1, alpha, om, nr, rn)
                if st != L.OK:
                    return st
                omega = om.value
                rec[4:7] = [omega, nr.value, rn.value]
                rho_old, rho = rho, rn.value
                if nr.value < tol:
                    rec[7] = 2.0
            for j in range(8):
                rec_out[8 * i + j] = rec[j]
            if rec[7] != 0.0:
                break
        _set(done, d)
        return L.OK

    def b2k_host_lanczos_restart(self, *args):
        # host-only helper: the real library runs it without a GPU
        return _real_lib().b2k_host_lanczos_restart(*args)

    # ---- block ------------------------------------------------------------------------------------
    def b2k_block_inner(self, h, X, p, Y, q, M):
        ctx = self._c(h)
        Mv = _view(M, p * q, C.c_double)
        Xs, Ys = self._cols(ctx, X, p), self._cols(ctx, Y, q)
        with _global_reductions(ctx, self._sh(ctx, list(X)[0])):
            Mv[:] = ko.block_inner([x.astype(np.float64) for x in Xs], [y.astype(np.float64) for y in Ys]).T.reshape(-1)
        return L.OK

    def b2k_block_axpy(self, h, Y, q, X, p, M, ldm):
        ctx = self._c(h)
        Mm = np.array(_view(M, ldm * q, C.c_double)).reshape(q, ldm).T[:p, :]
        Xs = self._cols(ctx, X, p)
        for j, c in enumerate(list(Y)[:q]):
            acc = self._vec(ctx, c).astype(np.float64)
            for i in range(p):
                acc = acc - Mm[i, j] * Xs[i]
            self._setvec(ctx, c, acc)
        return L.OK

    def b2k_op_create_stencil_free(self, h, out, nx, ny, nz, c):
        return self.b2k_op_create_stencil(h, out, nx, ny, nz, c)

    def b2k_op_apply_block(self, h, op, X, Y, p):
        for x, y in zip(list(X)[:p], list(Y)[:p]):
            st = self.b2k_op_apply(h, op, x, y)
            if st != L.OK:
                return st
        return L.OK

    def b2k_block_orthogonalize(self, h, R, p, V, k, passes, Hh, Gh):
        """block classical Gram-Schmidt, `passes` times (the flagged engine mode)"""
        ctx = self._c(h)
        sh = self._sh(ctx, list(R)[0])
        Rs = np.column_stack([self._vec(ctx, c).astype(np.float64) for c in list(R)[:p]])
        Hsum = np.zeros((k, p))
        if k > 0:
            Vs = np.column_stack([v.astype(np.float64) for v in self._cols(ctx, V, k)])
            for _ in range(passes):
                Hm = np.array([[ctx.allsum(np.dot(Vs[:, j], Rs[:, i]), sh)[0] for i in range(p)] for j in range(k)])
                Rs = Rs - Vs @ Hm
                Hsum += Hm
        if Hh:
            _view(Hh, k * p, C.c_double)[:] = Hsum.T.reshape(-1)
        if Gh:
            G = np.array([[ctx.allsum(np.dot(Rs[:, i], Rs[:, j]), sh)[0] for j in range(p)] for i in range(p)])
            _view(Gh, p * p, C.c_double)[:] = G.T.reshape(-1)
        for i, c in enumerate(list(R)[:p]):
            self._setvec(ctx, c, Rs[:, i])
        return L.OK

    def b2k_block_cholqr(self, h, X, p, tol, G0, Rh, ok):
        ctx = self._c(h)
        sh = self._sh(ctx, list(X)[0])
        Xs = np.column_stack([self._vec(ctx, c).astype(np.float64) for c in list(X)[:p]])
        Rtot = np.eye(p)
        rel = 1e-11 * (np.finfo(ctx.dtype).eps / np.finfo(np.float64).eps)    # block.cu: 9e4 u of the vector type
        _set(ok, 0)
        for rnd in range(2):
            G = np.array([[ctx.allsum(np.dot(Xs[:, i], Xs[:, j]), sh)[0] for j in range(p)] for i in range(p)])
            try:
                Lc = np.linalg.cholesky(G)
            except np.linalg.LinAlgError:
                return L.OK
            if rnd == 0 and np.any(np.diag(Lc) ** 2 <= np.maximum((100 * tol) ** 2, rel * np.diag(G))):
                return L.OK
            Xs = np.linalg.solve(Lc, Xs.T).T
            Rtot = Lc.T @ Rtot
        _view(Rh, p * p, C.c_double)[:] = Rtot.T.reshape(-1)
        for i, c in enumerate(list(X)[:p]):
            self._setvec(ctx, c, Xs[:, i])
        _set(ok, 1)
        return L.OK

    def b2k_block_reorthogonalize(self, h, R, p, V, k):
        ctx = self._c(h)
        Vs = [v.astype(np.float64) for v in self._cols(ctx, V, k)]
        Rs = [self._vec(ctx, c).astype(np.float64) for c in list(R)[:p]]
        with _global_reductions(ctx, self._sh(ctx, list(R)[0])):
            ko.block_reorthogonalize(Rs, Vs)
        for c, r in zip(list(R)[:p], Rs):
            self._setvec(ctx, c, r)
        return L.OK

    def b2k_block_qr(self, h, X, p, tol, Rh, good, drift):
        ctx = self._c(h)
        blk = [self._vec(ctx, c).astype(np.float64) for c in list(X)[:p]]
        with _global_reductions(ctx, self._sh(ctx, list(X)[0])):
            Rg, gidx, dr = ko.block_qr(blk, tol)
        Rfull = np.zeros((p, p))
        for row, gi in enumerate(gidx):
            Rfull[gi, :] = Rg[row, :]
        _view(Rh, p * p, C.c_double)[:] = Rfull.T.reshape(-1)
        for i in range(p):
            good[i] = 1 if i in gidx else 0
        _set(drift, int(dr))
        for c, b in zip(list(X)[:p], blk):
            self._setvec(ctx, c, b)
        return L.OK


_REAL = None


def _real_lib():
    global _REAL
    if _REAL is None:
        _REAL = C.CDLL(L.LIB_PATH)
        name = "b2k_host_lanczos_restart"
        getattr(_REAL, name).restype, getattr(_REAL, name).argtypes = L._PROTOS[name]
    return _REAL


class installed:
    """Context manager: route `_lib.load()` to a fresh simulator.  `fused=False` (default) also switches the
    fused entry points off, so the drivers run their literal VectorInterface sequences; `fused=True` leaves
    the product's defaults (b2k_lanczos_expand[_many], b2k_cg_step, b2k_bicgstab_half/_full)."""

    def __init__(self, fused: bool = False):
        self.fused = fused

    def __enter__(self):
        import importlib
        self.lz = importlib.import_module("krylovkit_jl_b200.factorizations.lanczos")
        self.ls = importlib.import_module("krylovkit_jl_b200.linsolve")
        self.saved = (L._lib, self.lz.USE_FUSED_EXPAND, self.ls.USE_FUSED_CG, self.ls.USE_FUSED_BICGSTAB)
        L._lib = HostSimLib()
        if not self.fused:
            self.lz.USE_FUSED_EXPAND = False
            self.ls.USE_FUSED_CG = False
            self.ls.USE_FUSED_BICGSTAB = False
        return L._lib

    def __exit__(self, *exc):
        L._lib, self.lz.USE_FUSED_EXPAND, self.ls.USE_FUSED_CG, self.ls.USE_FUSED_BICGSTAB = self.saved
        return False
