"""TEST INFRASTRUCTURE ONLY — an fma-order restatement of one chained LSMR iteration (b2k_lsmr_chain: the A and A'
SpMVs, k_lsmr_m, k_lsmr_n, the reorthogonalisation, k_lsmr_alpha and the two flush launches), built on spmv_restate
for the SpMV rows and tsk_restate for the classical sweep, plus `lsmr_scalars`, the device recurrence in plain double
arithmetic.

One iteration k from the reference loop's state at the top of iteration k (u and v normalised, v in ring slot
(k - 1) % R, R = max(K, 1), no update pending), with th_r = T((-theta)/rho) and add1(x, b, y) = x if b == 0 else
fma(1, x, rn(b y)) (add!!(y, x, 1, b) as k_axpby rounds it):
    Av  = A v                                  (SpMV rows, operand scaled by T(1) = v)
    Ah  = add1(Av, th_r, Ah);  u~ = fma(T(-alpha), u, Av);  beta = sqrt(CTA-ordered sum of u~^2)
    beta > tol:   y = A' (u~ * T(1/beta));  v~ = fma(T(-beta), v, y)
                  K <= 1: alpha = sqrt(sum of v~^2) (k_lsmr_n's grid);  K > 1: the sweep over the ring's first
                  min(K, k) slots (MGS: k_dot / k_axpy_dev pipelined, once or twice; CGS2 / MGS2B: two classical
                  passes), alpha = sqrt(sum of v~^2) on k_lsmr_alpha's grid
    the recurrence (lsmr_scalars) -> g, zeta/(rho rhobar), the new theta and rho
    flush, m side:  Ah-bar = add1(Ah, T(g), Ah-bar);  r = fma(T(-cz), Ah-bar, r);  u = rn(u~ T(1/beta)) unless beta <= tol
    flush, n side:  v' = rn(v~ T(1/alpha)) into slot k % R (beta <= tol: v' = v; alpha <= tol: v' = v~, in the spare);
                    h-bar = add1(h, T(g), h-bar);  x = fma(T(cz), h-bar, x);  h = add1(v', T(-theta'/rho'), h)
The sums of the streaming kernels: a thread (grid-strided 128-bit vectors in order, then the tail elements on CTA 0)
accumulates fma(t, t, acc) in T, the CTA sums the threads' doubles with block_sum and the last CTA the CTA partials
(spmv_restate.last_cta).
"""
from __future__ import annotations

import math

import numpy as np

import spmv_restate as R
import tsk_restate as TR

f64, f32 = np.float64, np.float32
BT, CTAS_PER_SM = 256, 4
VEC = {f64: 2, f32: 4}


def _hyp(a, b):
    return np.sqrt(a * a + b * b)


def lsmr_scalars(st, alpha, beta, bskip, tol):
    """The device recurrence (blas1.cu::lsmr_recurrence) in np.float64 arithmetic, every operation rounded on its own
    and non-finite values carried through rather than raised (a division by zero is the code-4 path): st = the
    10-double state of the iteration's start; alpha, beta of this iteration.  Returns (new state, record of 16)."""
    _, _, alphabar, rhoold, rhobarold, cbar0, sbar0, _, zetabar0, lam = (f64(t) for t in st)
    alpha, beta = f64(alpha), f64(beta)
    with np.errstate(all="ignore"):
        alphahat = _hyp(alphabar, lam)
        rho = _hyp(alphahat, beta)
        c, s = alphahat / rho, beta / rho
        theta = s * alpha
        alphabar = c * alpha
        thetabar = sbar0 * rho
        cbarrho = cbar0 * rho
        rhobar = _hyp(cbarrho, theta)
        cbar, sbar = cbarrho / rhobar, theta / rhobar
        zeta = cbar * zetabar0
        zetabar = -sbar * zetabar0
        g = (-thetabar * rho) / (rhoold * rhobarold)
        cz = zeta / (rho * rhobar)
    askip = not bskip and not alpha > tol
    fin = all(np.isfinite(t) for t in (alpha, beta, rho, rhobar, g, cz, zetabar))
    code = 1.0 if abs(zetabar) <= tol else 2.0 if bskip else 3.0 if askip else 4.0 if not fin else 0.0
    rec = [alpha, beta, rho, rhobar, theta, zeta, abs(zetabar), code, 0.0 if bskip else 1.0, alphabar, cbar, sbar, g,
           cz, 0.0, 0.0]
    return [alpha, beta, alphabar, rho, rhobar, cbar, sbar, theta, zetabar, lam], [f64(t) for t in rec]


def grid_for(n, per_thread, nsm):
    want = max(1, -(-n // (BT * per_thread)))
    return int(min(want, CTAS_PER_SM * nsm))


# Edge lengths of the streaming kernels of blas1.cu.  A kernel launches grid_for(n, per_thread) CTAs of BT threads;
# thread t visits the 128-bit vectors t, t + BT G, t + 2 BT G, ... (G the grid) in trips of `unroll` slots
# (B2K_TRIP(unroll)), and CTA 0 takes the n % V tail elements.
SMALL = (1, 2, 3, "V-1", "V+1", 255, 257)


def cap_size(per_thread, nsm):
    """the largest n whose grid is exactly 4 SMs CTAs without clamping, tail empty in both types"""
    return per_thread * BT * CTAS_PER_SM * nsm


def trips_size(dt, unroll, nsm):
    """at the capped grid: 2 unroll + 1 full vectors per thread plus one more for the first half of the threads (three
    trips, the last one's second slot live for half of them), and a tail of V - 1 elements"""
    T = BT * CTAS_PER_SM * nsm
    return VEC[dt] * ((2 * unroll + 1) * T + T // 2) + VEC[dt] - 1


def edge_size(name, dt, per_thread, unroll, nsm):
    if name == "cap":
        return cap_size(per_thread, nsm)
    if name == "trips":
        return trips_size(dt, unroll, nsm)
    if name == "V-1":
        return VEC[dt] - 1
    if name == "V+1":
        return VEC[dt] + 1
    return name


def trip_profile(n, dt, per_thread, unroll, nsm):
    """what a length does to a streaming kernel: (grid, capped, most trips of a thread, the second slot of the last
    trip live for some threads but not all, tail length)"""
    V = VEC[dt]
    g = grid_for(n, per_thread, nsm)
    T = g * BT
    nv = n // V
    t = np.arange(T)
    cnt = np.where(t < nv, -(-(nv - t) // T), 0)                 # vectors of thread t
    trips = -(-cnt // unroll)
    in_last = np.where(cnt > 0, cnt - unroll * (trips - 1), 0)   # live slots of its last trip
    partial = 0 < int(np.count_nonzero(in_last >= 2)) < int(np.count_nonzero(cnt))
    return g, g == CTAS_PER_SM * nsm, int(trips.max(initial=0)), partial, n - nv * V


def check_edge(name, n, dt, per_thread, unroll, nsm):
    """assert that n has the property its name promises for this kernel"""
    g, capped, trips, partial, tail = trip_profile(n, dt, per_thread, unroll, nsm)
    if name == "cap":
        assert capped and tail == 0 and n == BT * per_thread * g, (name, n)
    elif name == "trips":
        assert capped and trips >= 3 and partial and tail > 0, (name, n, trips, partial, tail)


def thread_dots(fma, dt, a, b, grid):
    """per-thread fma chains of a_i b_i in T in the streaming kernels' visiting order -> (grid * 256,) of T"""
    V = VEC[dt]
    n = len(a)
    nv = n // V
    T = grid * BT
    rounds = -(-nv // T) if nv else 0
    acc = np.zeros(T, dtype=dt)
    pa = np.zeros(rounds * T * V, dtype=dt)
    pb = np.zeros(rounds * T * V, dtype=dt)
    pa[:nv * V] = a[:nv * V]
    pb[:nv * V] = b[:nv * V]
    pa, pb = pa.reshape(rounds, T, V), pb.reshape(rounds, T, V)
    for r in range(rounds):
        live = np.arange(T) + r * T < nv
        for j in range(V):
            acc = np.where(live, fma(pa[r, :, j], pb[r, :, j], acc, dt), acc)
    tail = n - nv * V
    if tail:
        acc[:tail] = fma(a[nv * V:], b[nv * V:], acc[:tail], dt)
    return acc


def blas1_sum(fma, dt, a, b, grid):
    """the CTA-ordered sum of a_i b_i of a blas1.cu streaming kernel on `grid` CTAs (block_sum, then the last CTA)"""
    acc = thread_dots(fma, dt, a, b, grid).astype(f64).reshape(grid, BT)
    part = R.cta_reduce(acc, "stream")
    return R.last_cta(part, "stream")


def add1(fma, dt, x, b, y):
    """add!!(y, x, 1, b) as k_axpby rounds it"""
    if b == 0.0:
        return np.asarray(x, dtype=dt).copy()
    return fma(dt(1), x, (dt(b) * np.asarray(y, dtype=dt)).astype(dt), dt)


def mgs(fma, dt, Q, x, nsm):
    """one pipelined MGS sweep (k_dot with the fused update, then k_axpy_dev) of x over the columns Q in order"""
    g = grid_for(len(x), 8, nsm)
    s_prev = None
    for j, q in enumerate(Q):
        if j > 0:
            x = fma(-dt(s_prev), Q[j - 1], x, dt)
        s_prev = blas1_sum(fma, dt, q, x, g)
    return fma(-dt(s_prev), Q[-1], x, dt)


def csr(M, dt):
    return M.indptr, M.indices, M.data.astype(dt)


def iteration(fma, dt, A, At, st, vec, ring, K, alg, tol, nsm, k, alpha_dev=None, beta_dev=None):
    """One call of one iteration (the first of the call, so nothing pending on entry).  vec: dict of host vectors
    x, h, hbar, r, Ah, Ahbar, u; ring: list of R host columns (v_k in slot (k - 1) % R).  alpha_dev / beta_dev:
    take these for the vectors (the sums are then checked on their own).  Returns (vectors, ring, spare, alpha,
    beta, state, record).  Non-finite scalars (a code-4 stop) propagate into the vectors as they do on the device."""
    with np.errstate(all="ignore"):
        return _iteration(fma, dt, A, At, st, vec, ring, K, alg, tol, nsm, k, alpha_dev, beta_dev)


def _iteration(fma, dt, A, At, st, vec, ring, K, alg, tol, nsm, k, alpha_dev, beta_dev):
    import krylovkit_jl_b200._lib as L
    Rn = max(K, 1)
    m, n = A.shape
    v = ring[(k - 1) % Rn]
    alpha, beta0 = st[0], st[1]
    tr = (-st[7]) / st[3]
    Av = R.csr_rows(*csr(A, dt), v, dt, 1.0, "pipe")
    Ah = add1(fma, dt, Av, tr, vec["Ah"])
    ut = fma(-dt(alpha), vec["u"], Av, dt)
    beta = math.sqrt(blas1_sum(fma, dt, ut, ut, grid_for(m, 4, nsm)))
    b_use = beta if beta_dev is None else beta_dev
    bskip = not b_use > tol
    spare = None
    a_sum = None
    if not bskip:
        y = R.csr_rows(*csr(At, dt), ut, dt, 1.0 / b_use, "pipe")
        vt = fma(-dt(b_use), v, y, dt)
        if K <= 1:
            a_sum = math.sqrt(blas1_sum(fma, dt, vt, vt, grid_for(n, 4, nsm)))
        else:
            Q = ring[:min(K, k)]
            if alg in (L.MGS, L.MGS2):
                for _ in range(1 if alg == L.MGS else 2):
                    vt = mgs(fma, dt, Q, vt, nsm)
            else:
                _, vt, _ = TR.cgs(np.column_stack(Q), vt, 2, nsm, fma)
            a_sum = math.sqrt(blas1_sum(fma, dt, vt, vt, grid_for(n, 8, nsm)))
        spare = vt
        alpha = a_sum if alpha_dev is None else alpha_dev
    st1 = list(st)
    st1[1] = b_use
    st2, rec = lsmr_scalars(st1, alpha, b_use, bskip, tol)
    g, cz = rec[12], rec[13]
    askip = rec[8] == 1.0 and not alpha > tol
    out = {}
    out["Ah"] = Ah
    out["Ahbar"] = add1(fma, dt, Ah, g, vec["Ahbar"])
    out["r"] = fma(-dt(cz), out["Ahbar"], vec["r"], dt)
    out["u"] = ut if bskip else (ut * dt(1.0 / b_use)).astype(dt)
    ring = [c.copy() for c in ring]
    if bskip:
        vn = v
    elif askip:
        vn = spare
    else:
        vn = (spare * dt(1.0 / alpha)).astype(dt)
        ring[k % Rn] = vn
    out["hbar"] = add1(fma, dt, vec["h"], g, vec["hbar"])
    out["x"] = fma(dt(cz), out["hbar"], vec["x"], dt)
    out["h"] = add1(fma, dt, vn, (-st2[7]) / st2[3], vec["h"])
    return out, ring, spare, a_sum, beta, st2, rec
