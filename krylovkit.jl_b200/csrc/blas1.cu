// blas1.cu — VectorInterface-level kernels: fill, scale, axpby, axpy2, inner, norm,
// single-vector orthogonalisation.  All HBM-bound streaming kernels: 128-bit vectorised
// loads, grid = multiple of the SM count, deterministic two-stage reductions (per-CTA
// partial -> last CTA sums the partials in CTA order; no floating-point atomics).
#include "common.cuh"
#include <cmath>

namespace {

// device-chained CG iterations (b2k_cg_chain): state = {rho, beta} on the device, rec = {<p,q>, ||r||} of this
// iteration, stop = flag raised when ||r|| < tol (the launches enqueued behind it then do nothing)
struct CgChain {
    double* state;
    double* rec;
    int* stop;
    double tol;
};

// device-chained BiCGStab iterations (b2k_bicgstab_chain): st = {rho, rho_old, alpha, omega} on the device,
// rec = {rho, sigma, alpha, ||s||, omega, ||r||, next rho, stop code} of this iteration
struct BicgChain {
    double* st;
    double* rec;
    int* stop;
    double tol;
};

constexpr int BT = 256;            // threads per CTA
constexpr int CTAS_PER_SM = 4;

template <typename T> struct Vec16;
template <> struct Vec16<double> { using type = double2; static constexpr int N = 2; };
template <> struct Vec16<float>  { using type = float4;  static constexpr int N = 4; };

template <typename T> __device__ __forceinline__ void vload(const T* p, T (&v)[Vec16<T>::N]);
template <> __device__ __forceinline__ void vload<double>(const double* p, double (&v)[2]) {
    double2 t = *reinterpret_cast<const double2*>(p);
    v[0] = t.x; v[1] = t.y;
}
template <> __device__ __forceinline__ void vload<float>(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <typename T> __device__ __forceinline__ void vstore(T* p, const T (&v)[Vec16<T>::N]);
template <> __device__ __forceinline__ void vstore<double>(double* p, const double (&v)[2]) {
    *reinterpret_cast<double2*>(p) = make_double2(v[0], v[1]);
}
template <> __device__ __forceinline__ void vstore<float>(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

// Streaming loops are written as TRIPS of UN grid-strided vectors per thread: all loads of a trip are issued before its
// first store.  (A plain `#pragma unroll 4` grid-stride loop does NOT do that: the store of iteration u may alias the
// load of iteration u+1 as far as the compiler knows, so the unrolled body stays load -> compute -> store, 32 bytes in
// flight per thread, too few to cover the latency of cold data in HBM.)
// The order in which a thread visits its elements is unchanged, so every reduction keeps its bits.
#define B2K_TRIP(UN)                                                                                   \
    for (int64_t i0 = blockIdx.x * (int64_t)BT + threadIdx.x; i0 < nv; i0 += (int64_t)(UN) * stride)
#define B2K_EACH(UN, u, i)                                                                             \
    _Pragma("unroll") for (int u = 0; u < (UN); ++u)                                                   \
        if (const int64_t i = i0 + (int64_t)u * stride; i < nv)

// 128-bit accesses with an L2 eviction-priority hint (createpolicy policies, see common.cuh)
template <typename T> __device__ __forceinline__ void vload_hint(const T* p, T (&v)[Vec16<T>::N], uint64_t pol);
template <> __device__ __forceinline__ void vload_hint<double>(const double* p, double (&v)[2], uint64_t pol) {
    asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v[0]), "=d"(v[1]) : "l"(p), "l"(pol));
}
template <> __device__ __forceinline__ void vload_hint<float>(const float* p, float (&v)[4], uint64_t pol) {
    asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p), "l"(pol));
}
template <typename T> __device__ __forceinline__ void vstore_hint(T* p, const T (&v)[Vec16<T>::N], uint64_t pol);
template <> __device__ __forceinline__ void vstore_hint<double>(double* p, const double (&v)[2], uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v[0]), "d"(v[1]), "l"(pol) : "memory");
}
template <> __device__ __forceinline__ void vstore_hint<float>(float* p, const float (&v)[4], uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "l"(pol) : "memory");
}

inline int grid_for(const b2k_ctx* ctx, int64_t n, int per_thread) {
    int64_t want = (n + (int64_t)BT * per_thread - 1) / ((int64_t)BT * per_thread);
    int64_t cap = (int64_t)ctx->num_sms * CTAS_PER_SM;
    if (want < 1) want = 1;
    return (int)(want < cap ? want : cap);
}

// ------------------------------------------------------------------ elementwise ----

template <typename T>
__global__ void __launch_bounds__(BT) k_fill_splitmix(T* x, int64_t n, uint64_t seed,
                                                      uint64_t row_offset) {
    for (int64_t i = blockIdx.x * (int64_t)BT + threadIdx.x; i < n; i += (int64_t)gridDim.x * BT)
        x[i] = (T)splitmix_unit(seed, row_offset + (uint64_t)i);
}

template <typename T>
__global__ void __launch_bounds__(BT) k_fill(T* x, int64_t n, T value) {
    for (int64_t i = blockIdx.x * (int64_t)BT + threadIdx.x; i < n; i += (int64_t)gridDim.x * BT)
        x[i] = value;
}

// y = alpha * x
template <typename T>
__global__ void __launch_bounds__(BT) k_scale(T* __restrict__ y, const T* __restrict__ x,
                                              int64_t n, T alpha) {
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T a[4][V];
        B2K_EACH(4, u, i) vload<T>(x + i * V, a[u]);
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) a[u][j] *= alpha;
            vstore<T>(y + i * V, a[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        y[i] = alpha * x[i];
    }
}

// y = beta*y + alpha*x   (beta == 0 never reads y: hard zero semantics)
// Rounding: MODE 0 rn(alpha*x), MODE 1 fma(alpha, x, y), MODE 2 fma(alpha, x, rn(beta*y)).
// SELF (add!!(y, y, alpha, beta)): x is y, read once through y (x is not dereferenced), with the same rounding as a
// call on a copy of y — not rn((alpha + beta) * y), which differs in the last bit for most entries.
template <typename T, int MODE, bool SELF>   // MODE 0: beta==0, 1: beta==1, 2: general
__global__ void __launch_bounds__(BT) k_axpby(T* __restrict__ y, const T* __restrict__ x,
                                              int64_t n, T alpha, T beta) {
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T a[4][V], b[4][V];
        B2K_EACH(4, u, i) {
            if (!SELF) vload<T>(x + i * V, a[u]);
            if (SELF || MODE != 0) vload<T>(y + i * V, b[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const T xv = SELF ? b[u][j] : a[u][j];
                if (MODE == 0) b[u][j] = alpha * xv;
                else if (MODE == 1) b[u][j] = fma(alpha, xv, b[u][j]);
                else b[u][j] = fma(alpha, xv, beta * b[u][j]);
            }
            vstore<T>(y + i * V, b[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        const T xv = SELF ? y[i] : x[i];
        if (MODE == 0) y[i] = alpha * xv;
        else if (MODE == 1) y[i] = fma(alpha, xv, y[i]);
        else y[i] = fma(alpha, xv, beta * y[i]);
    }
}

// y = (y + a1*x1) + a2*x2, same rounding sequence as two consecutive add!! calls
template <typename T>
__global__ void __launch_bounds__(BT) k_axpy2(T* __restrict__ y, const T* __restrict__ x1, T a1,
                                              const T* __restrict__ x2, T a2, int64_t n) {
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T a[4][V], b[4][V], c[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(y + i * V, c[u]);
            vload<T>(x1 + i * V, a[u]);
            vload<T>(x2 + i * V, b[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) c[u][j] = fma(a2, b[u][j], fma(a1, a[u][j], c[u][j]));
            vstore<T>(y + i * V, c[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        y[i] = fma(a2, x2[i], fma(a1, x1[i], y[i]));
    }
}

__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }

// (q1,q2) <- (c*q1 - s*q2, s*q1 + c*q2)   — dense/givens.jl:22-36
// Rounded as rmul!(b, G) does it for a vector type with add / add!! (givens.jl:30-36):
//   q1' = add(q1, q2, -s, c)   = fma(-s, q2, rn(c*q1))
//   q2' = add!!(q2, q1, s, c)  = fma(s, q1, rn(c*q2))
// The pairing is spelled out with fma and an explicitly rounded product, so nvcc's contraction has no choice to make.
template <typename T>
__device__ __forceinline__ void givens_rn(T c, T s, T a, T b, T& o1, T& o2) {
    o1 = fma(-s, b, mul_rn(c, a));
    o2 = fma(s, a, mul_rn(c, b));
}

template <typename T>
__global__ void __launch_bounds__(BT) k_givens(T* __restrict__ q1, T* __restrict__ q2, int64_t n,
                                               T c, T s) {
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T a[4][V], b[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(q1 + i * V, a[u]);
            vload<T>(q2 + i * V, b[u]);
        }
        B2K_EACH(4, u, i) {
            T o1[V], o2[V];
#pragma unroll
            for (int j = 0; j < V; ++j) givens_rn(c, s, a[u][j], b[u][j], o1[j], o2[j]);
            vstore<T>(q1 + i * V, o1);
            vstore<T>(q2 + i * V, o2);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        T o1, o2;
        givens_rn(c, s, q1[i], q2[i], o1, o2);
        q1[i] = o1;
        q2[i] = o2;
    }
}

// ------------------------------------------------------------------ reductions ----
// out[0] = sum_i x[i]*y[i]; optional fused update: x <- x - s_prev * q_prev BEFORE the dot,
// with s_prev read from d_res[src] (device scalar of the previous reduction).  That is the
// pipelined MGS step (orthonormal.jl:417-421): v -= s_{j-1} q_{j-1}; s_j = <q_j, v>.
// FINAL: 0 = raw sum, 1 = sqrt(sum)
template <typename T, bool UPDATE, bool NORM>
__global__ void __launch_bounds__(BT)
k_dot(const T* __restrict__ q, T* __restrict__ x, int64_t n, const T* __restrict__ qprev,
      const double* __restrict__ sprev, double* __restrict__ part, unsigned* __restrict__ ticket,
      double* __restrict__ out, double* __restrict__ accum_into, int hints) {
    __shared__ double red[32];
    __shared__ bool last;
    // hints (the MGS sweep): x is re-read and re-written once per basis column — keep it in L2 (evict_last);
    // the basis columns pass once (evict_first)
    const uint64_t pol_keep = hints ? l2_policy_evict_last() : 0, pol_once = hints ? l2_policy_evict_first() : 0;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    T sp = 0;
    if (UPDATE) sp = (T)(*sprev);
    T acc = 0;
    B2K_TRIP(4) {
        T a[4][V], b[4][V], c[4][V];
        if (hints) {
            B2K_EACH(4, u, i) {
                vload_hint<T>(x + i * V, b[u], pol_keep);
                if (UPDATE) vload_hint<T>(qprev + i * V, c[u], pol_once);
                if (!NORM) vload_hint<T>(q + i * V, a[u], pol_once);
            }
        } else {
            B2K_EACH(4, u, i) {
                vload<T>(x + i * V, b[u]);
                if (UPDATE) vload<T>(qprev + i * V, c[u]);
                if (!NORM) vload<T>(q + i * V, a[u]);
            }
        }
        B2K_EACH(4, u, i) {
            if (UPDATE) {
#pragma unroll
                for (int j = 0; j < V; ++j) b[u][j] = fma(-sp, c[u][j], b[u][j]);
                if (hints) vstore_hint<T>(x + i * V, b[u], pol_keep);
                else vstore<T>(x + i * V, b[u]);
            }
            if (NORM) {
#pragma unroll
                for (int j = 0; j < V; ++j) acc = fma(b[u][j], b[u][j], acc);
            } else {
#pragma unroll
                for (int j = 0; j < V; ++j) acc = fma(a[u][j], b[u][j], acc);
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        T b = x[i];
        if (UPDATE) {
            b = fma(-sp, qprev[i], b);
            x[i] = b;
        }
        acc = NORM ? fma(b, b, acc) : fma(q[i], b, acc);
    }
    double s = block_sum((double)acc, red);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = s;
        __threadfence();
        unsigned t = atomicInc(ticket, gridDim.x - 1);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        double v = 0.0;
        for (int g = threadIdx.x; g < gridDim.x; g += BT) v += part[g];   // fixed assignment
        double tot = block_sum(v, red);
        if (threadIdx.x == 0) {
            *out = tot;
            if (accum_into) *accum_into += tot;
        }
    }
}

// final fix-up: x <- x - s*q with s = d_res[src] (tail of the pipelined MGS sweep)
template <typename T>
__global__ void __launch_bounds__(BT)
k_axpy_dev(T* __restrict__ x, const T* __restrict__ q, const double* __restrict__ s, int64_t n) {
    const T sp = (T)(*s);
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T a[4][V], b[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(x + i * V, b[u]);
            vload<T>(q + i * V, a[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) b[u][j] = fma(-sp, a[u][j], b[u][j]);
            vstore<T>(x + i * V, b[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        int64_t i = nv * V + threadIdx.x;
        x[i] = fma(-sp, q[i], x[i]);
    }
}

// CG update (src/linsolve/cg.jl:64-67): alpha = rho / <p,q> (both on the device); x += alpha p;
// r -= alpha q; out[0] = ||r||^2 — one pass over four vectors (6W) instead of three (7W + 2 syncs).
template <typename T>
__global__ void __launch_bounds__(BT)
k_cg_xr(T* __restrict__ x, T* __restrict__ r, const T* __restrict__ p, const T* __restrict__ q, int64_t n,
        double rho, const double* __restrict__ pq, double* __restrict__ part, unsigned* __restrict__ ticket,
        double* __restrict__ out, const CgChain ch) {
    __shared__ double red[32];
    __shared__ bool last;
    if (ch.stop && *reinterpret_cast<const volatile int*>(ch.stop)) return;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    if (ch.state) rho = *reinterpret_cast<const volatile double*>(ch.state);      // rho kept on the device
    const T alpha = (T)(rho / *pq);
    T acc = 0;
    B2K_TRIP(2) {
        T xv[2][V], rv[2][V], pv[2][V], qv[2][V];
        B2K_EACH(2, u, i) {
            vload<T>(x + i * V, xv[u]);
            vload<T>(r + i * V, rv[u]);
            vload<T>(p + i * V, pv[u]);
            vload<T>(q + i * V, qv[u]);
        }
        B2K_EACH(2, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                xv[u][j] = fma(alpha, pv[u][j], xv[u][j]);
                rv[u][j] = fma(-alpha, qv[u][j], rv[u][j]);
                acc = fma(rv[u][j], rv[u][j], acc);
            }
            vstore<T>(x + i * V, xv[u]);
            vstore<T>(r + i * V, rv[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        x[i] = fma(alpha, p[i], x[i]);
        const T rr = fma(-alpha, q[i], r[i]);
        r[i] = rr;
        acc = fma(rr, rr, acc);
    }
    const double sblk = block_sum((double)acc, red);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = sblk;
        __threadfence();
        const unsigned t = atomicInc(ticket, gridDim.x - 1);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        double v = 0.0;
        const volatile double* pv2 = part;
        for (int g = threadIdx.x; g < (int)gridDim.x; g += BT) v += pv2[g];
        const double tot = block_sum(v, red);
        if (threadIdx.x == 0) {
            *out = tot;
            if (ch.state) {
                // cg.jl:74-77 on the device: normr = sqrt(||r||^2); rho_old = rho; rho = normr^2; beta = rho / rho_old
                const double nr = sqrt(tot);
                const double rho_new = nr * nr;
                ch.state[1] = rho_new / rho;
                ch.state[0] = rho_new;
                ch.rec[0] = *pq;
                ch.rec[1] = nr;
                if (nr < ch.tol) *ch.stop = 1;     // cg.jl:68: the host takes over (explicit residual, restart)
            }
        }
    }
}

// x + beta*y with the product rounded first: what k_axpby<T, 2> computes for alpha = 1, fma(1, x, rn(beta*y)).
// (Written with the explicit-rounding intrinsics: `x + beta*y` would be contracted into ONE fma(beta, y, x).)
__device__ __forceinline__ double xpby_rn(double x, double beta, double y) { return __dadd_rn(x, __dmul_rn(beta, y)); }
__device__ __forceinline__ float xpby_rn(float x, float beta, float y) { return __fadd_rn(x, __fmul_rn(beta, y)); }

// p <- r + beta p with beta on the device (same bits as k_axpby<T, 2> with alpha = 1)
template <typename T>
__global__ void __launch_bounds__(BT) k_xpby_dev(T* __restrict__ y, const T* __restrict__ x, int64_t n,
                                                 const double* __restrict__ beta_dev, const int* __restrict__ stop) {
    if (stop && *reinterpret_cast<const volatile int*>(stop)) return;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    const T beta = (T)(*beta_dev);
    B2K_TRIP(4) {
        T a[4][V], b[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(x + i * V, a[u]);
            vload<T>(y + i * V, b[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) b[u][j] = xpby_rn(a[u][j], beta, b[u][j]);
            vstore<T>(y + i * V, b[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        y[i] = xpby_rn(x[i], beta, y[i]);
    }
}

// ---- BiCGStab (src/linsolve/bicgstab.jl) elementwise stages: each is one sweep, sums are formed with the
// same fma pairing as the literal add!! sequence they replace ----

// p <- r + beta*(p - omega*v)   (bicgstab.jl:101-102: p = add!!(p, v, -ω); p = add!!(p, r, 1, β))
template <typename T>
__global__ void __launch_bounds__(BT)
k_bicg_p(T* __restrict__ p, const T* __restrict__ r, const T* __restrict__ v, int64_t n, T beta, T omega,
         const BicgChain ch) {
    if (ch.stop && *reinterpret_cast<const volatile int*>(ch.stop)) return;
    if (ch.st) {   // bicgstab.jl:98-100 on the device: beta = (rho / rho_old) * (alpha / omega)
        const volatile double* st = ch.st;
        const double om = st[3];
        beta = (T)((st[0] / st[1]) * (st[2] / om));
        omega = (T)om;
    }
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    B2K_TRIP(4) {
        T pv[4][V], rv[4][V], vv[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(p + i * V, pv[u]);
            vload<T>(r + i * V, rv[u]);
            vload<T>(v + i * V, vv[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const T tmp = fma(-omega, vv[u][j], pv[u][j]);    // add!!(p, v, -ω)       (k_axpby MODE 1)
                pv[u][j] = fma((T)1, rv[u][j], beta * tmp);       // add!!(p, r, 1, β)     (k_axpby MODE 2)
            }
            vstore<T>(p + i * V, pv[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        const T tmp = fma(-omega, v[i], p[i]);
        p[i] = fma((T)1, r[i], beta * tmp);
    }
}

// two-stage deterministic finish shared by the kernels below: per-CTA partials, last CTA adds them in
// CTA order; NRED independent sums (part is NRED x gridDim.x)
template <int NRED>
__device__ __forceinline__ void finish_sums(const double (&blk)[NRED], double* __restrict__ part,
                                            unsigned* __restrict__ ticket, double* __restrict__ out,
                                            double* red, bool* last) {
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < NRED; ++k) part[(size_t)k * gridDim.x + blockIdx.x] = blk[k];
        __threadfence();
        const unsigned t = atomicInc(ticket, gridDim.x - 1);
        *last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (*last) {
        __threadfence();
        const volatile double* pv = part;
#pragma unroll
        for (int k = 0; k < NRED; ++k) {
            double v = 0.0;
            for (int g = threadIdx.x; g < (int)gridDim.x; g += BT) v += pv[(size_t)k * gridDim.x + g];
            const double tot = block_sum(v, red);
            if (threadIdx.x == 0) out[k] = tot;
        }
    }
}

// s <- r - alpha*v with alpha = rho / *sigma (device scalar); out[0] = ||s||^2   (bicgstab.jl:109-116)
template <typename T>
__global__ void __launch_bounds__(BT)
k_bicg_s(T* __restrict__ s, const T* __restrict__ r, const T* __restrict__ v, int64_t n, double rho,
         const double* __restrict__ sigma, double* __restrict__ part, unsigned* __restrict__ ticket,
         double* __restrict__ out, const BicgChain ch) {
    __shared__ double red[32];
    __shared__ bool last;
    if (ch.stop && *reinterpret_cast<const volatile int*>(ch.stop)) return;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    if (ch.st) rho = *reinterpret_cast<const volatile double*>(ch.st);
    const T alpha = (T)(rho / *sigma);
    T acc = 0;
    B2K_TRIP(4) {
        T rv[4][V], vv[4][V];
        B2K_EACH(4, u, i) {
            vload<T>(r + i * V, rv[u]);
            vload<T>(v + i * V, vv[u]);
        }
        B2K_EACH(4, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                rv[u][j] = fma(-alpha, vv[u][j], rv[u][j]);
                acc = fma(rv[u][j], rv[u][j], acc);
            }
            vstore<T>(s + i * V, rv[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        const T sv = fma(-alpha, v[i], r[i]);
        s[i] = sv;
        acc = fma(sv, sv, acc);
    }
    const double blk[1] = {block_sum((double)acc, red)};
    finish_sums<1>(blk, part, ticket, out, red, &last);
    if (ch.st && last && threadIdx.x == 0) {
        // bicgstab.jl:106-118 on the device: alpha = rho / sigma, the half-step residual norm and its test
        const double sg = *sigma, al = rho / sg, ns = sqrt(out[0]);
        ch.rec[0] = rho; ch.rec[1] = sg; ch.rec[2] = al; ch.rec[3] = ns;
        ch.st[2] = al;
        if (ns < ch.tol) {
            ch.rec[7] = 1.0;
            *ch.stop = 1;
        }
    }
}

// x <- (x + alpha*p) + omega*s ; r <- s - omega*t with omega = *ts / *tt (device scalars);
// out[0] = ||r||^2, out[1] = <rs, r>   (bicgstab.jl:143-150 and the next iteration's rho, :98)
template <typename T>
__global__ void __launch_bounds__(BT)
k_bicg_xr(T* __restrict__ x, T* __restrict__ r, const T* __restrict__ rs, const T* __restrict__ p,
          const T* __restrict__ s, const T* __restrict__ t, int64_t n, T alpha, const double* __restrict__ ts,
          const double* __restrict__ tt, double* __restrict__ part, unsigned* __restrict__ ticket,
          double* __restrict__ out, const BicgChain ch) {
    __shared__ double red[32];
    __shared__ bool last;
    if (ch.stop && *reinterpret_cast<const volatile int*>(ch.stop)) return;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    if (ch.st) alpha = (T)(*reinterpret_cast<const volatile double*>(ch.st + 2));
    const T omega = (T)(*ts / *tt);
    T a1 = 0, a2 = 0;
    B2K_TRIP(2) {
        T xv[2][V], pv[2][V], sv[2][V], tv[2][V], qv[2][V];
        B2K_EACH(2, u, i) {
            vload<T>(x + i * V, xv[u]);
            vload<T>(p + i * V, pv[u]);
            vload<T>(s + i * V, sv[u]);
            vload<T>(t + i * V, tv[u]);
            vload<T>(rs + i * V, qv[u]);
        }
        B2K_EACH(2, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                xv[u][j] = fma(omega, sv[u][j], fma(alpha, pv[u][j], xv[u][j]));
                tv[u][j] = fma(-omega, tv[u][j], sv[u][j]);
                a1 = fma(tv[u][j], tv[u][j], a1);
                a2 = fma(qv[u][j], tv[u][j], a2);
            }
            vstore<T>(x + i * V, xv[u]);
            vstore<T>(r + i * V, tv[u]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        x[i] = fma(omega, s[i], fma(alpha, p[i], x[i]));
        const T rr = fma(-omega, t[i], s[i]);
        r[i] = rr;
        a1 = fma(rr, rr, a1);
        a2 = fma(rs[i], rr, a2);
    }
    double blk[2];
    blk[0] = block_sum((double)a1, red);
    blk[1] = block_sum((double)a2, red);
    finish_sums<2>(blk, part, ticket, out, red, &last);
    if (ch.st && last && threadIdx.x == 0) {
        // bicgstab.jl:141-152 and the next iteration's :97-98 on the device
        const double om = *ts / *tt, nr = sqrt(out[0]), rho_next = out[1];
        ch.rec[4] = om; ch.rec[5] = nr; ch.rec[6] = rho_next;
        ch.st[3] = om;
        ch.st[1] = ch.st[0];
        ch.st[0] = rho_next;
        if (nr < ch.tol) {
            ch.rec[7] = 2.0;
            *ch.stop = 1;
        }
    }
}

}  // namespace

// ------------------------------------------------------------------ internal API ----
// Enqueue: d_res[slot] = <q, x> (or ||x||^2 if q == nullptr), optionally after the fused
// update x -= d_res[sprev_slot] * qprev.  If accum_slot >= 0, also d_res[accum_slot] += result.
// Single-GPU: complete on return of the stream work.  Dist: caller allreduces d_res[slot].
int32_t b2k_enqueue_dot(b2k_ctx* ctx, const void* q, void* x, int64_t n, const void* qprev,
                        int sprev_slot, int slot, int accum_slot) {
    const int grid = grid_for(ctx, n, 8);
    double* out = ctx->d_res + slot;
    double* acc = accum_slot >= 0 ? ctx->d_res + accum_slot : nullptr;
    const double* sp = sprev_slot >= 0 ? ctx->d_res + sprev_slot : nullptr;
    unsigned* ticket = ctx->d_sync;
#define LAUNCH(T, UPD, NRM)                                                              \
    k_dot<T, UPD, NRM><<<grid, BT, 0, ctx->stream>>>((const T*)q, (T*)x, n, (const T*)qprev, \
                                                     sp, ctx->d_part_s, ticket, out, acc, ctx->dot_hints)
    const bool upd = qprev != nullptr, nrm = q == nullptr;
    if (ctx->dtype == B2K_F64) {
        if (upd && nrm) LAUNCH(double, true, true);
        else if (upd) LAUNCH(double, true, false);
        else if (nrm) LAUNCH(double, false, true);
        else LAUNCH(double, false, false);
    } else {
        if (upd && nrm) LAUNCH(float, true, true);
        else if (upd) LAUNCH(float, true, false);
        else if (nrm) LAUNCH(float, false, true);
        else LAUNCH(float, false, false);
    }
#undef LAUNCH
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t b2k_enqueue_axpy_dev(b2k_ctx* ctx, void* x, const void* q, int s_slot, int64_t n) {
    const int grid = grid_for(ctx, n, 8);
    if (ctx->dtype == B2K_F64)
        k_axpy_dev<double><<<grid, BT, 0, ctx->stream>>>((double*)x, (const double*)q,
                                                         ctx->d_res + s_slot, n);
    else
        k_axpy_dev<float><<<grid, BT, 0, ctx->stream>>>((float*)x, (const float*)q,
                                                        ctx->d_res + s_slot, n);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

// ------------------------------------------------------------------ C ABI ----

extern "C" int32_t b2k_vec_fill_splitmix(b2k_ctx* ctx, b2k_vec v, uint64_t seed) {
    if (!ctx) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    if (r.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, r.n, 4);
    const uint64_t off = r.sharded ? (uint64_t)ctx->row_offset : 0ull;
    if (ctx->dtype == B2K_F64)
        k_fill_splitmix<double><<<grid, BT, 0, ctx->stream>>>((double*)r.ptr, r.n, seed, off);
    else
        k_fill_splitmix<float><<<grid, BT, 0, ctx->stream>>>((float*)r.ptr, r.n, seed, off);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_fill(b2k_ctx* ctx, b2k_vec v, double value) {
    if (!ctx) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    if (r.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, r.n, 4);
    if (ctx->dtype == B2K_F64)
        k_fill<double><<<grid, BT, 0, ctx->stream>>>((double*)r.ptr, r.n, value);
    else
        k_fill<float><<<grid, BT, 0, ctx->stream>>>((float*)r.ptr, r.n, (float)value);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_scale(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha) {
    if (!ctx) return B2K_EINVAL;
    VecRef ry, rx;
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    if (ry.n != rx.n) return b2k_fail(ctx, B2K_EDIM, "vec_scale: length mismatch");
    if (ry.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, ry.n, 8);
    if (ctx->dtype == B2K_F64)
        k_scale<double><<<grid, BT, 0, ctx->stream>>>((double*)ry.ptr, (const double*)rx.ptr,
                                                      ry.n, alpha);
    else
        k_scale<float><<<grid, BT, 0, ctx->stream>>>((float*)ry.ptr, (const float*)rx.ptr, ry.n,
                                                     (float)alpha);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_axpby(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha, double beta) {
    if (!ctx) return B2K_EINVAL;
    VecRef ry, rx;
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    if (ry.n != rx.n) return b2k_fail(ctx, B2K_EDIM, "vec_axpby: length mismatch");
    if (ry.n == 0) return B2K_OK;
    // add!!(y, y, alpha, beta): y <- (beta + alpha) * y would change rounding; do it literally, reading y once
    const bool self = ry.ptr == rx.ptr;
    const int grid = grid_for(ctx, ry.n, 8);
#define LAUNCH_S(T, MODE, SELF)                                                                              \
    k_axpby<T, MODE, SELF><<<grid, BT, 0, ctx->stream>>>((T*)ry.ptr, SELF ? nullptr : (const T*)rx.ptr, ry.n, \
                                                         (T)alpha, (T)beta)
#define LAUNCH(T, MODE)                       \
    do {                                      \
        if (self) LAUNCH_S(T, MODE, true);    \
        else LAUNCH_S(T, MODE, false);        \
    } while (0)
    if (ctx->dtype == B2K_F64) {
        if (beta == 0.0) LAUNCH(double, 0);
        else if (beta == 1.0) LAUNCH(double, 1);
        else LAUNCH(double, 2);
    } else {
        if (beta == 0.0) LAUNCH(float, 0);
        else if (beta == 1.0) LAUNCH(float, 1);
        else LAUNCH(float, 2);
    }
#undef LAUNCH
#undef LAUNCH_S
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_axpy2(b2k_ctx* ctx, b2k_vec y, b2k_vec x1, double a1, b2k_vec x2,
                                 double a2) {
    if (!ctx) return B2K_EINVAL;
    VecRef ry, r1, r2;
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    B2K_TRY(b2k_resolve(ctx, x1, &r1));
    B2K_TRY(b2k_resolve(ctx, x2, &r2));
    if (ry.n != r1.n || ry.n != r2.n) return b2k_fail(ctx, B2K_EDIM, "vec_axpy2: length mismatch");
    if (ry.ptr == r1.ptr || ry.ptr == r2.ptr)
        return b2k_fail(ctx, B2K_EINVAL, "vec_axpy2: y must not alias x1/x2");
    if (ry.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, ry.n, 8);
    if (ctx->dtype == B2K_F64)
        k_axpy2<double><<<grid, BT, 0, ctx->stream>>>((double*)ry.ptr, (const double*)r1.ptr, a1,
                                                      (const double*)r2.ptr, a2, ry.n);
    else
        k_axpy2<float><<<grid, BT, 0, ctx->stream>>>((float*)ry.ptr, (const float*)r1.ptr,
                                                     (float)a1, (const float*)r2.ptr, (float)a2,
                                                     ry.n);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_basis_givens(b2k_ctx* ctx, b2k_vec q1, b2k_vec q2, double c, double s) {
    if (!ctx) return B2K_EINVAL;
    VecRef r1, r2;
    B2K_TRY(b2k_resolve(ctx, q1, &r1));
    B2K_TRY(b2k_resolve(ctx, q2, &r2));
    if (r1.n != r2.n) return b2k_fail(ctx, B2K_EDIM, "basis_givens: length mismatch");
    if (r1.ptr == r2.ptr) return b2k_fail(ctx, B2K_EINVAL, "basis_givens: q1 == q2");
    if (r1.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, r1.n, 8);
    if (ctx->dtype == B2K_F64)
        k_givens<double><<<grid, BT, 0, ctx->stream>>>((double*)r1.ptr, (double*)r2.ptr, r1.n, c, s);
    else
        k_givens<float><<<grid, BT, 0, ctx->stream>>>((float*)r1.ptr, (float*)r2.ptr, r1.n,
                                                      (float)c, (float)s);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_inner(b2k_ctx* ctx, b2k_vec x, b2k_vec y, double* out) {
    if (!ctx || !out) return B2K_EINVAL;
    VecRef rx, ry;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    if (rx.n != ry.n) return b2k_fail(ctx, B2K_EDIM, "vec_inner: length mismatch");
    B2K_TRY(b2k_enqueue_dot(ctx, rx.ptr, ry.ptr, rx.n, nullptr, -1, 0, -1));
    B2K_TRY(b2k_fetch_results(ctx, 1, rx.sharded));
    *out = ctx->h_res[0];
    return B2K_OK;
}

extern "C" int32_t b2k_vec_norm(b2k_ctx* ctx, b2k_vec x, double* out) {
    if (!ctx || !out) return B2K_EINVAL;
    VecRef rx;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rx.ptr, rx.n, nullptr, -1, 0, -1));
    B2K_TRY(b2k_fetch_results(ctx, 1, rx.sharded));
    *out = sqrt(ctx->h_res[0]);
    return B2K_OK;
}

// orthogonalize!!(v, q, alg) against one normalised vector — src/orthonormal.jl:455-489
extern "C" int32_t b2k_vec_orthogonalize(b2k_ctx* ctx, b2k_vec v, b2k_vec q, int32_t alg,
                                         double eta, double* s_out, double* nrm_out) {
    if (!ctx || !s_out) return B2K_EINVAL;
    VecRef rv, rq;
    B2K_TRY(b2k_resolve(ctx, v, &rv));
    B2K_TRY(b2k_resolve(ctx, q, &rq));
    if (rv.n != rq.n) return b2k_fail(ctx, B2K_EDIM, "vec_orthogonalize: length mismatch");
    if (rv.ptr == rq.ptr) return b2k_fail(ctx, B2K_EINVAL, "vec_orthogonalize: v == q");
    const int64_t n = rv.n;
    const int sh = rv.sharded;
    const bool dist = ctx->nranks > 1 && sh;
    auto dot = [&](int slot) -> int32_t {   // d_res[slot] = <q, v>
        B2K_TRY(b2k_enqueue_dot(ctx, rq.ptr, rv.ptr, n, nullptr, -1, slot, -1));
        return b2k_allreduce(ctx, ctx->d_res + slot, 1, sh);
    };
    auto nrm2 = [&](int slot) -> int32_t {
        B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rv.ptr, n, nullptr, -1, slot, -1));
        return b2k_allreduce(ctx, ctx->d_res + slot, 1, sh);
    };
    (void)dist;
    double s = 0.0;
    if (alg == B2K_MGS2B) alg = B2K_MGS2;      // one vector: blocked and sequential sweeps are the same thing
    if (alg == B2K_CGS || alg == B2K_MGS) {
        B2K_TRY(dot(0));
        B2K_TRY(b2k_enqueue_axpy_dev(ctx, rv.ptr, rq.ptr, 0, n));
        B2K_TRY(nrm2(1));
        B2K_TRY(b2k_fetch_results(ctx, 2, 0));
        s = ctx->h_res[0];
    } else if (alg == B2K_CGS2 || alg == B2K_MGS2) {
        B2K_TRY(dot(0));
        B2K_TRY(b2k_enqueue_axpy_dev(ctx, rv.ptr, rq.ptr, 0, n));
        B2K_TRY(dot(2));
        B2K_TRY(b2k_enqueue_axpy_dev(ctx, rv.ptr, rq.ptr, 2, n));
        B2K_TRY(nrm2(1));
        B2K_TRY(b2k_fetch_results(ctx, 3, 0));
        s = ctx->h_res[0] + ctx->h_res[2];
    } else if (alg == B2K_CGSIR || alg == B2K_MGSIR) {
        B2K_TRY(nrm2(1));
        B2K_TRY(dot(0));
        B2K_TRY(b2k_enqueue_axpy_dev(ctx, rv.ptr, rq.ptr, 0, n));
        B2K_TRY(nrm2(2));
        B2K_TRY(b2k_fetch_results(ctx, 3, 0));
        double nold = sqrt(ctx->h_res[1]);
        s = ctx->h_res[0];
        double nnew = sqrt(ctx->h_res[2]);
        const double eps = (ctx->dtype == B2K_F64) ? 0x1p-52 : 0x1p-23;    // eps(T), orthonormal.jl:481
        while (eps < nnew && nnew < eta * nold) {
            nold = nnew;
            B2K_TRY(dot(0));
            B2K_TRY(b2k_enqueue_axpy_dev(ctx, rv.ptr, rq.ptr, 0, n));
            B2K_TRY(nrm2(2));
            B2K_TRY(b2k_fetch_results(ctx, 3, 0));
            s += ctx->h_res[0];
            nnew = sqrt(ctx->h_res[2]);
        }
        *s_out = s;
        if (nrm_out) *nrm_out = nnew;
        return B2K_OK;
    } else {
        return b2k_fail(ctx, B2K_EINVAL, "vec_orthogonalize: unknown orthogonalizer %d", alg);
    }
    *s_out = s;
    if (nrm_out) *nrm_out = sqrt(ctx->h_res[1]);
    return B2K_OK;
}

// spmv.cu
int32_t b2k_enqueue_apply(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y, double a0,
                          double a1, bool shifted, const VecRef* dotv, int dot_slot);

// One conjugate-gradient iteration — src/linsolve/cg.jl:62-67 — with a single host round trip:
//   p <- beta*p + r ; q <- (a0 + a1*A) p with <p,q> fused into the SpMV ; alpha = rho/<p,q> on the
//   device ; x += alpha p ; r -= alpha q ; ||r||.   beta = 0 gives the first iteration (p = r).
extern "C" int32_t b2k_cg_step(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec p, b2k_vec q,
                               double a0, double a1, double beta, double rho, double* pq_out,
                               double* normr_out) {
    if (!ctx || !op || !pq_out || !normr_out) return B2K_EINVAL;
    VecRef rx, rr, rp, rq;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, r, &rr));
    B2K_TRY(b2k_resolve(ctx, p, &rp));
    B2K_TRY(b2k_resolve(ctx, q, &rq));
    if (rx.n != rr.n || rx.n != rp.n || rx.n != rq.n) return b2k_fail(ctx, B2K_EDIM, "cg_step: length mismatch");
    B2K_TRY(b2k_vec_axpby(ctx, p, r, 1.0, beta));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rp, rq, a0, a1, shifted, &rp, 0));
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 1, rp.sharded));
    const int grid = grid_for(ctx, rx.n, 8);
    if (ctx->dtype == B2K_F64)
        k_cg_xr<double><<<grid, BT, 0, ctx->stream>>>((double*)rx.ptr, (double*)rr.ptr, (const double*)rp.ptr,
                                                      (const double*)rq.ptr, rx.n, rho, ctx->d_res,
                                                      ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, CgChain{});
    else
        k_cg_xr<float><<<grid, BT, 0, ctx->stream>>>((float*)rx.ptr, (float*)rr.ptr, (const float*)rp.ptr,
                                                     (const float*)rq.ptr, rx.n, rho, ctx->d_res,
                                                     ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, CgChain{});
    B2K_LAUNCH_CHECK(ctx);
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + 1, 1, rx.sharded));
    B2K_TRY(b2k_fetch_results(ctx, 2, 0));
    *pq_out = ctx->h_res[0];
    *normr_out = sqrt(ctx->h_res[1]);
    return B2K_OK;
}


// Up to `nsteps` CG iterations (cg.jl:62-101, every iteration after the first) enqueued back to back with rho,
// beta, <p,q> and ||r|| kept on the device: three launches per iteration (p <- r + beta p; q = A p with <p,q> in
// its epilogue; x, r update + ||r||) and ONE host synchronisation per call.  The reference tests ||r|| < tol
// after every iteration; so does the last kernel of each iteration, and the launches behind a hit do nothing.
// pq_out / normr_out get one entry per completed iteration; the iteration that reported ||r|| < tol is the last.
extern "C" int32_t b2k_cg_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec p, b2k_vec q,
                                double a0, double a1, double beta, double rho, double tol, int32_t nsteps,
                                double* pq_out, double* normr_out, int32_t* steps_done) {
    if (!ctx || !op || !pq_out || !normr_out || !steps_done || nsteps < 1) return B2K_EINVAL;
    *steps_done = 0;
    if (nsteps > B2K_MAX_CHAIN) nsteps = B2K_MAX_CHAIN;
    VecRef rx, rr, rp, rq;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, r, &rr));
    B2K_TRY(b2k_resolve(ctx, p, &rp));
    B2K_TRY(b2k_resolve(ctx, q, &rq));
    if (rx.n != rr.n || rx.n != rp.n || rx.n != rq.n) return b2k_fail(ctx, B2K_EDIM, "cg_chain: length mismatch");
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "cg_chain: single-GPU contexts (use b2k_cg_step)");
    int64_t orows = 0, ocols = 0;
    int32_t okind = -1;
    B2K_TRY(b2k_op_info(op, &orows, &ocols, nullptr, &okind));
    if (okind != 0) return b2k_fail(ctx, B2K_ENOTSUP, "cg_chain: CSR operators only");
    double* state = ctx->d_steps;                       // {rho, beta}
    double* rec0 = ctx->d_steps + B2K_REC;
    int* d_stop = reinterpret_cast<int*>(ctx->d_sync + B2K_SYNC_STOP);
    const double seed[2] = {rho, beta};
    B2K_TRY(b2k_put_coef(ctx, seed, 2, 0));
    B2K_CUDA(ctx, cudaMemcpyAsync(state, ctx->d_coef, 2 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    B2K_CUDA(ctx, cudaMemsetAsync(d_stop, 0, sizeof(int), ctx->stream));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    const int grid = grid_for(ctx, rx.n, 8);
    for (int32_t i = 0; i < nsteps; ++i) {
        double* rec = rec0 + (size_t)B2K_REC * i;
        if (ctx->dtype == B2K_F64)
            k_xpby_dev<double><<<grid, BT, 0, ctx->stream>>>((double*)rp.ptr, (const double*)rr.ptr, rx.n, state + 1, d_stop);
        else
            k_xpby_dev<float><<<grid, BT, 0, ctx->stream>>>((float*)rp.ptr, (const float*)rr.ptr, rx.n, state + 1, d_stop);
        B2K_LAUNCH_CHECK(ctx);
        SpmvFuse fz;
        memset(&fz, 0, sizeof(fz));
        fz.stop = d_stop;
        B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rp, rq, a0, a1, shifted, &rp, ctx->d_res, &fz));
        CgChain ch;
        ch.state = state; ch.rec = rec; ch.stop = d_stop; ch.tol = tol;
        if (ctx->dtype == B2K_F64)
            k_cg_xr<double><<<grid, BT, 0, ctx->stream>>>((double*)rx.ptr, (double*)rr.ptr, (const double*)rp.ptr,
                                                          (const double*)rq.ptr, rx.n, 0.0, ctx->d_res,
                                                          ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, ch);
        else
            k_cg_xr<float><<<grid, BT, 0, ctx->stream>>>((float*)rx.ptr, (float*)rr.ptr, (const float*)rp.ptr,
                                                         (const float*)rq.ptr, rx.n, 0.0, ctx->d_res,
                                                         ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, ch);
        B2K_LAUNCH_CHECK(ctx);
    }
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, rec0, sizeof(double) * B2K_REC * nsteps, cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    int32_t d = nsteps;
    for (int32_t i = 0; i < nsteps; ++i) {
        pq_out[i] = ctx->h_res[(size_t)B2K_REC * i];
        normr_out[i] = ctx->h_res[(size_t)B2K_REC * i + 1];
        if (normr_out[i] < tol) { d = i + 1; break; }
    }
    *steps_done = d;
    return B2K_OK;
}

// BiCGStab iteration in two calls with one host round trip each — src/linsolve/bicgstab.jl:97-117 and
// :139-150.  The half-step convergence test (:118) sits between them, on the host, as in the reference.
//   half: p <- r + beta*(p - omega*v)  [first != 0: p <- r];  v <- (a0 + a1 A) p with sigma = <rs, v> taken
//         from the SpMV pass;  alpha = rho/sigma on the device;  s <- r - alpha*v with ||s||.
//   full: t <- (a0 + a1 A) s with <t, s> from the SpMV pass;  <t, t>;  omega = <t,s>/<t,t> on the device;
//         x <- x + alpha*p + omega*s;  r <- s - omega*t with ||r|| and the next rho = <rs, r>.
extern "C" int32_t b2k_bicgstab_half(b2k_ctx* ctx, const b2k_op* op, b2k_vec rs, b2k_vec r, b2k_vec p, b2k_vec v,
                                     b2k_vec s, double a0, double a1, double beta, double omega, double rho,
                                     int32_t first, double* sigma_out, double* norms_out) {
    if (!ctx || !op || !sigma_out || !norms_out) return B2K_EINVAL;
    VecRef rrs, rr, rp, rv, rsv;
    B2K_TRY(b2k_resolve(ctx, rs, &rrs));
    B2K_TRY(b2k_resolve(ctx, r, &rr));
    B2K_TRY(b2k_resolve(ctx, p, &rp));
    B2K_TRY(b2k_resolve(ctx, v, &rv));
    B2K_TRY(b2k_resolve(ctx, s, &rsv));
    const int64_t n = rr.n;
    if (rrs.n != n || rp.n != n || rv.n != n || rsv.n != n)
        return b2k_fail(ctx, B2K_EDIM, "bicgstab_half: length mismatch");
    const int grid = grid_for(ctx, n, 8);
    if (first) {
        B2K_TRY(b2k_vec_copy(ctx, p, r));
    } else if (ctx->dtype == B2K_F64) {
        k_bicg_p<double><<<grid, BT, 0, ctx->stream>>>((double*)rp.ptr, (const double*)rr.ptr,
                                                       (const double*)rv.ptr, n, beta, omega, BicgChain{});
        B2K_LAUNCH_CHECK(ctx);
    } else {
        k_bicg_p<float><<<grid, BT, 0, ctx->stream>>>((float*)rp.ptr, (const float*)rr.ptr, (const float*)rv.ptr,
                                                      n, (float)beta, (float)omega, BicgChain{});
        B2K_LAUNCH_CHECK(ctx);
    }
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rp, rv, a0, a1, shifted, &rrs, 0));      // d_res[0] = sigma
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 1, rr.sharded));
    if (ctx->dtype == B2K_F64)
        k_bicg_s<double><<<grid, BT, 0, ctx->stream>>>((double*)rsv.ptr, (const double*)rr.ptr,
                                                       (const double*)rv.ptr, n, rho, ctx->d_res, ctx->d_part_s,
                                                       ctx->d_sync, ctx->d_res + 1, BicgChain{});
    else
        k_bicg_s<float><<<grid, BT, 0, ctx->stream>>>((float*)rsv.ptr, (const float*)rr.ptr, (const float*)rv.ptr,
                                                      n, rho, ctx->d_res, ctx->d_part_s, ctx->d_sync,
                                                      ctx->d_res + 1, BicgChain{});
    B2K_LAUNCH_CHECK(ctx);
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + 1, 1, rr.sharded));
    B2K_TRY(b2k_fetch_results(ctx, 2, 0));
    *sigma_out = ctx->h_res[0];
    *norms_out = sqrt(ctx->h_res[1]);
    return B2K_OK;
}

extern "C" int32_t b2k_bicgstab_full(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec rs, b2k_vec p,
                                     b2k_vec s, b2k_vec t, double a0, double a1, double alpha,
                                     double* omega_out, double* normr_out, double* rho_out) {
    if (!ctx || !op || !omega_out || !normr_out || !rho_out) return B2K_EINVAL;
    VecRef rx, rr, rrs, rp, rsv, rt;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, r, &rr));
    B2K_TRY(b2k_resolve(ctx, rs, &rrs));
    B2K_TRY(b2k_resolve(ctx, p, &rp));
    B2K_TRY(b2k_resolve(ctx, s, &rsv));
    B2K_TRY(b2k_resolve(ctx, t, &rt));
    const int64_t n = rr.n;
    if (rx.n != n || rrs.n != n || rp.n != n || rsv.n != n || rt.n != n)
        return b2k_fail(ctx, B2K_EDIM, "bicgstab_full: length mismatch");
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rsv, rt, a0, a1, shifted, &rsv, 0));     // d_res[0] = <s, t>
    B2K_TRY(b2k_enqueue_dot(ctx, rt.ptr, rt.ptr, n, nullptr, -1, 1, -1));       // d_res[1] = <t, t>
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 2, rr.sharded));
    const int grid = grid_for(ctx, n, 8);
    if (ctx->dtype == B2K_F64)
        k_bicg_xr<double><<<grid, BT, 0, ctx->stream>>>((double*)rx.ptr, (double*)rr.ptr, (const double*)rrs.ptr,
                                                        (const double*)rp.ptr, (const double*)rsv.ptr,
                                                        (const double*)rt.ptr, n, alpha, ctx->d_res,
                                                        ctx->d_res + 1, ctx->d_part_s, ctx->d_sync,
                                                        ctx->d_res + 2, BicgChain{});
    else
        k_bicg_xr<float><<<grid, BT, 0, ctx->stream>>>((float*)rx.ptr, (float*)rr.ptr, (const float*)rrs.ptr,
                                                       (const float*)rp.ptr, (const float*)rsv.ptr,
                                                       (const float*)rt.ptr, n, (float)alpha, ctx->d_res,
                                                       ctx->d_res + 1, ctx->d_part_s, ctx->d_sync,
                                                       ctx->d_res + 2, BicgChain{});
    B2K_LAUNCH_CHECK(ctx);
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + 2, 2, rr.sharded));
    B2K_TRY(b2k_fetch_results(ctx, 4, 0));
    *omega_out = ctx->h_res[0] / ctx->h_res[1];
    *normr_out = sqrt(ctx->h_res[2]);
    *rho_out = ctx->h_res[3];
    return B2K_OK;
}

// Up to `nsteps` BiCGStab iterations (bicgstab.jl:95-171, every iteration after the first) enqueued back to back:
// rho, rho_old, alpha, omega live on the device, the two convergence tests of an iteration (:118 after the half
// step, :152 after the full step) are made by the kernels that produce the norms, and the launches behind a hit do
// nothing.  ONE host synchronisation per call instead of two per iteration.  rec_out gets 8 doubles per completed
// iteration: {rho, sigma, alpha, ||s||, omega, ||r||, next rho, stop code (0: none, 1: ||s|| < tol — the full step
// of that iteration has NOT run —, 2: ||r|| < tol)}.  The host handles what follows a hit (explicit residual).
extern "C" int32_t b2k_bicgstab_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec rs, b2k_vec p,
                                      b2k_vec v, b2k_vec s, b2k_vec t, double a0, double a1, double rho,
                                      double rho_old, double alpha, double omega, double tol, int32_t nsteps,
                                      double* rec_out, int32_t* steps_done) {
    if (!ctx || !op || !rec_out || !steps_done || nsteps < 1) return B2K_EINVAL;
    *steps_done = 0;
    if (nsteps > B2K_MAX_CHAIN - 1) nsteps = B2K_MAX_CHAIN - 1;
    VecRef rx, rr, rrs, rp, rv, rsv, rt;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, r, &rr));
    B2K_TRY(b2k_resolve(ctx, rs, &rrs));
    B2K_TRY(b2k_resolve(ctx, p, &rp));
    B2K_TRY(b2k_resolve(ctx, v, &rv));
    B2K_TRY(b2k_resolve(ctx, s, &rsv));
    B2K_TRY(b2k_resolve(ctx, t, &rt));
    const int64_t n = rr.n;
    if (rx.n != n || rrs.n != n || rp.n != n || rv.n != n || rsv.n != n || rt.n != n)
        return b2k_fail(ctx, B2K_EDIM, "bicgstab_chain: length mismatch");
    if (ctx->nranks > 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "bicgstab_chain: single-GPU contexts (use b2k_bicgstab_half/_full)");
    int64_t orows = 0, ocols = 0;
    int32_t okind = -1;
    B2K_TRY(b2k_op_info(op, &orows, &ocols, nullptr, &okind));
    if (okind != 0) return b2k_fail(ctx, B2K_ENOTSUP, "bicgstab_chain: CSR operators only");
    double* st = ctx->d_steps;                          // {rho, rho_old, alpha, omega}
    double* rec0 = ctx->d_steps + B2K_REC;
    int* d_stop = reinterpret_cast<int*>(ctx->d_sync + B2K_SYNC_STOP);
    const double seed[4] = {rho, rho_old, alpha, omega};
    B2K_TRY(b2k_put_coef(ctx, seed, 4, 0));
    B2K_CUDA(ctx, cudaMemcpyAsync(st, ctx->d_coef, 4 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    B2K_CUDA(ctx, cudaMemsetAsync(rec0, 0, sizeof(double) * B2K_REC * nsteps, ctx->stream));
    B2K_CUDA(ctx, cudaMemsetAsync(d_stop, 0, sizeof(int), ctx->stream));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    const int grid = grid_for(ctx, n, 8);
    const bool f64 = ctx->dtype == B2K_F64;
    SpmvFuse fz;
    memset(&fz, 0, sizeof(fz));
    fz.stop = d_stop;
    for (int32_t i = 0; i < nsteps; ++i) {
        BicgChain ch;
        ch.st = st; ch.rec = rec0 + (size_t)B2K_REC * i; ch.stop = d_stop; ch.tol = tol;
        if (f64)
            k_bicg_p<double><<<grid, BT, 0, ctx->stream>>>((double*)rp.ptr, (const double*)rr.ptr,
                                                           (const double*)rv.ptr, n, 0.0, 0.0, ch);
        else
            k_bicg_p<float><<<grid, BT, 0, ctx->stream>>>((float*)rp.ptr, (const float*)rr.ptr,
                                                          (const float*)rv.ptr, n, 0.f, 0.f, ch);
        B2K_LAUNCH_CHECK(ctx);
        B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rp, rv, a0, a1, shifted, &rrs, ctx->d_res, &fz));   // sigma
        if (f64)
            k_bicg_s<double><<<grid, BT, 0, ctx->stream>>>((double*)rsv.ptr, (const double*)rr.ptr,
                                                           (const double*)rv.ptr, n, 0.0, ctx->d_res, ctx->d_part_s,
                                                           ctx->d_sync, ctx->d_res + 1, ch);
        else
            k_bicg_s<float><<<grid, BT, 0, ctx->stream>>>((float*)rsv.ptr, (const float*)rr.ptr,
                                                          (const float*)rv.ptr, n, 0.0, ctx->d_res, ctx->d_part_s,
                                                          ctx->d_sync, ctx->d_res + 1, ch);
        B2K_LAUNCH_CHECK(ctx);
        B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rsv, rt, a0, a1, shifted, &rsv, ctx->d_res, &fz));  // <s, t>
        B2K_TRY(b2k_enqueue_dot(ctx, rt.ptr, rt.ptr, n, nullptr, -1, 1, -1));                        // <t, t>
        if (f64)
            k_bicg_xr<double><<<grid, BT, 0, ctx->stream>>>((double*)rx.ptr, (double*)rr.ptr, (const double*)rrs.ptr,
                                                            (const double*)rp.ptr, (const double*)rsv.ptr,
                                                            (const double*)rt.ptr, n, 0.0, ctx->d_res,
                                                            ctx->d_res + 1, ctx->d_part_s, ctx->d_sync,
                                                            ctx->d_res + 2, ch);
        else
            k_bicg_xr<float><<<grid, BT, 0, ctx->stream>>>((float*)rx.ptr, (float*)rr.ptr, (const float*)rrs.ptr,
                                                           (const float*)rp.ptr, (const float*)rsv.ptr,
                                                           (const float*)rt.ptr, n, 0.f, ctx->d_res,
                                                           ctx->d_res + 1, ctx->d_part_s, ctx->d_sync,
                                                           ctx->d_res + 2, ch);
        B2K_LAUNCH_CHECK(ctx);
    }
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, rec0, sizeof(double) * B2K_REC * nsteps, cudaMemcpyDeviceToHost,
                                  ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    int32_t d = nsteps;
    for (int32_t i = 0; i < nsteps; ++i)
        if (ctx->h_res[(size_t)B2K_REC * i + 7] != 0.0) { d = i + 1; break; }
    memcpy(rec_out, ctx->h_res, sizeof(double) * B2K_REC * d);
    *steps_done = d;
    return B2K_OK;
}
