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
// STOP (the MGS sweeps of b2k_lsmr_chain): the launch does nothing once *stop is raised.
template <typename T, bool UPDATE, bool NORM, bool STOP = false>
__global__ void __launch_bounds__(BT)
k_dot(const T* __restrict__ q, T* __restrict__ x, int64_t n, const T* __restrict__ qprev,
      const double* __restrict__ sprev, double* __restrict__ part, unsigned* __restrict__ ticket,
      double* __restrict__ out, double* __restrict__ accum_into, int hints, const int* stop) {
    __shared__ double red[32];
    __shared__ bool last;
    if constexpr (STOP) {
        if (*reinterpret_cast<const volatile int*>(stop)) return;
    }
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
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT, [&](int, double tot) {
        *out = tot;
        if (accum_into) *accum_into += tot;
    });
}

// final fix-up: x <- x - s*q with s = d_res[src] (tail of the pipelined MGS sweep)
template <typename T, bool STOP = false>
__global__ void __launch_bounds__(BT)
k_axpy_dev(T* __restrict__ x, const T* __restrict__ q, const double* __restrict__ s, int64_t n, const int* stop) {
    if constexpr (STOP) {
        if (*reinterpret_cast<const volatile int*>(stop)) return;
    }
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
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT, [&](int, double tot) {
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
    });
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
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT, [&](int k, double tot) { out[k] = tot; });
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
    finish_sums<2>(blk, part, ticket, red, &last, BT, [&](int k, double tot) { out[k] = tot; });
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

// ---- MINRES (Paige & Saunders 1975, Lanczos + Givens QR; b2k_minres_chain) ----
// Scalar state of the recurrence, on the device for the length of a call.  At the start of iteration k:
// p_cur = p_{k-1} (unnormalised, v_k = p_cur * INVB), p_prev = p_{k-2} (v_{k-1} = p_prev * INVB_PREV).
// P* = the direction / solution update of iteration k-1, which needs gamma_{k-1} and so beta_k: it is applied by the
// kernel of iteration k (or by the flush launch); PEND says there is one.  DONE counts the iterations this call has
// run: it fixes which buffer plays which role (the roles rotate with every iteration, skipped launches do not count).
enum { MR_BETA = 0, MR_INVB, MR_INVB_PREV, MR_C, MR_S, MR_DBAR, MR_EPS, MR_PHIBAR,
       MR_PDELTA, MR_PEPS, MR_PINVG, MR_PPHI, MR_PEND, MR_DONE, MR_NSTATE = 16 };

struct MinresChain {
    double* st;
    double* rec;            // {alpha, beta_{k+1}, gamma, phi, |phibar|, stop code, delta, eps_k}
    int* stop;
    const double* alpha;    // <v_k, q> from the SpMV epilogue
    double tol;
};

// One pass per MINRES iteration k (LANCZOS), after q = (a0 + a1 A) v_k:
//   p_k = (q - alpha v_k) - beta_k v_{k-1}, sum p_k^2              [two add!! of the literal driver]
//   d_{k-1} = ((v_{k-1} - delta d_{k-2}) - eps d_{k-3}) / gamma    [two add!!, one scale!!]
//   x += phi d_{k-1}                                               [one add!!]
// v_{k-1} = rn(p_prev * 1/beta_{k-1}) and v_k are formed in registers exactly as scale!! rounds them; p_k goes over
// p_{k-2}, d_{k-1} over d_{k-3}.  Reads q, p_cur, p_prev, d1, d2, x and writes p, d, x: 9 W.  The last CTA then runs the
// scalar recurrence of iteration k in Float64, every product and sum rounded on its own (no fma contraction), so a
// host restatement in plain double arithmetic gives the same bits.
// !LANCZOS is the flush launch: only the pending direction / solution update, whether or not the chain has stopped.
template <typename T, bool LANCZOS>
__global__ void __launch_bounds__(BT)
k_minres_step(T* __restrict__ x, T* pA, T* pB, const T* __restrict__ q, T* dA, T* dB, int64_t n,
              double* __restrict__ part, unsigned* __restrict__ ticket, const MinresChain ch) {
    __shared__ double red[32];
    __shared__ bool last;
    if (LANCZOS && *reinterpret_cast<const volatile int*>(ch.stop)) return;
    const volatile double* st = ch.st;
    const bool pend = st[MR_PEND] != 0.0;
    if (!LANCZOS && !pend) return;
    const int done = (int)st[MR_DONE];
    T* const pp = (done & 1) ? pB : pA;
    const T* const pc = (done & 1) ? pA : pB;
    const bool dswap = done > 0 && ((done - 1) & 1);        // direction updates applied so far: done - 1
    const T* const d1 = dswap ? dB : dA;
    T* const d2 = dswap ? dA : dB;
    const double alpha = LANCZOS ? *ch.alpha : 0.0, beta = st[MR_BETA], invb = st[MR_INVB];
    const T ip = (T)st[MR_INVB_PREV], ic = (T)invb, na = (T)(-alpha), nb = (T)(-beta);
    const T nd = (T)(-st[MR_PDELTA]), ne = (T)(-st[MR_PEPS]), ig = (T)st[MR_PINVG], ph = (T)st[MR_PPHI];
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    T acc = 0;
    auto each = [&](T pv, T cv, T qv, T av, T bv, T& xv, T& pout, T& dout) {
        const T vp = mul_rn(pv, ip);
        if (LANCZOS) {
            pout = fma(nb, vp, fma(na, mul_rn(cv, ic), qv));
            acc = fma(pout, pout, acc);
        }
        if (pend) {
            dout = mul_rn(fma(ne, bv, fma(nd, av, vp)), ig);
            xv = fma(ph, dout, xv);
        }
    };
    B2K_TRIP(2) {
        T pv[2][V], cv[2][V] = {}, qv[2][V] = {}, av[2][V] = {}, bv[2][V] = {}, xv[2][V] = {};
        B2K_EACH(2, u, i) {
            vload<T>(pp + i * V, pv[u]);
            if (LANCZOS) {
                vload<T>(pc + i * V, cv[u]);
                vload<T>(q + i * V, qv[u]);
            }
            if (pend) {
                vload<T>(d1 + i * V, av[u]);
                vload<T>(d2 + i * V, bv[u]);
                vload<T>(x + i * V, xv[u]);
            }
        }
        B2K_EACH(2, u, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) each(pv[u][j], cv[u][j], qv[u][j], av[u][j], bv[u][j], xv[u][j], pv[u][j], bv[u][j]);
            if (LANCZOS) vstore<T>(pp + i * V, pv[u]);
            if (pend) {
                vstore<T>(d2 + i * V, bv[u]);
                vstore<T>(x + i * V, xv[u]);
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        T xv = pend ? x[i] : (T)0, pout = 0, dout = 0;
        each(pp[i], LANCZOS ? pc[i] : (T)0, LANCZOS ? q[i] : (T)0, pend ? d1[i] : (T)0, pend ? d2[i] : (T)0, xv, pout, dout);
        if (LANCZOS) pp[i] = pout;
        if (pend) {
            d2[i] = dout;
            x[i] = xv;
        }
    }
    if (!LANCZOS) return;
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT, [&](int, double tot) {
        const double bn = sqrt(tot);                                        // beta_{k+1}
        const double c0 = st[MR_C], s0 = st[MR_S], dbar = st[MR_DBAR], eps = st[MR_EPS], phibar = st[MR_PHIBAR];
        const double delta = __dadd_rn(__dmul_rn(c0, dbar), __dmul_rn(s0, alpha));
        const double gbar = __dadd_rn(__dmul_rn(s0, dbar), -__dmul_rn(c0, alpha));
        const double gamma = sqrt(__dadd_rn(__dmul_rn(gbar, gbar), __dmul_rn(bn, bn)));
        // gamma == 0: the shifted operator is singular on the Krylov space.  The pending update is kept, with zero
        // weights (d_k = 0, x unchanged), so the roles rotate the same way on every exit.
        const bool sing = gamma == 0.0;
        const double c = sing ? 0.0 : __ddiv_rn(gbar, gamma), s = sing ? 0.0 : __ddiv_rn(bn, gamma);
        const double phi = sing ? 0.0 : __dmul_rn(c, phibar), phibar_n = sing ? phibar : __dmul_rn(s, phibar);
        const double code = sing ? 2.0 : (fabs(phibar_n) < ch.tol ? 1.0 : (bn == 0.0 ? 3.0 : 0.0));
        double* w = ch.st;
        w[MR_INVB_PREV] = invb;
        w[MR_BETA] = bn;
        w[MR_INVB] = __ddiv_rn(1.0, bn);
        w[MR_C] = c; w[MR_S] = s;
        w[MR_DBAR] = -__dmul_rn(c0, bn);
        w[MR_EPS] = __dmul_rn(s0, bn);
        w[MR_PHIBAR] = phibar_n;
        w[MR_PDELTA] = delta; w[MR_PEPS] = eps;
        w[MR_PINVG] = sing ? 0.0 : __ddiv_rn(1.0, gamma);
        w[MR_PPHI] = phi;
        w[MR_PEND] = 1.0;
        w[MR_DONE] = (double)(done + 1);
        ch.rec[0] = alpha; ch.rec[1] = bn; ch.rec[2] = gamma; ch.rec[3] = phi; ch.rec[4] = fabs(phibar_n);
        ch.rec[5] = code; ch.rec[6] = delta; ch.rec[7] = eps;
        if (code != 0.0) *ch.stop = 1;
    });
}

// ---- LSMR (lsmr.jl:61-149; b2k_lsmr_chain) ----
// add!!(y, x, 1, b) as k_axpby rounds it: b == 0 gives x (MODE 0), otherwise fma(1, x, rn(b y)) (MODE 1 and 2).
template <typename T>
__device__ __forceinline__ T axpy1_rn(T x, T b, bool bzero, T y) {
    return bzero ? x : fma((T)1, x, mul_rn(b, y));
}

// sqrt(a^2 + b^2) with every product and sum rounded on its own (the host restatement's plain double arithmetic);
// overflows once a or b exceeds about 1.3e154, where hypot would not
__device__ __forceinline__ double hyp_rn(double a, double b) {
    return __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
}

// The scalar half of one LSMR iteration (lsmr.jl:92-113 with lambda), one thread, Float64, in the operation order of
// lssolve.py::_lsmr (so a host restatement in plain double arithmetic gives the same bits).  nrm2 = ||v~||^2 of this
// iteration (ignored when beta <= tol: alpha and v are kept).  Writes the record of the iteration and the state the
// pending updates and the next iteration read; raises the stop flags on a stop code.
__device__ void lsmr_recurrence(const LsmrDev& d, double nrm2) {
    volatile double* w = d.st;
    const bool bskip = w[LS_BSKIP] != 0.0;
    const double beta = w[LS_BETA];
    const double alpha = bskip ? w[LS_ALPHA] : __dsqrt_rn(nrm2);
    const double lam = w[LS_LAM], rhoold = w[LS_RHO], rhobarold = w[LS_RHOBAR];
    const double cbar0 = w[LS_CBAR], sbar0 = w[LS_SBAR], zetabar0 = w[LS_ZETABAR];
    const double alphahat = hyp_rn(w[LS_ALPHABAR], lam);
    const double rho = hyp_rn(alphahat, beta);
    const double c = __ddiv_rn(alphahat, rho), s = __ddiv_rn(beta, rho);
    const double theta = __dmul_rn(s, alpha);
    const double alphabar = __dmul_rn(c, alpha);
    const double thetabar = __dmul_rn(sbar0, rho);
    const double cbarrho = __dmul_rn(cbar0, rho);
    const double rhobar = hyp_rn(cbarrho, theta);
    const double cbar = __ddiv_rn(cbarrho, rhobar), sbar = __ddiv_rn(theta, rhobar);
    const double zeta = __dmul_rn(cbar, zetabar0);
    const double zetabar = __dmul_rn(-sbar, zetabar0);
    const double g = __ddiv_rn(__dmul_rn(-thetabar, rho), __dmul_rn(rhoold, rhobarold));
    const double cz = __ddiv_rn(zeta, __dmul_rn(rho, rhobar));
    const bool askip = !bskip && !(alpha > d.tol);
    const bool finite = isfinite(alpha) && isfinite(beta) && isfinite(rho) && isfinite(rhobar) && isfinite(g) &&
                        isfinite(cz) && isfinite(zetabar);
    const double code = fabs(zetabar) <= d.tol ? 1.0 : bskip ? 2.0 : askip ? 3.0 : !finite ? 4.0 : 0.0;
    const int done = (int)w[LS_DONE];
    double* rec = d.rec0 + (size_t)LS_REC * done;
    rec[0] = alpha; rec[1] = beta; rec[2] = rho; rec[3] = rhobar; rec[4] = theta; rec[5] = zeta; rec[6] = fabs(zetabar);
    rec[7] = code; rec[8] = bskip ? 0.0 : 1.0; rec[9] = alphabar; rec[10] = cbar; rec[11] = sbar; rec[12] = g;
    rec[13] = cz;
    w[LS_ALPHA] = alpha; w[LS_ALPHABAR] = alphabar; w[LS_RHO] = rho; w[LS_RHOBAR] = rhobar; w[LS_CBAR] = cbar;
    w[LS_SBAR] = sbar; w[LS_THETA] = theta; w[LS_ZETABAR] = zetabar;
    w[LS_INVA] = (bskip || askip) ? 1.0 : __ddiv_rn(1.0, alpha);
    w[LS_G] = g; w[LS_CZ] = cz; w[LS_ASKIP] = askip ? 1.0 : 0.0;
    w[LS_DONE] = (double)(done + 1);
    if (code != 0.0) {
        *d.stop = 1;
        *d.skip = 1;
    }
}

// The u side of iteration k (m rows), after Av = A v_k:
//   pend:  Ah-bar <- add!!(Ah-bar, Ah, 1, g);  r <- add!!(r, Ah-bar, -zeta/(rho rhobar))   [iteration k-1's tail]
//          Ah <- add!!(Ah, Av, 1, -theta/rho);  u~ <- add!!(Av, rn(u~ (1/beta)), -alpha), sum u~^2
// u~ stays unnormalised; the last CTA writes beta_{k+1}, 1/beta_{k+1} and the A'-side skip flag (beta <= tol).
// FLUSH: only the pending tail, and u <- rn(u~ (1/beta)) unless beta <= tol (the reference leaves u unscaled then).
template <typename T, bool FLUSH>
__global__ void __launch_bounds__(BT)
k_lsmr_m(T* __restrict__ r, T* __restrict__ Ah, T* __restrict__ Ahb, T* __restrict__ u, const T* __restrict__ Av,
         int64_t n, bool pend, double* __restrict__ part, unsigned* __restrict__ ticket, const LsmrDev d) {
    __shared__ double red[32];
    __shared__ bool last;
    if (!FLUSH && *reinterpret_cast<const volatile int*>(d.stop)) return;
    const volatile double* st = d.st;
    const double gd = st[LS_G], tr = __ddiv_rn(-st[LS_THETA], st[LS_RHO]);
    const T g = (T)gd, ncz = (T)(-st[LS_CZ]), ntr = (T)tr, na = (T)(-st[LS_ALPHA]), ib = (T)st[LS_INVB];
    const bool gz = gd == 0.0, tz = tr == 0.0;
    const bool su = !FLUSH || st[LS_BSKIP] == 0.0;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    T acc = 0;
    auto each = [&](T& rv, T& ahv, T& hbv, T& uv, T avv) {
        if (pend) {
            hbv = axpy1_rn(ahv, g, gz, hbv);
            rv = fma(ncz, hbv, rv);
        }
        if (!FLUSH) {
            ahv = axpy1_rn(avv, ntr, tz, ahv);
            uv = fma(na, mul_rn(uv, ib), avv);
            acc = fma(uv, uv, acc);
        } else if (su) {
            uv = mul_rn(uv, ib);
        }
    };
    B2K_TRIP(2) {
        T rv[2][V] = {}, ahv[2][V], hbv[2][V] = {}, uv[2][V], avv[2][V] = {};
        B2K_EACH(2, q, i) {
            vload<T>(Ah + i * V, ahv[q]);
            vload<T>(u + i * V, uv[q]);
            if (pend) {
                vload<T>(r + i * V, rv[q]);
                vload<T>(Ahb + i * V, hbv[q]);
            }
            if (!FLUSH) vload<T>(Av + i * V, avv[q]);
        }
        B2K_EACH(2, q, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) each(rv[q][j], ahv[q][j], hbv[q][j], uv[q][j], avv[q][j]);
            if (pend) {
                vstore<T>(r + i * V, rv[q]);
                vstore<T>(Ahb + i * V, hbv[q]);
            }
            if (!FLUSH) vstore<T>(Ah + i * V, ahv[q]);
            if (su) vstore<T>(u + i * V, uv[q]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        T rv = pend ? r[i] : (T)0, ahv = Ah[i], hbv = pend ? Ahb[i] : (T)0, uv = u[i];
        each(rv, ahv, hbv, uv, FLUSH ? (T)0 : Av[i]);
        if (pend) {
            r[i] = rv;
            Ahb[i] = hbv;
        }
        if (!FLUSH) Ah[i] = ahv;
        if (su) u[i] = uv;
    }
    if (FLUSH) return;
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT, [&](int, double tot) {
        const double beta = __dsqrt_rn(tot);
        const bool bskip = !(beta > d.tol);
        double* w = d.st;
        w[LS_BETA] = beta;
        w[LS_INVB] = __ddiv_rn(1.0, beta);
        w[LS_BSKIP] = bskip ? 1.0 : 0.0;
        *d.skip = bskip ? 1 : 0;
    });
}

// The v side of iteration k (n rows), after y = A' u_{k+1} (skipped when beta <= tol).  P is v_k's ring slot; the
// operand source and y are (P, Q) in the first iteration of a call (v_k normalised in its slot, y in the spare column
// Q) and (Q, P) after it (v~_k unnormalised in Q, y in the slot v_k replaces):
//   v_k = rn(src (1/alpha_k)) -> P
//   pend: h-bar <- add!!(h-bar, h, 1, g); x <- add!!(x, h-bar, zeta/(rho rhobar)); h <- add!!(h, v_k, 1, -theta/rho)
//   unless beta <= tol: v~_{k+1} = add!!(y, v_k, -beta) -> Q
// NORM (no reorthogonalisation): sum v~_{k+1}^2, and the last CTA runs the recurrence.
template <typename T, bool NORM>
__global__ void __launch_bounds__(BT)
k_lsmr_n(T* __restrict__ x, T* __restrict__ h, T* __restrict__ hb, T* P, T* Q, int64_t n, bool swap, bool pend,
         double* __restrict__ part, unsigned* __restrict__ ticket, const LsmrDev d) {
    __shared__ double red[32];
    __shared__ bool last;
    if (*reinterpret_cast<const volatile int*>(d.stop)) return;
    const volatile double* st = d.st;
    const double gd = st[LS_G], tr = __ddiv_rn(-st[LS_THETA], st[LS_RHO]);
    const T g = (T)gd, cz = (T)st[LS_CZ], ntr = (T)tr, ia = (T)st[LS_INVA], nb = (T)(-st[LS_BETA]);
    const bool gz = gd == 0.0, tz = tr == 0.0, bskip = st[LS_BSKIP] != 0.0;
    const T* src = swap ? Q : P;
    const T* yv = swap ? P : Q;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    T acc = 0;
    auto each = [&](T sv, T y, T& xv, T& hv, T& hbv, T& vout, T& tout) {
        const T v = mul_rn(sv, ia);
        vout = v;
        if (pend) {
            hbv = axpy1_rn(hv, g, gz, hbv);
            xv = fma(cz, hbv, xv);
            hv = axpy1_rn(v, ntr, tz, hv);
        }
        if (!bskip) {
            tout = fma(nb, v, y);
            if (NORM) acc = fma(tout, tout, acc);
        }
    };
    B2K_TRIP(2) {
        T sv[2][V], y[2][V] = {}, xv[2][V] = {}, hv[2][V] = {}, hbv[2][V] = {}, vo[2][V], to[2][V] = {};
        B2K_EACH(2, q, i) {
            vload<T>(src + i * V, sv[q]);
            if (!bskip) vload<T>(yv + i * V, y[q]);
            if (pend) {
                vload<T>(x + i * V, xv[q]);
                vload<T>(h + i * V, hv[q]);
                vload<T>(hb + i * V, hbv[q]);
            }
        }
        B2K_EACH(2, q, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) each(sv[q][j], y[q][j], xv[q][j], hv[q][j], hbv[q][j], vo[q][j], to[q][j]);
            if (swap) vstore<T>(P + i * V, vo[q]);
            if (!bskip) vstore<T>(Q + i * V, to[q]);
            if (pend) {
                vstore<T>(x + i * V, xv[q]);
                vstore<T>(h + i * V, hv[q]);
                vstore<T>(hb + i * V, hbv[q]);
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        T xv = pend ? x[i] : (T)0, hv = pend ? h[i] : (T)0, hbv = pend ? hb[i] : (T)0, vo, to = 0;
        each(src[i], bskip ? (T)0 : yv[i], xv, hv, hbv, vo, to);
        if (swap) P[i] = vo;
        if (!bskip) Q[i] = to;
        if (pend) {
            x[i] = xv;
            h[i] = hv;
            hb[i] = hbv;
        }
    }
    if (!NORM) return;
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT,
                   [&](int, double tot) { lsmr_recurrence(d, tot); });
}

// alpha after the reorthogonalisation (K > 1): the CTA-ordered sum of v~^2, then the recurrence in the last CTA
template <typename T>
__global__ void __launch_bounds__(BT)
k_lsmr_alpha(const T* __restrict__ Q, int64_t n, double* __restrict__ part, unsigned* __restrict__ ticket,
             const LsmrDev d) {
    __shared__ double red[32];
    __shared__ bool last;
    if (*reinterpret_cast<const volatile int*>(d.stop)) return;
    if (d.st[LS_BSKIP] != 0.0) {             // alpha and v are kept: no sum
        if (blockIdx.x == 0 && threadIdx.x == 0) lsmr_recurrence(d, 0.0);
        return;
    }
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    T acc = 0;
    B2K_TRIP(4) {
        T a[4][V];
        B2K_EACH(4, q, i) vload<T>(Q + i * V, a[q]);
        B2K_EACH(4, q, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) acc = fma(a[q][j], a[q][j], acc);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const T t = Q[nv * V + threadIdx.x];
        acc = fma(t, t, acc);
    }
    finish_sums<1>({block_sum((double)acc, red)}, part, ticket, red, &last, BT,
                   [&](int, double tot) { lsmr_recurrence(d, tot); });
}

// The flush of the v side: the tail of the last iteration k that ran, whether or not the chain has stopped.
// v_{k+1} = rn(v~ (1/alpha)) into ring slot k % nring; beta <= tol: v is v_k, already in slot (k-1) % nring;
// alpha <= tol: v is v~ itself, left in the spare column.  Then the pending h-bar, x, h updates with that v.
template <typename T>
__global__ void __launch_bounds__(BT)
k_lsmr_flush_n(T* __restrict__ x, T* __restrict__ h, T* __restrict__ hb, T* spare, int64_t n,
               const __grid_constant__ LsmrDev d) {
    const volatile double* st = d.st;
    const int k = d.iter0 + (int)st[LS_DONE];
    const bool bskip = st[LS_BSKIP] != 0.0, askip = st[LS_ASKIP] != 0.0;
    const T* src = bskip ? (const T*)d.ring[(k - 1) % d.nring] : spare;
    T* dst = (bskip || askip) ? nullptr : (T*)d.ring[k % d.nring];
    const double gd = st[LS_G], tr = __ddiv_rn(-st[LS_THETA], st[LS_RHO]);
    const T g = (T)gd, cz = (T)st[LS_CZ], ntr = (T)tr, ia = (T)st[LS_INVA];
    const bool gz = gd == 0.0, tz = tr == 0.0;
    constexpr int V = Vec16<T>::N;
    const int64_t nv = n / V;
    const int64_t stride = (int64_t)gridDim.x * BT;
    auto each = [&](T sv, T& xv, T& hv, T& hbv, T& vout) {
        const T v = mul_rn(sv, ia);
        vout = v;
        hbv = axpy1_rn(hv, g, gz, hbv);
        xv = fma(cz, hbv, xv);
        hv = axpy1_rn(v, ntr, tz, hv);
    };
    B2K_TRIP(2) {
        T sv[2][V], xv[2][V], hv[2][V], hbv[2][V], vo[2][V];
        B2K_EACH(2, q, i) {
            vload<T>(src + i * V, sv[q]);
            vload<T>(x + i * V, xv[q]);
            vload<T>(h + i * V, hv[q]);
            vload<T>(hb + i * V, hbv[q]);
        }
        B2K_EACH(2, q, i) {
#pragma unroll
            for (int j = 0; j < V; ++j) each(sv[q][j], xv[q][j], hv[q][j], hbv[q][j], vo[q][j]);
            if (dst) vstore<T>(dst + i * V, vo[q]);
            vstore<T>(x + i * V, xv[q]);
            vstore<T>(h + i * V, hv[q]);
            vstore<T>(hb + i * V, hbv[q]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n - nv * V)) {
        const int64_t i = nv * V + threadIdx.x;
        T xv = x[i], hv = h[i], hbv = hb[i], vo;
        each(src[i], xv, hv, hbv, vo);
        if (dst) dst[i] = vo;
        x[i] = xv;
        h[i] = hv;
        hb[i] = hbv;
    }
}

}  // namespace

// ---- LSMR chain launches (b2k_lsmr_chain, basis.cu) ----
int32_t b2k_lsmr_enqueue_m(b2k_ctx* ctx, int64_t m, void* r, void* Ah, void* Ahbar, void* u, const void* Av,
                           bool pend, bool flush, const LsmrDev& d) {
    const int grid = grid_for(ctx, m, 4);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        b2k_flag(flush, [&](auto fl) {
            k_lsmr_m<T, fl><<<grid, BT, 0, ctx->stream>>>((T*)r, (T*)Ah, (T*)Ahbar, (T*)u, (const T*)Av, m, pend,
                                                          ctx->d_part_s, ctx->d_sync, d);
        });
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t b2k_lsmr_enqueue_n(b2k_ctx* ctx, int64_t n, void* x, void* h, void* hbar, void* P, void* Q, bool swap,
                           bool pend, bool norm, const LsmrDev& d) {
    const int grid = grid_for(ctx, n, 4);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        b2k_flag(norm, [&](auto nr) {
            k_lsmr_n<T, nr><<<grid, BT, 0, ctx->stream>>>((T*)x, (T*)h, (T*)hbar, (T*)P, (T*)Q, n, swap, pend,
                                                          ctx->d_part_s, ctx->d_sync, d);
        });
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t b2k_lsmr_enqueue_alpha(b2k_ctx* ctx, int64_t n, const void* Q, const LsmrDev& d) {
    const int grid = grid_for(ctx, n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_lsmr_alpha<T><<<grid, BT, 0, ctx->stream>>>((const T*)Q, n, ctx->d_part_s, ctx->d_sync, d);
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t b2k_lsmr_enqueue_flush_n(b2k_ctx* ctx, int64_t n, void* x, void* h, void* hbar, void* spare,
                                 const LsmrDev& d) {
    const int grid = grid_for(ctx, n, 4);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_lsmr_flush_n<T><<<grid, BT, 0, ctx->stream>>>((T*)x, (T*)h, (T*)hbar, (T*)spare, n, d);
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

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
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        b2k_flag(qprev != nullptr, [&](auto upd) {
            b2k_flag(q == nullptr, [&](auto nrm) {
                b2k_flag(ctx->dot_stop != nullptr, [&](auto st) {
                    k_dot<T, upd, nrm, st><<<grid, BT, 0, ctx->stream>>>((const T*)q, (T*)x, n, (const T*)qprev, sp,
                                                                         ctx->d_part_s, ticket, out, acc,
                                                                         ctx->dot_hints, ctx->dot_stop);
                });
            });
        });
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t b2k_enqueue_axpy_dev(b2k_ctx* ctx, void* x, const void* q, int s_slot, int64_t n) {
    const int grid = grid_for(ctx, n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        b2k_flag(ctx->dot_stop != nullptr, [&](auto st) {
            k_axpy_dev<T, st><<<grid, BT, 0, ctx->stream>>>((T*)x, (const T*)q, ctx->d_res + s_slot, n, ctx->dot_stop);
        });
    });
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
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_fill_splitmix<T><<<grid, BT, 0, ctx->stream>>>((T*)r.ptr, r.n, seed, off);
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_fill(b2k_ctx* ctx, b2k_vec v, double value) {
    if (!ctx) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    if (r.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, r.n, 4);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_fill<T><<<grid, BT, 0, ctx->stream>>>((T*)r.ptr, r.n, T(value));
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_scale(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha) {
    if (!ctx) return B2K_EINVAL;
    VecRef v[2];
    B2K_TRY(b2k_resolve_vecs(ctx, "vec_scale", {y, x}, v));
    const VecRef &ry = v[0], &rx = v[1];
    if (ry.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, ry.n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_scale<T><<<grid, BT, 0, ctx->stream>>>((T*)ry.ptr, (const T*)rx.ptr, ry.n, T(alpha));
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_axpby(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha, double beta) {
    if (!ctx) return B2K_EINVAL;
    VecRef v[2];
    B2K_TRY(b2k_resolve_vecs(ctx, "vec_axpby", {y, x}, v));
    const VecRef &ry = v[0], &rx = v[1];
    if (ry.n == 0) return B2K_OK;
    // add!!(y, y, alpha, beta): y <- (beta + alpha) * y would change rounding; do it literally, reading y once
    const bool self = ry.ptr == rx.ptr;
    const int grid = grid_for(ctx, ry.n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        b2k_flag(self, [&](auto sf) {
            auto launch = [&](auto mode) {
                k_axpby<T, mode, sf><<<grid, BT, 0, ctx->stream>>>((T*)ry.ptr, sf ? nullptr : (const T*)rx.ptr,
                                                                   ry.n, T(alpha), T(beta));
            };
            if (beta == 0.0) launch(std::integral_constant<int, 0>());
            else if (beta == 1.0) launch(std::integral_constant<int, 1>());
            else launch(std::integral_constant<int, 2>());
        });
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_axpy2(b2k_ctx* ctx, b2k_vec y, b2k_vec x1, double a1, b2k_vec x2,
                                 double a2) {
    if (!ctx) return B2K_EINVAL;
    VecRef v[3];
    B2K_TRY(b2k_resolve_vecs(ctx, "vec_axpy2", {y, x1, x2}, v));
    const VecRef &ry = v[0], &r1 = v[1], &r2 = v[2];
    if (ry.ptr == r1.ptr || ry.ptr == r2.ptr)
        return b2k_fail(ctx, B2K_EINVAL, "vec_axpy2: y must not alias x1/x2");
    if (ry.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, ry.n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_axpy2<T><<<grid, BT, 0, ctx->stream>>>((T*)ry.ptr, (const T*)r1.ptr, T(a1), (const T*)r2.ptr, T(a2), ry.n);
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_basis_givens(b2k_ctx* ctx, b2k_vec q1, b2k_vec q2, double c, double s) {
    if (!ctx) return B2K_EINVAL;
    VecRef v[2];
    B2K_TRY(b2k_resolve_vecs(ctx, "basis_givens", {q1, q2}, v));
    const VecRef &r1 = v[0], &r2 = v[1];
    if (r1.ptr == r2.ptr) return b2k_fail(ctx, B2K_EINVAL, "basis_givens: q1 == q2");
    if (r1.n == 0) return B2K_OK;
    const int grid = grid_for(ctx, r1.n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_givens<T><<<grid, BT, 0, ctx->stream>>>((T*)r1.ptr, (T*)r2.ptr, r1.n, T(c), T(s));
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_inner(b2k_ctx* ctx, b2k_vec x, b2k_vec y, double* out) {
    if (!ctx || !out) return B2K_EINVAL;
    VecRef v[2];
    B2K_TRY(b2k_resolve_vecs(ctx, "vec_inner", {x, y}, v));
    const VecRef &rx = v[0], &ry = v[1];
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
    VecRef vq[2];
    B2K_TRY(b2k_resolve_vecs(ctx, "vec_orthogonalize", {v, q}, vq));
    const VecRef &rv = vq[0], &rq = vq[1];
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
        const double eps = b2k_eps(ctx);
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
    VecRef v[4];
    B2K_TRY(b2k_resolve_vecs(ctx, "cg_step", {x, r, p, q}, v));
    const VecRef &rx = v[0], &rr = v[1], &rp = v[2], &rq = v[3];
    B2K_TRY(b2k_vec_axpby(ctx, p, r, 1.0, beta));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rp, rq, a0, a1, shifted, &rp, 0));
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 1, rp.sharded));
    const int grid = grid_for(ctx, rx.n, 8);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_cg_xr<T><<<grid, BT, 0, ctx->stream>>>((T*)rx.ptr, (T*)rr.ptr, (const T*)rp.ptr, (const T*)rq.ptr, rx.n, rho,
                                                 ctx->d_res, ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, CgChain{});
    });
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
    VecRef v[4];
    B2K_TRY(b2k_resolve_vecs(ctx, "cg_chain", {x, r, p, q}, v, true));
    const VecRef &rx = v[0], &rr = v[1], &rp = v[2], &rq = v[3];
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "cg_chain: single-GPU contexts (use b2k_cg_step)");
    int64_t orows = 0, ocols = 0;
    int32_t okind = -1;
    B2K_TRY(b2k_op_info(op, &orows, &ocols, nullptr, &okind));
    if (okind != 0) return b2k_fail(ctx, B2K_ENOTSUP, "cg_chain: CSR operators only");
    B2kChain fr(ctx, B2K_REC);                          // state {rho, beta}
    const double seed[2] = {rho, beta};
    B2K_TRY(fr.seed(seed, 2, 0));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    const int grid = grid_for(ctx, rx.n, 8);
    B2K_TRY(fr.enqueue([&]() -> int32_t {
        for (int32_t i = 0; i < nsteps; ++i) {
            const CgChain ch{fr.st, fr.rec0 + (size_t)B2K_REC * i, fr.stop, tol};
            b2k_dispatch(ctx, [&](auto t) {
                using T = decltype(t);
                k_xpby_dev<T><<<grid, BT, 0, ctx->stream>>>((T*)rp.ptr, (const T*)rr.ptr, rx.n, fr.st + 1, fr.stop);
            });
            B2K_LAUNCH_CHECK(ctx);
            SpmvFuse fz;
            memset(&fz, 0, sizeof(fz));
            fz.stop = fr.stop;
            B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rp, rq, a0, a1, shifted, &rp, ctx->d_res, &fz));
            b2k_dispatch(ctx, [&](auto t) {
                using T = decltype(t);
                k_cg_xr<T><<<grid, BT, 0, ctx->stream>>>((T*)rx.ptr, (T*)rr.ptr, (const T*)rp.ptr, (const T*)rq.ptr,
                                                         rx.n, 0.0, ctx->d_res, ctx->d_part_s, ctx->d_sync,
                                                         ctx->d_res + 1, ch);
            });
            B2K_LAUNCH_CHECK(ctx);
        }
        return B2K_OK;
    }));
    B2K_TRY(fr.fetch(nsteps));
    const int32_t d = fr.count(nsteps, [&](const double* rec) { return rec[1] < tol; });
    for (int32_t i = 0; i < d; ++i) {
        pq_out[i] = fr.hrec[(size_t)B2K_REC * i];
        normr_out[i] = fr.hrec[(size_t)B2K_REC * i + 1];
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
    VecRef vr[5];
    B2K_TRY(b2k_resolve_vecs(ctx, "bicgstab_half", {rs, r, p, v, s}, vr));
    const VecRef &rrs = vr[0], &rr = vr[1], &rp = vr[2], &rv = vr[3], &rsv = vr[4];
    const int64_t n = rr.n;
    const int grid = grid_for(ctx, n, 8);
    if (first) {
        B2K_TRY(b2k_vec_copy(ctx, p, r));
    } else {
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_bicg_p<T><<<grid, BT, 0, ctx->stream>>>((T*)rp.ptr, (const T*)rr.ptr, (const T*)rv.ptr, n, T(beta),
                                                      T(omega), BicgChain{});
        });
        B2K_LAUNCH_CHECK(ctx);
    }
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rp, rv, a0, a1, shifted, &rrs, 0));      // d_res[0] = sigma
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 1, rr.sharded));
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_bicg_s<T><<<grid, BT, 0, ctx->stream>>>((T*)rsv.ptr, (const T*)rr.ptr, (const T*)rv.ptr, n, rho, ctx->d_res,
                                                  ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, BicgChain{});
    });
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
    VecRef vr[6];
    B2K_TRY(b2k_resolve_vecs(ctx, "bicgstab_full", {x, r, rs, p, s, t}, vr));
    const VecRef &rx = vr[0], &rr = vr[1], &rrs = vr[2], &rp = vr[3], &rsv = vr[4], &rt = vr[5];
    const int64_t n = rr.n;
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    B2K_TRY(b2k_enqueue_apply(ctx, op, rsv, rt, a0, a1, shifted, &rsv, 0));     // d_res[0] = <s, t>
    B2K_TRY(b2k_enqueue_dot(ctx, rt.ptr, rt.ptr, n, nullptr, -1, 1, -1));       // d_res[1] = <t, t>
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, 2, rr.sharded));
    const int grid = grid_for(ctx, n, 8);
    b2k_dispatch(ctx, [&](auto tt) {
        using T = decltype(tt);
        k_bicg_xr<T><<<grid, BT, 0, ctx->stream>>>((T*)rx.ptr, (T*)rr.ptr, (const T*)rrs.ptr, (const T*)rp.ptr,
                                                   (const T*)rsv.ptr, (const T*)rt.ptr, n, T(alpha), ctx->d_res,
                                                   ctx->d_res + 1, ctx->d_part_s, ctx->d_sync, ctx->d_res + 2,
                                                   BicgChain{});
    });
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
    VecRef vr[7];
    B2K_TRY(b2k_resolve_vecs(ctx, "bicgstab_chain", {x, r, rs, p, v, s, t}, vr, true));
    const VecRef &rx = vr[0], &rr = vr[1], &rrs = vr[2], &rp = vr[3], &rv = vr[4], &rsv = vr[5], &rt = vr[6];
    const int64_t n = rr.n;
    if (ctx->nranks > 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "bicgstab_chain: single-GPU contexts (use b2k_bicgstab_half/_full)");
    int64_t orows = 0, ocols = 0;
    int32_t okind = -1;
    B2K_TRY(b2k_op_info(op, &orows, &ocols, nullptr, &okind));
    if (okind != 0) return b2k_fail(ctx, B2K_ENOTSUP, "bicgstab_chain: CSR operators only");
    B2kChain fr(ctx, B2K_REC);                          // state {rho, rho_old, alpha, omega}
    const double seed[4] = {rho, rho_old, alpha, omega};
    B2K_TRY(fr.seed(seed, 4, nsteps));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    const int grid = grid_for(ctx, n, 8);
    SpmvFuse fz;
    memset(&fz, 0, sizeof(fz));
    fz.stop = fr.stop;
    B2K_TRY(fr.enqueue([&]() -> int32_t {
        for (int32_t i = 0; i < nsteps; ++i) {
            const BicgChain ch{fr.st, fr.rec0 + (size_t)B2K_REC * i, fr.stop, tol};
            b2k_dispatch(ctx, [&](auto tt) {
                using T = decltype(tt);
                k_bicg_p<T><<<grid, BT, 0, ctx->stream>>>((T*)rp.ptr, (const T*)rr.ptr, (const T*)rv.ptr, n, T(0),
                                                          T(0), ch);
            });
            B2K_LAUNCH_CHECK(ctx);
            B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rp, rv, a0, a1, shifted, &rrs, ctx->d_res, &fz));   // sigma
            b2k_dispatch(ctx, [&](auto tt) {
                using T = decltype(tt);
                k_bicg_s<T><<<grid, BT, 0, ctx->stream>>>((T*)rsv.ptr, (const T*)rr.ptr, (const T*)rv.ptr, n, 0.0,
                                                          ctx->d_res, ctx->d_part_s, ctx->d_sync, ctx->d_res + 1, ch);
            });
            B2K_LAUNCH_CHECK(ctx);
            B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rsv, rt, a0, a1, shifted, &rsv, ctx->d_res, &fz));  // <s, t>
            B2K_TRY(b2k_enqueue_dot(ctx, rt.ptr, rt.ptr, n, nullptr, -1, 1, -1));                        // <t, t>
            b2k_dispatch(ctx, [&](auto tt) {
                using T = decltype(tt);
                k_bicg_xr<T><<<grid, BT, 0, ctx->stream>>>((T*)rx.ptr, (T*)rr.ptr, (const T*)rrs.ptr, (const T*)rp.ptr,
                                                           (const T*)rsv.ptr, (const T*)rt.ptr, n, T(0), ctx->d_res,
                                                           ctx->d_res + 1, ctx->d_part_s, ctx->d_sync, ctx->d_res + 2,
                                                           ch);
            });
            B2K_LAUNCH_CHECK(ctx);
        }
        return B2K_OK;
    }));
    B2K_TRY(fr.fetch(nsteps));
    const int32_t d = fr.count(nsteps, [](const double* rec) { return rec[7] != 0.0; });
    memcpy(rec_out, fr.hrec, sizeof(double) * B2K_REC * d);
    *steps_done = d;
    return B2K_OK;
}

// Up to `nsteps` MINRES iterations enqueued back to back, two launches each — the SpMV with the 1/beta_k
// normalisation of its operand applied in the gather and alpha = <v_k, q> in its epilogue, then k_minres_step — and a
// flush launch that applies the last pending direction / solution update.  ONE host synchronisation per call.
extern "C" int32_t b2k_minres_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec p_prev, b2k_vec p_cur, b2k_vec q,
                                    b2k_vec d1, b2k_vec d2, double a0, double a1, const double* state_in, double tol,
                                    int32_t nsteps, double* rec_out, double* state_out, int32_t* steps_done) {
    if (!ctx || !op || !state_in || !rec_out || !state_out || !steps_done || nsteps < 1) return B2K_EINVAL;
    if (nsteps > B2K_MAX_CHAIN - 1) nsteps = B2K_MAX_CHAIN - 1;
    VecRef r[6];
    B2K_TRY(b2k_resolve_vecs(ctx, "minres_chain", {x, p_prev, p_cur, q, d1, d2}, r, true));
    const int64_t n = r[0].n;
    int64_t orows = 0, ocols = 0;
    int32_t okind = -1;
    B2K_TRY(b2k_op_info(op, &orows, &ocols, nullptr, &okind));
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "minres_chain: single-GPU contexts only");
    if (okind == 1) return b2k_fail(ctx, B2K_ENOTSUP, "minres_chain: CSR / stencil operators only");
    if (orows != n || ocols != n) return b2k_fail(ctx, B2K_EDIM, "minres_chain: length mismatch");
    *steps_done = 0;
    B2kChain fr(ctx, MR_NSTATE);
    double seed[MR_NSTATE] = {};
    memcpy(seed, state_in, 8 * sizeof(double));
    B2K_TRY(fr.seed(seed, MR_NSTATE, nsteps));
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    const int grid = grid_for(ctx, n, 4);
    SpmvFuse fz;
    memset(&fz, 0, sizeof(fz));
    fz.stop = fr.stop;
    fz.xscale = fr.st + MR_INVB;
    fz.dot_self = 1;
    MinresChain ch;
    ch.st = fr.st; ch.stop = fr.stop; ch.alpha = ctx->d_res; ch.tol = tol;
    B2K_TRY(fr.enqueue([&]() -> int32_t {
        for (int32_t i = 0; i <= nsteps; ++i) {
            ch.rec = fr.rec0 + (size_t)B2K_REC * i;
            // the operand is p_cur of this iteration: the roles swap with every iteration that runs, and a launch
            // behind a raised stop flag does nothing, so the host's count is the device's whenever it matters
            if (i < nsteps)
                B2K_TRY(b2k_enqueue_apply_fused(ctx, op, r[(i & 1) ? 1 : 2], r[3], a0, a1, shifted, nullptr, ctx->d_res,
                                                &fz));
            b2k_dispatch(ctx, [&](auto t) {
                using T = decltype(t);
                b2k_flag(i < nsteps, [&](auto lz) {            // the last launch is the flush
                    k_minres_step<T, lz><<<grid, BT, 0, ctx->stream>>>((T*)r[0].ptr, (T*)r[1].ptr, (T*)r[2].ptr,
                                                                       (const T*)r[3].ptr, (T*)r[4].ptr, (T*)r[5].ptr,
                                                                       n, ctx->d_part_s, ctx->d_sync, ch);
                });
            });
            B2K_LAUNCH_CHECK(ctx);
        }
        return B2K_OK;
    }));
    B2K_TRY(fr.fetch(nsteps, 8));
    const int32_t d = fr.count(nsteps, [](const double* rec) { return rec[5] != 0.0; });
    memcpy(rec_out, fr.hrec, sizeof(double) * B2K_REC * d);
    memcpy(state_out, fr.hst, 8 * sizeof(double));
    *steps_done = d;
    return B2K_OK;
}
