// tsk.cuh — the tall-skinny streaming engine.
//
// Every basis operation of the Krylov hot path (project!!, unproject!!, the Gram-Schmidt
// family, basistransform!, block products, and the dense GEMV of the GKL path) is a sweep
// over an n x k column-major panel Q with n >> k.  All of them are HBM-bound (<= 0.25
// flop/B in FP64), so the engine is built around one thing: keeping ~200 KB of bulk
// async copies (TMA, cp.async.bulk -> SASS UBLKCP) in flight per SM without spending
// registers on it.
//
//   * one persistent CTA per SM (grid = min(#SM, #row tiles)), 384 threads:
//     warps 0-7 = consumers, warps 8-11 = producers (chunk g -> producer g % 4);
//   * a row tile is R = 256 rows; a ring slot holds R rows x C columns (16 KB:
//     C = 8 for f64, 16 for f32); NS = 12 slots form the ring, each with a full/empty
//     mbarrier pair; the producer's lanes issue one 1-D bulk copy per column (2 KB f64),
//     so arbitrary (non-contiguous) column handle lists cost nothing extra;
//   * the vector being orthogonalised rides in a separate 3-deep ring ("w slots"); the two
//     extra vectors of the Lanczos three-term prologue are basis columns and ride in the
//     panel ring's first chunk (PhaseParams::prologue);
//   * UPDATE phases map thread <-> row (sequential fma over the columns: the same
//     association as the reference's chain of add!! calls, orthonormal.jl:146-148);
//     PROJECT phases map warp <-> column, lane <-> rows (128-bit LDS), accumulators in
//     registers for the whole sweep, one warp-shuffle reduction per CTA at the end;
//   * a fused UPDATE+PROJECT phase keeps the whole R x k tile resident in the ring so Q is
//     read from HBM once for both (this is what makes CGS2 (3k+5)W instead of (4k+6)W);
//   * reductions are deterministic: per-CTA partials at fixed slots, summed in CTA order
//     by every consumer of the next phase (or by the finalize kernel).  No FP atomics.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace tsk {

template <typename T> struct Cfg;
template <> struct Cfg<double> {
    static constexpr int R = 256, C = 8, VEC = 2;
    using V16 = double2;
    __device__ static __forceinline__ void unpack(const double2& v, double* o) { o[0] = v.x; o[1] = v.y; }
};
template <> struct Cfg<float> {
    static constexpr int R = 256, C = 16, VEC = 4;
    using V16 = float4;
    __device__ static __forceinline__ void unpack(const float4& v, float* o) {
        o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    }
};

constexpr int NS = 12;         // ring slots
constexpr int NW = 3;          // w slots
constexpr int NCONS = 256;     // consumer threads
constexpr int NPROD = 4;        // producer warps: ONE warp issuing the 2 KB bulk copies one after another
                               // caps the bytes a CTA can have in flight
constexpr int NTHREADS = NCONS + 32 * NPROD;
constexpr int MAXCH = 16;      // chunks per pass  -> KCAP = MAXCH * C columns per pass
constexpr int SLOT_BYTES = 16384;
static_assert(NS % NPROD == 0, "a ring slot must always be refilled by the same producer warp");

template <typename T> constexpr int kcap() { return MAXCH * Cfg<T>::C; }

// shared memory carve-up (bytes)
constexpr int OFF_RING = 0;
constexpr int OFF_WRING = NS * SLOT_BYTES;                  // 196608
constexpr int WSLOT_MAX = 3 * 256 * 8;                      // 6144
constexpr int OFF_W1 = OFF_WRING + NW * WSLOT_MAX;          // 215040
constexpr int OFF_CS = OFF_W1 + 2 * 256 * 8;                // 219136
constexpr int OFF_RED = OFF_CS + 1024;                      // 220160
constexpr int OFF_BAR = OFF_RED + 512;                      // 220672
constexpr int SMEM_BYTES = OFF_BAR + (2 * NS + 2 * NW) * 8; // 220912

struct ColList {
    int32_t c[256];
};

template <typename T>
struct PhaseParams {
    const T* base;   // panel base (column 0 of the slab / dense matrix)
    int64_t ld;      // leading dimension (elements)
    int64_t n;       // rows
    int32_t k;       // columns in this pass (<= kcap<T>())
    // the streamed vector
    const T* x;
    T* xout;         // may be nullptr
    // Lanczos three-term prologue: x' = (x + c1*v_prev) + c2*v.  v_prev and v are the last two basis columns;
    // the host lists the columns rotated by two, [v_prev, v, q_0, ..., q_{k-3}], so both arrive with the first
    // chunk of every tile and are read from the ring once for the prologue and the projection (or update) alike.
    // Coefficients and partials keep the original column index.
    int32_t prologue;
    T c1, c2;
    const double* c1_dev;   // if set: c1 = -(*c1_dev)  (beta of the previous step, kept on the device)
    const double* c2_dev;   // if set: c2 = -(*c2_dev), a device scalar produced by the previous kernel
    int32_t c2_sets;        // > 1: c2 = -(sum_g c2_dev[g * c2_stride]), the per-rank partials in the peer window
    int32_t c2_stride;
    // row-sharded contexts: the rows the neighbours need for their next SpMV are stored into their windows as
    // the final vector is written (UPDATE phase with store_x): first send_lo rows -> halo_dn, last send_hi -> halo_up
    T* halo_dn;
    T* halo_up;
    int64_t send_lo, send_hi;
    int32_t store_x; // write x'' (UPDATE) to xout
    int32_t l2_hints; // panel loads evict_first, the stored vector evict_last (common.cuh)
    // UPDATE: x'' = betax*x' + sum_j Q[:,j]*cs[j],  cs[j] = alphac * sum_g coef[g*stride+j]
    const double* coef;
    const T* coef_t;     // alternative: coefficients stored as a device vector of T
    int32_t coef_sets;
    int32_t coef_stride;
    int32_t coef_ranks;  // the sets are per-rank sums (peer window): added in rank order (coef_ranksum)
    T alphac, betax;
    int32_t beta_mode;   // 0: hard zero, 1: one, 2: general
    // outputs
    double* part_h;  // [grid][B2K_KSTRIDE] projection partials (PROJECT)
    double* part_n;  // [grid] partial ||x''||^2 (may be nullptr)
};

struct Pipe {
    uint32_t s = 0, ph = 0, ws = 0, wph = 0;
    uint32_t g = 0;   // running chunk counter (producers: chunk g belongs to producer warp g % NPROD)
};

struct SmemView {
    uint8_t* raw;
    uint32_t ring, wring, full, empty, wfull, wempty;   // shared-space addresses
    __device__ explicit SmemView(uint8_t* p) : raw(p) {
        ring = smem_u32(p + OFF_RING);
        wring = smem_u32(p + OFF_WRING);
        full = smem_u32(p + OFF_BAR);
        empty = full + NS * 8;
        wfull = empty + NS * 8;
        wempty = wfull + NW * 8;
    }
};

__device__ __forceinline__ void pipe_setup(const SmemView& sm, bool zero_ring) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(sm.full + 8 * i, 1);
            mbar_init(sm.empty + 8 * i, NCONS / 32);
        }
        for (int i = 0; i < NW; ++i) {
            mbar_init(sm.wfull + 8 * i, 1);
            mbar_init(sm.wempty + 8 * i, NCONS / 32);
        }
        fence_mbar_init();
    }
    if (zero_ring) {
        // the CTA that owns the ragged last tile multiplies stale slot rows by zero:
        // make sure "stale" can never be a NaN bit pattern left by a previous kernel.
        uint4* q = reinterpret_cast<uint4*>(sm.raw);
        for (int i = threadIdx.x; i < OFF_CS / 16; i += blockDim.x) q[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();
}

// ---------------------------------------------------------------- partial sums ----
// Deterministic sum over G per-CTA partials of one coefficient, shared by the UPDATE phases and
// by k_finalize so that the coefficient APPLIED to the vector and the one REPORTED to the host
// are the same bits.  L = coef_lanes(k) lanes (a power of two, L*k <= 256) share a column: lane
// l adds the partials g = l, l+L, ... in order (loads batched 4 deep), then a fixed xor tree
// combines the lanes.  One memory round trip instead of G dependent ones.
__device__ __forceinline__ int coef_lanes(int k) {
    int L = 16;
    while (L > 1 && L * k > NCONS) L >>= 1;
    return L;
}
__device__ __forceinline__ double partial_lane_sum(const double* P, int G, int stride, int l, int L) {
    double a = 0.0;
    int g = l;
    // twelve loads in flight per lane (132 CTAs / 4 lanes = 33 partials per lane at k = 60: three round trips to L2
    // instead of nine — this sum sits on the critical path of every phase boundary, 2-3 times per Lanczos step);
    // the additions stay in the order g = l, l + L, l + 2L, ...
    for (; g + 11 * L < G; g += 12 * L) {
        double t[12];
#pragma unroll
        for (int u = 0; u < 12; ++u) t[u] = __ldcg(P + (size_t)(g + u * L) * stride);
#pragma unroll
        for (int u = 0; u < 12; ++u) a += t[u];
    }
    for (; g + 3 * L < G; g += 4 * L) {
        const double t0 = __ldcg(P + (size_t)g * stride), t1 = __ldcg(P + (size_t)(g + L) * stride);
        const double t2 = __ldcg(P + (size_t)(g + 2 * L) * stride), t3 = __ldcg(P + (size_t)(g + 3 * L) * stride);
        a += t0; a += t1; a += t2; a += t3;
    }
    for (; g < G; g += L) a += __ldcg(P + (size_t)g * stride);
    return a;
}
// all 32 lanes of the warp must call this (inactive columns pass valid = false)
__device__ __forceinline__ double coef_colsum(const double* P, int G, int stride, int j, int l, int L,
                                              bool valid) {
    double a = valid ? partial_lane_sum(P + j, G, stride, l, L) : 0.0;
    for (int o = L >> 1; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    return a;
}

// The coefficient of column j from the nranks per-rank sums of a row-sharded launch (peer window): added in rank
// order from 0.0 by lane 0 of the column, as peer_sum1 and the synchronous step's all-reduce add them, so that a chained
// step has the bits of a synchronous one at any number of ranks (coef_colsum's lane tree would add ranks 0 and 2 first
// at three ranks).  Only lane 0's value is used.
__device__ __forceinline__ double coef_ranksum(const double* P, int G, int stride, int j, int l, bool valid) {
    double a = 0.0;
    if (valid && l == 0)
        for (int g = 0; g < G; ++g) a += __ldcg(P + (size_t)g * stride + j);
    return a;
}

// ---------------------------------------------------------------- producer ----
template <typename T>
__device__ __forceinline__ void producer_phase(const PhaseParams<T>& p, const ColList& cl,
                                               const SmemView& sm, Pipe& st) {
    using CF = Cfg<T>;
    constexpr int R = CF::R, C = CF::C;
    const int lane = threadIdx.x & 31;
    const uint32_t me = (threadIdx.x - NCONS) >> 5;     // producer warp index
    const int nch = (p.k + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    const uint64_t pol = p.l2_hints ? l2_policy_evict_first() : 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        const uint32_t bytes = (uint32_t)((rt * sizeof(T) + 15) & ~(size_t)15);
        // the vector tile: producer warp 0
        if (me == 0) {
            mbar_wait(sm.wempty + 8 * st.ws, st.wph ^ 1);
            if (lane == 0) {
                mbar_expect_tx(sm.wfull + 8 * st.ws, bytes);
                bulk_g2s(sm.wring + st.ws * WSLOT_MAX, p.x + r0, bytes, sm.wfull + 8 * st.ws);
            }
        }
        if (++st.ws == NW) { st.ws = 0; st.wph ^= 1; }
        // the panel tile, C columns per slot; chunk g is issued by producer warp g % NPROD
        // (NS % NPROD == 0, so a slot is always refilled by the same warp)
        for (int c = 0; c < nch; ++c) {
            if ((st.g % NPROD) == me) {
                mbar_wait(sm.empty + 8 * st.s, st.ph ^ 1);
                const int ncol = (p.k - c * C) < C ? (p.k - c * C) : C;
                if (lane == 0) mbar_expect_tx(sm.full + 8 * st.s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol) {
                    const T* src = p.base + (int64_t)cl.c[c * C + lane] * p.ld + r0;
                    if (p.l2_hints)
                        bulk_g2s_hint(sm.ring + st.s * SLOT_BYTES + lane * R * (int)sizeof(T), src, bytes,
                                      sm.full + 8 * st.s, pol);
                    else
                        bulk_g2s(sm.ring + st.s * SLOT_BYTES + lane * R * (int)sizeof(T), src, bytes,
                                 sm.full + 8 * st.s);
                }
            }
            ++st.g;
            if (++st.s == NS) { st.s = 0; st.ph ^= 1; }
        }
    }
}

// ---------------------------------------------------------------- consumers ----
template <typename T> struct VecOps;
template <> struct VecOps<double> {
    __device__ static __forceinline__ void fma_acc(double& acc, const double2& q, const double2& x) {
        acc = fma(q.x, x.x, acc);
        acc = fma(q.y, x.y, acc);
    }
    // the elements of rows >= rt (r0 = row of q.x) become 0
    __device__ static __forceinline__ double2 mask(double2 q, int r0, int rt) {
        if (r0 >= rt) q.x = 0.0;
        if (r0 + 1 >= rt) q.y = 0.0;
        return q;
    }
};
template <> struct VecOps<float> {
    __device__ static __forceinline__ void fma_acc(float& acc, const float4& q, const float4& x) {
        acc = fmaf(q.x, x.x, acc);
        acc = fmaf(q.y, x.y, acc);
        acc = fmaf(q.z, x.z, acc);
        acc = fmaf(q.w, x.w, acc);
    }
    __device__ static __forceinline__ float4 mask(float4 q, int r0, int rt) {
        if (r0 >= rt) q.x = 0.0f;
        if (r0 + 1 >= rt) q.y = 0.0f;
        if (r0 + 2 >= rt) q.z = 0.0f;
        if (r0 + 3 >= rt) q.w = 0.0f;
        return q;
    }
};

// PRO: the Lanczos three-term prologue (PhaseParams::prologue).  A template parameter, so that the sweeps without it
// compile to exactly the code they had before the prologue moved into the panel ring.
template <typename T, bool UPDATE, bool PROJECT, bool PRO>
__device__ __forceinline__ void consumer_phase(const PhaseParams<T>& p, const SmemView& sm,
                                               Pipe& st) {
    using CF = Cfg<T>;
    using V16 = typename CF::V16;
    constexpr int R = CF::R, C = CF::C, VEC = CF::VEC;
    constexpr int CPW = C / 8;             // columns per warp per chunk
    constexpr int NLD = R / (32 * VEC);    // 128-bit loads per column per lane
    const int tid = threadIdx.x;           // 0..255
    const int lane = tid & 31, w = tid >> 5;
    const int nch = (p.k + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    T* cs = reinterpret_cast<T*>(sm.raw + OFF_CS);
    T* w1 = reinterpret_cast<T*>(sm.raw + OFF_W1);
    double* red = reinterpret_cast<double*>(sm.raw + OFF_RED);
    if (UPDATE) {
        // every CTA reduces the previous phase's partials itself (fixed order, see coef_colsum); cs is kept in
        // ring order
        if (p.coef_t) {
            for (int j = tid; j < p.k; j += NCONS) cs[PRO ? (j + 2) % p.k : j] = p.alphac * p.coef_t[j];
        } else {
            const int L = coef_lanes(p.k);
            const int j = tid / L, l = tid % L;
            const bool valid = j < p.k;
            const double h = p.coef_ranks ? coef_ranksum(p.coef, p.coef_sets, p.coef_stride, j, l, valid)
                                          : coef_colsum(p.coef, p.coef_sets, p.coef_stride, j, l, L, valid);
            if (valid && l == 0) cs[PRO ? (j + 2) % p.k : j] = p.alphac * (T)h;
        }
        named_bar_sync(1, NCONS);
    }

    T acc_h[MAXCH][CPW];
#pragma unroll
    for (int c = 0; c < MAXCH; ++c)
#pragma unroll
        for (int cc = 0; cc < CPW; ++cc) acc_h[c][cc] = (T)0;
    T nrm = (T)0;
    int buf = 0;
    const uint64_t pol_last = p.l2_hints ? l2_policy_evict_last() : 0;
    T c1 = p.c1, c2 = p.c2;
    if (p.c1_dev) c1 = (T)(-(*reinterpret_cast<const volatile double*>(p.c1_dev)));
    if (p.c2_dev) {
        double a2 = 0.0;
        const int ns = p.c2_sets > 1 ? p.c2_sets : 1;
        for (int g = 0; g < ns; ++g)      // rank order: same bits on every rank (and in the finaliser)
            a2 += *reinterpret_cast<const volatile double*>(p.c2_dev + (size_t)g * p.c2_stride);
        c2 = (T)(-a2);
    }

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        mbar_wait(sm.wfull + 8 * st.ws, st.wph);
        const T* wv = reinterpret_cast<const T*>(sm.raw + OFF_WRING + st.ws * WSLOT_MAX);
        T xv = wv[tid];
        T vprev = (T)0, vcur = (T)0;
        if (PRO) {
            // v_prev and v are the first two columns of the tile's first chunk
            mbar_wait(sm.full + 8 * st.s, st.ph);
            const T* slot = reinterpret_cast<const T*>(sm.raw + OFF_RING + st.s * SLOT_BYTES);
            vprev = slot[tid];
            vcur = slot[R + tid];
            xv = fma(c1, vprev, xv);
            xv = fma(c2, vcur, xv);
        }
        if (tid >= rt) xv = (T)0;
        T acc = xv;
        const uint32_t s0 = st.s, ph0 = st.ph;
        if (UPDATE) {
            acc = (p.beta_mode == 0) ? (T)0 : (p.beta_mode == 1 ? xv : p.betax * xv);
            for (int c = 0; c < nch; ++c) {
                mbar_wait(sm.full + 8 * st.s, st.ph);
                const T* slot = reinterpret_cast<const T*>(sm.raw + OFF_RING + st.s * SLOT_BYTES);
                const int ncol = (p.k - c * C) < C ? (p.k - c * C) : C;
                const int j0 = (PRO && c == 0) ? 2 : 0;    // v_prev and v are added last, in original column order
                if (ncol == C && j0 == 0) {
                    T cv[C];
#pragma unroll
                    for (int i = 0; i < C / VEC; ++i)
                        CF::unpack(*reinterpret_cast<const V16*>(cs + c * C + i * VEC), cv + i * VEC);
#pragma unroll
                    for (int jj = 0; jj < C; ++jj) acc = fma(slot[jj * R + tid], cv[jj], acc);
                } else {
                    for (int jj = j0; jj < ncol; ++jj) acc = fma(slot[jj * R + tid], cs[c * C + jj], acc);
                }
                if (!PROJECT) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(sm.empty + 8 * st.s);
                }
                if (++st.s == NS) { st.s = 0; st.ph ^= 1; }
            }
            if (PRO) {
                acc = fma(vprev, cs[0], acc);
                acc = fma(vcur, cs[1], acc);
            }
            if (tid >= rt) acc = (T)0;
        }
        if (p.store_x && tid < rt) {
            if (p.l2_hints) st_hint(p.xout + r0 + tid, acc, pol_last);
            else p.xout[r0 + tid] = acc;
            if (UPDATE && !PROJECT) {
                const int64_t r = r0 + tid;
                if (p.halo_dn && r < p.send_lo) p.halo_dn[r] = acc;
                if (p.halo_up && r >= p.n - p.send_hi) p.halo_up[r - (p.n - p.send_hi)] = acc;
            }
        }
        if (p.part_n) nrm = fma(acc, acc, nrm);
        if (PROJECT) {
            T* wb = w1 + buf * R;
            wb[tid] = acc;
            named_bar_sync(1, NCONS);
            V16 xr[NLD];
#pragma unroll
            for (int i = 0; i < NLD; ++i)
                xr[i] = *reinterpret_cast<const V16*>(wb + VEC * lane + 32 * VEC * i);
            uint32_t ss = UPDATE ? s0 : st.s, pp = UPDATE ? ph0 : st.ph;
            // The bulk copies of a ragged tile fill rows < rt only: the slot rows past them still hold an earlier
            // tile's values (of whichever column used the slot then).  x is 0 there, but Inf * 0 is NaN, so the
            // ragged tile zeroes those elements of q before the products; full tiles take the unmasked copy.
            auto sweep = [&](auto masked) {
#pragma unroll
                for (int c = 0; c < MAXCH; ++c) {
                    if (c < nch) {
                        if (!UPDATE) mbar_wait(sm.full + 8 * ss, pp);
                        const T* slot = reinterpret_cast<const T*>(sm.raw + OFF_RING + ss * SLOT_BYTES);
#pragma unroll
                        for (int cc = 0; cc < CPW; ++cc) {
                            const int cj = cc * 8 + w;
                            if (c * C + cj < p.k) {
                                const T* colp = slot + cj * R;
#pragma unroll
                                for (int i = 0; i < NLD; ++i) {
                                    V16 q = *reinterpret_cast<const V16*>(colp + VEC * lane + 32 * VEC * i);
                                    if constexpr (decltype(masked)::value)
                                        q = VecOps<T>::mask(q, VEC * lane + 32 * VEC * i, rt);
                                    VecOps<T>::fma_acc(acc_h[c][cc], q, xr[i]);
                                }
                            }
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(sm.empty + 8 * ss);
                        if (++ss == NS) { ss = 0; pp ^= 1; }
                    }
                }
            };
            if (rt == R) sweep(std::false_type{});
            else sweep(std::true_type{});
            if (!UPDATE) { st.s = ss; st.ph = pp; }
            buf ^= 1;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(sm.wempty + 8 * st.ws);
        if (++st.ws == NW) { st.ws = 0; st.wph ^= 1; }
    }

    if (PROJECT) {
#pragma unroll
        for (int c = 0; c < MAXCH; ++c) {
#pragma unroll
            for (int cc = 0; cc < CPW; ++cc) {
                const int j = c * C + cc * 8 + w;            // ring position
                double v = warp_sum((double)acc_h[c][cc]);   // warp-uniform branch below
                if (c < nch && j < p.k && lane == 0)
                    p.part_h[(size_t)blockIdx.x * B2K_KSTRIDE + (PRO ? (j < 2 ? j + p.k - 2 : j - 2) : j)] = v;
            }
        }
    }
    if (p.part_n) {
        double v = warp_sum((double)nrm);
        if (lane == 0) red[w] = v;
        named_bar_sync(1, NCONS);
        if (tid == 0) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < NCONS / 32; ++i) s += red[i];
            p.part_n[blockIdx.x] = s;
        }
    }
}

// ---------------------------------------------------------------- finalize ----
// res[off + j] = sum_g A[g*stride + j] (+ sum_g B[g*stride + j]);  res[noff] = sum_g N[g] — executed by NCONS
// threads, same lane layout and summation order as the UPDATE phases (coef_colsum), so the coefficient REPORTED
// equals the one APPLIED bit for bit.  Used by k_finalize (one launch) and, when a Gram-Schmidt launch carries a
// FinalizeParams, by the last CTA of that launch itself (ticket): no extra launch, and the Lanczos scalars of
// the step land in a device record the NEXT step's kernels read — the host never has to be in the loop:
//   rec[0] = <v, A v> (written by the SpMV)      rec[1] = alpha = rec[0] + h[alpha_col]   (lanczos.jl:321)
//   rec[2] = beta = sqrt(||w||^2)                 rec[3] = 1/beta                           rec[4] = ||w||^2
// and *stop = 1 if beta <= tol, or (stop_nonfinite) beta is not finite (the steps already enqueued behind this one
// then do nothing).
struct FinalizeParams {
    const double* A;
    const double* B;
    const double* N;
    int G, stride, k;
    double* res;        // may be nullptr
    int off, noff;
    double* rec;        // may be nullptr
    int alpha_col;
    double tol;
    int* stop;
    unsigned* ticket;
    int enabled;
    // row-sharded (peer window): A/B are then the per-rank sums in MY window (G = nranks, stride = PEER_SLOT), added in
    // rank order (coef_ranksum), N the LOCAL per-CTA norm partials (G_local of them); the norm and <v, A v> are summed
    // over ranks here
    int peer;
    int G_local;
    int stop_nonfinite;
};

// `sh` : >= 2 doubles of shared memory; `barrier_id` : named barrier the NCONS calling threads may use
__device__ __forceinline__ void finalize_block(const FinalizeParams& f, int tid, double* sh,
                                               const PeerStep* ps = nullptr) {
    double hval = 0.0;
    if (f.k > 0) {
        const int L = coef_lanes(f.k);
        const int j = tid / L, l = tid % L;
        const bool valid = j < f.k;
        double a = f.peer ? coef_ranksum(f.A, f.G, f.stride, j, l, valid) : coef_colsum(f.A, f.G, f.stride, j, l, L, valid);
        if (f.B) a += coef_colsum(f.B, f.G, f.stride, j, l, L, valid);
        if (valid && l == 0) {
            if (f.res) f.res[f.off + j] = a;
            if (j == f.alpha_col) hval = a;
        }
        if (f.rec && valid && l == 0 && j == f.alpha_col) sh[0] = hval;
    }
    double n2 = 0.0;
    if (f.N && tid < 32) {
        double a = (tid < 16) ? partial_lane_sum(f.N, f.peer ? f.G_local : f.G, 1, tid, 16) : 0.0;
        for (int o = 8; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        n2 = a;
    }
    double alpha0 = f.rec ? f.rec[0] : 0.0;
    if (f.peer && ps) {
        // ||w||^2: publish my partial to every rank, wait for theirs in my window, add in rank order
        if (tid == 0) peer_publish1(ps->pd, PEER_CH_NORM, ps->seq_norm, n2);
        peer_wait(ps->pd, PEER_CH_NORM, ps->seq_norm, tid);
        named_bar_sync(1, NCONS);
        if (tid == 0) {
            n2 = peer_sum1(ps->pd, PEER_CH_NORM, ps->seq_norm, 0);
            if (ps->seq_alpha) alpha0 = peer_sum1(ps->pd, PEER_CH_ALPHA, ps->seq_alpha, 0);
            if (ps->seq_halo) {       // every CTA fenced its halo stores before taking its ticket
                __threadfence_system();
                if (ps->send_lo) st_relaxed_sys_u64(peer_hflag(ps->pd, ps->pd.rank - 1, ps->seq_halo, 1), ps->seq_halo);
                if (ps->send_hi) st_relaxed_sys_u64(peer_hflag(ps->pd, ps->pd.rank + 1, ps->seq_halo, 0), ps->seq_halo);
            }
        }
    }
    if (f.N && tid == 0 && f.res) f.res[f.noff] = n2;
    if (f.rec) {
        named_bar_sync(1, NCONS);
        if (tid == 0) {
            f.rec[0] = alpha0;
            const double alpha = alpha0 + sh[0];
            const double beta = sqrt(n2);
            f.rec[1] = alpha;
            f.rec[2] = beta;
            f.rec[3] = 1.0 / beta;
            f.rec[4] = n2;
            if (f.stop && (beta <= f.tol || (f.stop_nonfinite && !isfinite(beta)))) *f.stop = 1;
        }
    }
}

// Barrier among the CTA's threads at a phase boundary.  run_ahead: only the NCONS consumer threads take part
// (named barrier 1) and the producer warps go straight on filling the ring with the next phase's tiles — allowed
// only when no earlier phase stored into a vector the next phase streams (launch_fused decides).  Otherwise all
// threads, so that no bulk copy of the next phase is issued before every CTA's stores are visible to it.
__device__ __forceinline__ void boundary_sync(bool run_ahead) {
    if (run_ahead) named_bar_sync(1, NCONS);
    else __syncthreads();
}

// grid-wide barrier for the cooperative fused kernel.  `target` is the value the
// monotonically increasing counter reaches when every CTA has arrived.  Called by every thread of the CTA, or by
// the consumer threads only when run_ahead (boundary_sync).
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned target, bool run_ahead) {
    __threadfence();
    if (!run_ahead) asm volatile("fence.proxy.async;" ::: "memory");
    boundary_sync(run_ahead);
    if (threadIdx.x == 0) {
        atomicAdd(counter, 1u);
        while ((int)(*(volatile unsigned*)counter - target) < 0) {
        }
        __threadfence();
    }
    boundary_sync(run_ahead);
}

}  // namespace tsk
