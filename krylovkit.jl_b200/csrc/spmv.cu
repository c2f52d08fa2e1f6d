// spmv.cu — operators: CSR SpMV (apply, src/apply.jl:1), shifted apply (apply.jl:4-11),
// fused <v, A x>, dense column-major GEMV N/T through the tall-skinny engine
// (apply_normal / apply_adjoint, apply.jl:14-15), and on-device stencil assembly.
//
// CSR SpMV design ("CSR-stream"): the matrices of the configs have ~5-7 nonzeros per
// row, so a warp-per-row kernel would idle most lanes and a thread-per-row kernel reads
// vals/colidx with a 40-56 B stride.  Instead a CTA owns a run of consecutive rows whose
// nonzeros fit a 1536-entry shared-memory tile: the nonzero stream (vals, colidx) is read
// fully coalesced, multiplied with the gathered x (L1/L2-served: the band structure keeps
// the working set of x tiny), parked in shared memory, then each thread sums the products
// of its row(s) in CSR order.  Products are rounded before summation and summed in
// ascending column order: bit-identical to SparseArrays' CSC kernel for a symmetric A.
// Rows longer than the tile get a CTA to themselves (block-stride + tree reduction).
// Algorithmic traffic: nnz*(sizeof(T)+4) + 4(n+1) + 2*sizeof(T)*n bytes per apply.
#include "common.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <cmath>

// basis.cu
int32_t b2k_panel_unproject_dev(b2k_ctx* ctx, void* base, int64_t ld, int64_t n, int32_t k,
                                const VecRef& y, const void* coef_t);
int32_t b2k_panel_project_dev(b2k_ctx* ctx, void* base, int64_t ld, int64_t n, int32_t k,
                              const VecRef& x, void* out_vec, int32_t sharded);

constexpr int SP_BT = 256;
constexpr int SP_NNZ = 1536;      // nonzeros per CTA tile
constexpr int SP_ROWS = 2048;     // max rows per CTA tile (empty rows)

struct b2k_op {
    int32_t kind = 0;             // 0 = CSR, 1 = dense, 2 = matrix-free stencil
    // matrix-free stencil (kind 2): grid and coefficients; rows [row0, row0 + n_rows) of the global grid
    int64_t  snx = 0, sny = 0, snz = 0, srow0 = 0;
    double   sc[7] = {0, 0, 0, 0, 0, 0, 0};
    int64_t n_rows = 0, n_cols = 0, nnz = 0;
    // CSR (device)
    int32_t* rowptr = nullptr;
    int32_t* colidx = nullptr;    // local column index; >= n_loc_cols means halo slot
    void*    vals = nullptr;
    int32_t* rowblk = nullptr;    // CTA row-block boundaries
    int32_t* pblk = nullptr;      // rowptr[rowblk[b]] (first nonzero of each block)
    int32_t  nblk = 0;
    double*  part = nullptr;      // per-CTA dot partials (CSR / stencil); per-CTA z partials of the one-pass dense step
    size_t   part_bytes = 0;      // size of `part` when the one-pass dense step allocated it
    // halo plan (dist)
    int64_t  n_loc_cols = 0;      // columns owned locally = length of the local x
    int64_t  halo_lo = 0, halo_hi = 0;         // entries needed from rank-1 / rank+1
    int64_t  send_lo = 0, send_hi = 0;         // entries rank-1 / rank+1 need from me
    void*    halo = nullptr;      // [halo_lo | halo_hi] receive buffer
    int32_t  peer_halo = 0;       // receive buffers live in the NVLink peer window (symmetric heap offset)
    size_t   halo_off = 0, halo_region = 0;    // window offset of [parity 0 | parity 1], bytes per parity
    int64_t  dn_lo = 0;           // rank-1's halo_lo: my head rows land behind its lo entries
    int32_t  gather_all = 0;      // fallback: allgather the whole x
    void*    xall = nullptr;
    // dense (device, column-major m x n, leading dim ld)
    void*    A = nullptr;
    int64_t  ld = 0;
};

namespace {

// Products and sums rounded on their own: with nvcc's default -fmad=true, `acc += (double)(a * b)` is one DFMA for
// T = double (the cast is a no-op), so the product would not be rounded before it is added.
template <typename T> __device__ __forceinline__ T mul_rn(T a, T b);
template <> __device__ __forceinline__ double mul_rn<double>(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ float mul_rn<float>(float a, float b) { return __fmul_rn(a, b); }
template <typename T> __device__ __forceinline__ T add_rn(T a, T b);
template <> __device__ __forceinline__ double add_rn<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float add_rn<float>(float a, float b) { return __fadd_rn(a, b); }

template <typename T>
__global__ void __launch_bounds__(SP_BT)
k_spmv_stream(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
              const T* __restrict__ vals, const T* __restrict__ x, const T* __restrict__ halo,
              int32_t n_loc, T* __restrict__ y, const int32_t* __restrict__ rowblk, T a0, T a1,
              int shifted, const T* __restrict__ xs, const T* __restrict__ dotv,
              double* __restrict__ part, unsigned* __restrict__ ticket, double* __restrict__ out,
              const SpmvFuse fz, const __grid_constant__ PeerStep ps) {
    __shared__ T prod[SP_NNZ];
    __shared__ double red[32];
    __shared__ bool last;
    if (fz.stop && *reinterpret_cast<const volatile int*>(fz.stop)) return;
    if (ps.on && ps.seq_halo) {        // boundary rows of x arrive from the neighbours through the peer window
        if (threadIdx.x == 0) {
            if (ps.wait_lo) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 0), ps.seq_halo);
            if (ps.wait_hi) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 1), ps.seq_halo);
        }
        __syncthreads();
    }
    const bool scaled = fz.xscale != nullptr;
    const T sc = scaled ? (T)(*fz.xscale) : (T)1;
    T* const vout = reinterpret_cast<T*>(fz.vout);
    const int tid = threadIdx.x;
    const int r0 = rowblk[blockIdx.x], r1 = rowblk[blockIdx.x + 1];
    const int p0 = rowptr[r0], p1 = rowptr[r1];
    const int nnzb = p1 - p0;
    T dacc = (T)0;
    if (nnzb <= SP_NNZ) {
        // phase 1: coalesced nonzero stream -> products in shared memory
        constexpr int U = SP_NNZ / SP_BT;   // 8
        T v[U];
        int32_t c[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = tid + u * SP_BT;
            if (i < nnzb) {
                v[u] = __ldcs(vals + p0 + i);
                c[u] = __ldcs(colidx + p0 + i);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = tid + u * SP_BT;
            if (i < nnzb) {
                const int32_t cc = c[u];
                T xv = (cc < n_loc) ? __ldg(x + cc) : __ldg(halo + (cc - n_loc));
                if (scaled) xv *= sc;
                prod[i] = v[u] * xv;
            }
        }
        __syncthreads();
        // phase 2: one thread per row sums its products in CSR order
        for (int r = r0 + tid; r < r1; r += SP_BT) {
            const int a = rowptr[r] - p0, b = rowptr[r + 1] - p0;
            T s = (T)0;
            for (int p = a; p < b; ++p) s += prod[p];
            if (shifted) s = fma(a0, xs[r], a1 * s);
            y[r] = s;
            T dv = (T)0;
            if (vout || fz.dot_self) {
                dv = __ldg(x + r) * sc;                 // the normalised x_r (square operator, local row r)
                if (vout) vout[r] = dv;
            }
            if (dotv && !fz.dot_self) dv = dotv[r];
            if (dotv || fz.dot_self) {
                T sd = s;
                if (fz.dot_sub_vec) sd = fma(-(T)(*fz.dot_sub_scale), reinterpret_cast<const T*>(fz.dot_sub_vec)[r], s);
                dacc = fma(dv, sd, dacc);
            }
        }
    } else {
        // long row: the CTA owns exactly one row
        double acc = 0.0;
        for (int i = tid; i < nnzb; i += SP_BT) {
            const int32_t cc = colidx[p0 + i];
            T xv = (cc < n_loc) ? __ldg(x + cc) : __ldg(halo + (cc - n_loc));
            if (scaled) xv *= sc;
            acc += (double)mul_rn<T>(vals[p0 + i], xv);
        }
        const double tot = block_sum(acc, red);
        if (tid == 0) {
            T s = (T)tot;
            if (shifted) s = fma(a0, xs[r0], a1 * s);
            y[r0] = s;
            T dv = (T)0;
            if (vout || fz.dot_self) {
                dv = __ldg(x + r0) * sc;
                if (vout) vout[r0] = dv;
            }
            if (dotv && !fz.dot_self) dv = dotv[r0];
            if (dotv || fz.dot_self) {
                T sd = s;
                if (fz.dot_sub_vec) sd = fma(-(T)(*fz.dot_sub_scale), reinterpret_cast<const T*>(fz.dot_sub_vec)[r0], s);
                dacc = dv * sd;
            }
        }
    }
    if (dotv || fz.dot_self) {
        const double s = block_sum((double)dacc, red);
        if (tid == 0) {
            part[blockIdx.x] = s;
            __threadfence();
            const unsigned t = atomicInc(ticket, gridDim.x - 1);
            last = (t == gridDim.x - 1);
        }
        __syncthreads();
        if (last) {
            __threadfence();
            double v2 = 0.0;
            const volatile double* pv = part;
            for (int g = tid; g < (int)gridDim.x; g += SP_BT) v2 += pv[g];
            const double tot = block_sum(v2, red);
            if (tid == 0) {
                *out = tot;
                if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
            }
        }
    }
}


// ---------------------------------------------------------------------------------------
// Pipelined CSR-stream SpMV (the default): persistent CTAs (3 per SM), a producer warp
// streams each row block's nonzeros (vals, colidx) and its rowptr segment into a 3-stage
// shared-memory ring with 1-D TMA bulk copies (UBLKCP) signalled on mbarriers; the 8
// consumer warps gather x, multiply in place, and sum rows out of shared memory while the
// next blocks are already in flight.  Same arithmetic (products rounded, summed in CSR
// order) as k_spmv_stream, which remains as the reference implementation for tests.
constexpr int SPP_NSTG = 3;
constexpr int SPP_RMAX = 1024;            // rowptr entries staged per block
constexpr int SPP_TV = SP_NNZ + 8;        // staged nonzeros (block + alignment slack)
constexpr int SPP_CONS = 256;
constexpr int SPP_THREADS = SPP_CONS + 32;
template <typename T, int NSTG = SPP_NSTG> struct SppLayout {
    static constexpr int VAL_BYTES = SPP_TV * (int)sizeof(T);
    static constexpr int COL_BYTES = SPP_TV * 4;
    static constexpr int RP_BYTES = (SPP_RMAX + 8) * 4;
    static constexpr int STAGE = VAL_BYTES + COL_BYTES + RP_BYTES;
    static constexpr int OFF_BAR = NSTG * STAGE;
    static constexpr int OFF_RED = OFF_BAR + 2 * NSTG * 8 + 16;
    static constexpr int SMEM = OFF_RED + 32 * 8 + 16;
};

__global__ void k_pblk(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ rowblk, int count,
                       int32_t* __restrict__ pblk) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < count) pblk[b] = rowptr[rowblk[b]];
}

// NSTG ring stages, MINB CTAs per SM (variants: (3, 3); (2, 4): fewer stages, more resident warps to hide the
// latency of the x gather)
template <typename T, int NSTG, int MINB>
__global__ void __launch_bounds__(SPP_THREADS, MINB)
k_spmv_pipe(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
            const T* __restrict__ vals, const T* __restrict__ x, const T* __restrict__ halo,
            int32_t n_loc, T* __restrict__ y, const int32_t* __restrict__ rowblk,
            const int32_t* __restrict__ pblk, int nblk, T a0, T a1, int shifted,
            const T* __restrict__ xs, const T* __restrict__ dotv, double* __restrict__ part,
            unsigned* __restrict__ ticket, double* __restrict__ out, const SpmvFuse fz,
            const __grid_constant__ PeerStep ps) {
    using LY = SppLayout<T, NSTG>;
    extern __shared__ __align__(128) uint8_t smem[];
    if (fz.stop && *reinterpret_cast<const volatile int*>(fz.stop)) return;
    const uint32_t full = smem_u32(smem + LY::OFF_BAR), empty = full + NSTG * 8;
    double* red = reinterpret_cast<double*>(smem + LY::OFF_RED);
    int* flag = reinterpret_cast<int*>(smem + LY::OFF_RED + 32 * 8);
    if (threadIdx.x == 0) {
        for (int i = 0; i < NSTG; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, SPP_CONS / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= SPP_CONS) {
        // ------------------------------ producer warp ------------------------------
        int tile = blockIdx.x;
        int d = 0;   // lanes 0..3 hold r0, r1, p0, p1 of the current tile
        if (tile < nblk && lane < 4) d = (lane < 2) ? rowblk[tile + lane] : pblk[tile + lane - 2];
        for (; tile < nblk; tile += gridDim.x) {
            const int r0 = __shfl_sync(0xffffffffu, d, 0), r1 = __shfl_sync(0xffffffffu, d, 1);
            const int p0 = __shfl_sync(0xffffffffu, d, 2), p1 = __shfl_sync(0xffffffffu, d, 3);
            const int nt = tile + gridDim.x;      // prefetch the next descriptor before blocking
            if (nt < nblk && lane < 4) d = (lane < 2) ? rowblk[nt + lane] : pblk[nt + lane - 2];
            mbar_wait(empty + 8 * s, ph ^ 1);
            const int nnzb = p1 - p0, nrows = r1 - r0;
            if (nnzb <= SP_NNZ) {
                const int p0a = p0 & ~3, cnt = ((p1 + 3) & ~3) - p0a;
                const int r0a = r0 & ~3;
                const int rcnt = (nrows <= SPP_RMAX) ? (((r1 + 1 + 3) & ~3) - r0a) : 0;
                const uint32_t vb = (uint32_t)cnt * (uint32_t)sizeof(T), cb = (uint32_t)cnt * 4u,
                               rb = (uint32_t)rcnt * 4u;
                const uint32_t st = smem_u32(smem + s * LY::STAGE);
                if (lane == 0) mbar_expect_tx(full + 8 * s, vb + cb + rb);
                __syncwarp();
                if (fz.l2_hints) {
                    const uint64_t pol = l2_policy_evict_first();
                    if (lane == 0 && vb) bulk_g2s_hint(st, vals + p0a, vb, full + 8 * s, pol);
                    if (lane == 1 && cb) bulk_g2s_hint(st + LY::VAL_BYTES, colidx + p0a, cb, full + 8 * s, pol);
                    if (lane == 2 && rb) bulk_g2s_hint(st + LY::VAL_BYTES + LY::COL_BYTES, rowptr + r0a, rb, full + 8 * s, pol);
                } else {
                    if (lane == 0 && vb) bulk_g2s(st, vals + p0a, vb, full + 8 * s);
                    if (lane == 1 && cb) bulk_g2s(st + LY::VAL_BYTES, colidx + p0a, cb, full + 8 * s);
                    if (lane == 2 && rb) bulk_g2s(st + LY::VAL_BYTES + LY::COL_BYTES, rowptr + r0a, rb, full + 8 * s);
                }
            } else {
                if (lane == 0) mbar_arrive(full + 8 * s);   // long row: consumers read global memory
            }
            if (++s == NSTG) { s = 0; ph ^= 1; }
        }
        return;
    }
    // ---------------------------------- consumers ----------------------------------
    const int tid = threadIdx.x, w = tid >> 5;
    const bool tr0 = fz.trace && blockIdx.x == 0 && tid == 0;
    if (tr0) b2k_trace(fz.trace, 1);
    if (ps.on && ps.seq_halo) {        // boundary rows of x arrive from the neighbours through the peer window;
        if (tid == 0) {                // the producer warp streams the matrix meanwhile
            if (ps.wait_lo) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 0), ps.seq_halo);
            if (ps.wait_hi) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 1), ps.seq_halo);
        }
        named_bar_sync(1, SPP_CONS);
    }
    if (tr0) b2k_trace(fz.trace, 2);
    const bool scaled = fz.xscale != nullptr;
    const T sc = scaled ? (T)(*fz.xscale) : (T)1;
    T* const vout = reinterpret_cast<T*>(fz.vout);
    const bool self = (vout != nullptr) || fz.dot_self;
    const bool want_dot = (dotv != nullptr) || fz.dot_self;
    const uint64_t pol_last = fz.l2_hints ? l2_policy_evict_last() : 0;
    const T* const dsub = reinterpret_cast<const T*>(fz.dot_sub_vec);
    const T dsc = dsub ? (T)(*fz.dot_sub_scale) : (T)0;
    T dacc = (T)0;
    int tile = blockIdx.x;
    int4 dn = make_int4(0, 0, 0, 0);
    if (tile < nblk) dn = make_int4(rowblk[tile], rowblk[tile + 1], pblk[tile], pblk[tile + 1]);
    for (; tile < nblk; tile += gridDim.x) {
        const int r0 = dn.x, r1 = dn.y, p0 = dn.z, p1 = dn.w;
        const int nt = tile + gridDim.x;
        if (nt < nblk) dn = make_int4(rowblk[nt], rowblk[nt + 1], pblk[nt], pblk[nt + 1]);
        const int nnzb = p1 - p0, nrows = r1 - r0;
        mbar_wait(full + 8 * s, ph);
        if (nnzb <= SP_NNZ) {
            T* vs = reinterpret_cast<T*>(smem + s * LY::STAGE);
            const int32_t* cs = reinterpret_cast<const int32_t*>(smem + s * LY::STAGE + LY::VAL_BYTES);
            const int32_t* rs = reinterpret_cast<const int32_t*>(smem + s * LY::STAGE + LY::VAL_BYTES + LY::COL_BYTES);
            const int p0a = p0 & ~3, r0a = r0 & ~3, off = p0 - p0a;
            constexpr int U = SP_NNZ / SPP_CONS;
            T xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) {
                    const int32_t cc = cs[off + i];
                    xv[u] = (cc < n_loc) ? __ldg(x + cc) : __ldg(halo + (cc - n_loc));
                }
            }
            if (scaled) {
#pragma unroll
                for (int u = 0; u < U; ++u) xv[u] *= sc;      // v_j = r_j * (1/β), rounded like scale!!
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) vs[off + i] *= xv[u];
            }
            named_bar_sync(1, SPP_CONS);
            const bool rp_staged = nrows <= SPP_RMAX;
            for (int r = r0 + tid; r < r1; r += SPP_CONS) {
                // issue the (optional) per-row global loads first so they overlap the row sum
                T dv = (dotv && !fz.dot_self) ? __ldg(dotv + r) : (T)0;
                const T xself = self ? __ldg(x + r) : (T)0;
                const T xsr = shifted ? __ldg(xs + r) : (T)0;
                const T dsv = dsub ? __ldg(dsub + r) : (T)0;
                int a, b;
                if (rp_staged) { a = rs[r - r0a]; b = rs[r + 1 - r0a]; }
                else { a = rowptr[r]; b = rowptr[r + 1]; }
                a -= p0a; b -= p0a;
                T sum = (T)0;
                for (int p = a; p < b; ++p) sum += vs[p];
                if (shifted) sum = fma(a0, xsr, a1 * sum);
                if (fz.l2_hints) st_hint(y + r, sum, pol_last);
                else y[r] = sum;
                if (self) {
                    const T vn = xself * sc;
                    if (vout) vout[r] = vn;
                    if (fz.dot_self) dv = vn;
                }
                dacc = fma(dv, dsub ? fma(-dsc, dsv, sum) : sum, dacc);
            }
        } else {
            double acc = 0.0;
            for (int i = tid; i < nnzb; i += SPP_CONS) {
                const int32_t cc = colidx[p0 + i];
                T xv = (cc < n_loc) ? __ldg(x + cc) : __ldg(halo + (cc - n_loc));
                if (scaled) xv *= sc;
                acc += (double)mul_rn<T>(vals[p0 + i], xv);
            }
            acc = warp_sum(acc);
            if (lane == 0) red[w] = acc;
            named_bar_sync(1, SPP_CONS);
            if (tid == 0) {
                double tot = 0.0;
                for (int i = 0; i < SPP_CONS / 32; ++i) tot += red[i];
                T sum = (T)tot;
                if (shifted) sum = fma(a0, xs[r0], a1 * sum);
                y[r0] = sum;
                T dv = (dotv && !fz.dot_self) ? dotv[r0] : (T)0;
                if (self) {
                    const T vn = __ldg(x + r0) * sc;
                    if (vout) vout[r0] = vn;
                    if (fz.dot_self) dv = vn;
                }
                if (want_dot) dacc = fma(dv, dsub ? fma(-dsc, dsub[r0], sum) : sum, dacc);
            }
            named_bar_sync(1, SPP_CONS);
        }
        fence_proxy_async();   // generic-proxy writes to the stage precede its reuse by the TMA unit
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + 8 * s);
        if (++s == NSTG) { s = 0; ph ^= 1; }
    }
    if (tr0) b2k_trace(fz.trace, 3);
    if (want_dot) {
        double v = warp_sum((double)dacc);
        if (lane == 0) red[w] = v;
        named_bar_sync(1, SPP_CONS);
        if (tid == 0) {
            double tot = 0.0;
            for (int i = 0; i < SPP_CONS / 32; ++i) tot += red[i];
            part[blockIdx.x] = tot;
            __threadfence();
            const unsigned t = atomicInc(ticket, gridDim.x - 1);
            *flag = (t == gridDim.x - 1);
        }
        named_bar_sync(1, SPP_CONS);
        if (*flag) {
            __threadfence();
            double v2 = 0.0;
            const volatile double* pv = part;
            for (int g = tid; g < (int)gridDim.x; g += SPP_CONS) v2 += pv[g];
            v2 = warp_sum(v2);
            named_bar_sync(1, SPP_CONS);
            if (lane == 0) red[w] = v2;
            named_bar_sync(1, SPP_CONS);
            if (tid == 0) {
                double tot = 0.0;
                for (int i = 0; i < SPP_CONS / 32; ++i) tot += red[i];
                *out = tot;
                if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
                if (fz.trace) b2k_trace(fz.trace, 4);
            }
        }
    }
}

// SpMM for apply(A, ::Block) (blocklanczos.jl:38): the nonzero stream of a row block is staged ONCE (same TMA
// ring as k_spmv_pipe) and used for all p <= 8 vectors of the block: 12*nnz + p*16n bytes instead of
// p*(12*nnz + 16n).  Per vector the consumers do what k_spmv_pipe does — thread <-> nonzero gathers x_i and writes the
// rounded product into a product buffer (two of them, alternating, so one barrier per vector), thread <-> row sums
// its products in CSR order — bit-identical to p single-vector applies.  (The first version let one thread per row
// walk its nonzeros for all p vectors: a fifth of the gathers in flight — slower than four SpMVs.)
constexpr int SPM_NSTG = 2;
template <typename T> struct SpmLayout {
    using LY = SppLayout<T, SPM_NSTG>;
    static constexpr int OFF_PROD = LY::SMEM;                              // two product buffers
    static constexpr int PROD_BYTES = SPP_TV * (int)sizeof(T);
    static constexpr int SMEM = OFF_PROD + 2 * PROD_BYTES;
};
constexpr int SPM_PMAX = 8;
struct SpmmCols {
    int32_t x[SPM_PMAX], y[SPM_PMAX];
};

template <typename T>
__global__ void __launch_bounds__(SPP_THREADS, 3)
k_spmm_pipe(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const T* __restrict__ vals,
            T* __restrict__ base, int64_t ld, const __grid_constant__ SpmmCols cols, int np,
            const int32_t* __restrict__ rowblk, const int32_t* __restrict__ pblk, int nblk) {
    using LY = SppLayout<T, SPM_NSTG>;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t full = smem_u32(smem + LY::OFF_BAR), empty = full + SPM_NSTG * 8;
    double* red = reinterpret_cast<double*>(smem + LY::OFF_RED);
    if (threadIdx.x == 0) {
        for (int i = 0; i < SPM_NSTG; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, SPP_CONS / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= SPP_CONS) {
        // producer warp: identical to k_spmv_pipe
        int tile = blockIdx.x;
        int d = 0;
        if (tile < nblk && lane < 4) d = (lane < 2) ? rowblk[tile + lane] : pblk[tile + lane - 2];
        for (; tile < nblk; tile += gridDim.x) {
            const int r0 = __shfl_sync(0xffffffffu, d, 0), r1 = __shfl_sync(0xffffffffu, d, 1);
            const int p0 = __shfl_sync(0xffffffffu, d, 2), p1 = __shfl_sync(0xffffffffu, d, 3);
            const int nt = tile + gridDim.x;
            if (nt < nblk && lane < 4) d = (lane < 2) ? rowblk[nt + lane] : pblk[nt + lane - 2];
            mbar_wait(empty + 8 * s, ph ^ 1);
            const int nnzb = p1 - p0, nrows = r1 - r0;
            if (nnzb <= SP_NNZ) {
                const int p0a = p0 & ~3, cnt = ((p1 + 3) & ~3) - p0a;
                const int r0a = r0 & ~3;
                const int rcnt = (nrows <= SPP_RMAX) ? (((r1 + 1 + 3) & ~3) - r0a) : 0;
                const uint32_t vb = (uint32_t)cnt * (uint32_t)sizeof(T), cb = (uint32_t)cnt * 4u, rb = (uint32_t)rcnt * 4u;
                const uint32_t st = smem_u32(smem + s * LY::STAGE);
                if (lane == 0) mbar_expect_tx(full + 8 * s, vb + cb + rb);
                __syncwarp();
                if (lane == 0 && vb) bulk_g2s(st, vals + p0a, vb, full + 8 * s);
                if (lane == 1 && cb) bulk_g2s(st + LY::VAL_BYTES, colidx + p0a, cb, full + 8 * s);
                if (lane == 2 && rb) bulk_g2s(st + LY::VAL_BYTES + LY::COL_BYTES, rowptr + r0a, rb, full + 8 * s);
            } else {
                if (lane == 0) mbar_arrive(full + 8 * s);
            }
            if (++s == SPM_NSTG) { s = 0; ph ^= 1; }
        }
        return;
    }
    const int tid = threadIdx.x, w = tid >> 5;
    auto xcol = [&](int i) -> const T* { return base + (int64_t)cols.x[i] * ld; };
    auto ycol = [&](int i) -> T* { return base + (int64_t)cols.y[i] * ld; };
    int tile = blockIdx.x;
    int4 dn = make_int4(0, 0, 0, 0);
    if (tile < nblk) dn = make_int4(rowblk[tile], rowblk[tile + 1], pblk[tile], pblk[tile + 1]);
    for (; tile < nblk; tile += gridDim.x) {
        const int r0 = dn.x, r1 = dn.y, p0 = dn.z, p1 = dn.w;
        const int nt = tile + gridDim.x;
        if (nt < nblk) dn = make_int4(rowblk[nt], rowblk[nt + 1], pblk[nt], pblk[nt + 1]);
        const int nnzb = p1 - p0, nrows = r1 - r0;
        mbar_wait(full + 8 * s, ph);
        if (nnzb <= SP_NNZ) {
            const T* vs = reinterpret_cast<const T*>(smem + s * LY::STAGE);
            const int32_t* cs = reinterpret_cast<const int32_t*>(smem + s * LY::STAGE + LY::VAL_BYTES);
            const int32_t* rs = reinterpret_cast<const int32_t*>(smem + s * LY::STAGE + LY::VAL_BYTES + LY::COL_BYTES);
            const int p0a = p0 & ~3, r0a = r0 & ~3;
            const bool rp_staged = nrows <= SPP_RMAX;
            const int off = p0 - p0a;
            constexpr int U = SP_NNZ / SPP_CONS;
            // my nonzeros' values and columns are the same for every vector of the block: registers
            T vv[U];
            int32_t cc[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                vv[u] = (i < nnzb) ? vs[off + i] : (T)0;
                cc[u] = (i < nnzb) ? cs[off + i] : 0;
            }
            for (int iv = 0; iv < np; ++iv) {
                T* prod = reinterpret_cast<T*>(smem + SpmLayout<T>::OFF_PROD + (iv & 1) * SpmLayout<T>::PROD_BYTES);
                const T* xi = xcol(iv);
                T xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) xv[u] = __ldg(xi + cc[u]);
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int i = tid + u * SPP_CONS;
                    if (i < nnzb) prod[off + i] = mul_rn<T>(vv[u], xv[u]);
                }
                named_bar_sync(1, SPP_CONS);
                T* yi = ycol(iv);
                for (int r = r0 + tid; r < r1; r += SPP_CONS) {
                    int a, b;
                    if (rp_staged) { a = rs[r - r0a]; b = rs[r + 1 - r0a]; }
                    else { a = rowptr[r]; b = rowptr[r + 1]; }
                    a -= p0a; b -= p0a;
                    T sum = (T)0;
                    for (int q = a; q < b; ++q) sum = add_rn<T>(sum, prod[q]);
                    yi[r] = sum;
                }
                // the buffer written next is the one summed one vector ago: every thread has passed that sum
                // before it reaches the barrier above again
            }
            named_bar_sync(1, SPP_CONS);      // all row sums done before the stage (rowptr segment) is released
        } else {
            // long row: the CTA owns exactly one row; one vector of the block at a time
            for (int i = 0; i < np; ++i) {
                double acc = 0.0;
                for (int q = tid; q < nnzb; q += SPP_CONS)
                    acc += (double)mul_rn<T>(vals[p0 + q], __ldg(xcol(i) + colidx[p0 + q]));
                acc = warp_sum(acc);
                named_bar_sync(1, SPP_CONS);
                if (lane == 0) red[w] = acc;
                named_bar_sync(1, SPP_CONS);
                if (tid == 0) {
                    double tot = 0.0;
                    for (int ww = 0; ww < SPP_CONS / 32; ++ww) tot += red[ww];
                    ycol(i)[r0] = (T)tot;
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + 8 * s);
        if (++s == SPM_NSTG) { s = 0; ph ^= 1; }
    }
}

// Matrix-free stencil apply (SURVEY §8f-4): y = A x for the 5-/7-point Dirichlet stencil WITHOUT a stored matrix —
// 16 n bytes per apply instead of 12 nnz + 20 n (160 MB instead of 800 MB at n = 1e7).  One thread per row; the
// neighbours x[i ± 1], x[i ± nx], x[i ± nx ny] are L1/L2 hits (each row of the grid is read by three consecutive
// thread rows).  Products are rounded before they are added, in ascending column order — the CSR kernels' order — so
// the result is bit-identical to the assembled operator of b2k_op_create_stencil.  Carries the same fusions as
// k_spmv_pipe (shift, dot epilogue, normalise-on-load + vout, MGS-order dot, skip flag, peer window).
struct StencilApply {
    int64_t nx, ny, nz, row0;       // global grid, first global row of this shard
    int64_t n_rows;                 // local rows
    int64_t n_loc;                  // local x entries (== n_rows); beyond: halo [lo | hi]
    int64_t halo_lo;                // entries of the lo halo (plane below the shard)
    double c[7];
};

template <typename T>
__global__ void __launch_bounds__(256)
k_stencil_apply(const __grid_constant__ StencilApply sa, const T* __restrict__ x, const T* __restrict__ halo,
                T* __restrict__ y, T a0, T a1, int shifted, const T* __restrict__ dotv, double* __restrict__ part,
                unsigned* __restrict__ ticket, double* __restrict__ out, const SpmvFuse fz,
                const __grid_constant__ PeerStep ps) {
    __shared__ double red[32];
    __shared__ bool last;
    if (fz.stop && *reinterpret_cast<const volatile int*>(fz.stop)) return;
    if (ps.on && ps.seq_halo) {
        if (threadIdx.x == 0) {
            if (ps.wait_lo) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 0), ps.seq_halo);
            if (ps.wait_hi) peer_spin(ps.pd, peer_hflag(ps.pd, ps.pd.rank, ps.seq_halo, 1), ps.seq_halo);
        }
        __syncthreads();
    }
    const bool scaled = fz.xscale != nullptr;
    const T sc = scaled ? (T)(*fz.xscale) : (T)1;
    T* const vout = reinterpret_cast<T*>(fz.vout);
    const bool want_dot = (dotv != nullptr) || fz.dot_self;
    const T* const dsub = reinterpret_cast<const T*>(fz.dot_sub_vec);
    const T dsc = dsub ? (T)(*fz.dot_sub_scale) : (T)0;
    const int64_t plane = sa.nx * sa.ny;
    const T c0 = (T)sa.c[0], cw = (T)sa.c[1], ce = (T)sa.c[2], cs = (T)sa.c[3], cn = (T)sa.c[4], cd = (T)sa.c[5],
            cu = (T)sa.c[6];
    // x at local index l (may be below 0 / beyond n_loc: halo), already normalised
    auto X = [&](int64_t l) -> T {
        T v;
        if (l >= 0 && l < sa.n_loc) v = __ldg(x + l);
        else if (l < 0) v = __ldg(halo + (sa.halo_lo + l));
        else v = __ldg(halo + sa.halo_lo + (l - sa.n_loc));
        return scaled ? v * sc : v;
    };
    T dacc = (T)0;
    const bool small = plane * sa.nz < ((int64_t)1 << 31);
    const uint32_t nx32 = (uint32_t)sa.nx, ny32 = (uint32_t)sa.ny;
    // one stencil row: returns (a0 + a1 A) x at local row i and x_i itself (normalised)
    auto row = [&](int64_t i, T& xi) -> T {
        const int64_t g = sa.row0 + i;
        int64_t ix, iy, iz;
        if (small) {          // 32-bit index arithmetic: a 64-bit div/mod pair costs more than the whole stencil
            const uint32_t g32 = (uint32_t)g, t32 = g32 / nx32;
            ix = g32 - t32 * nx32;
            const uint32_t z32 = t32 / ny32;
            iy = t32 - z32 * ny32;
            iz = z32;
        } else {
            ix = g % sa.nx; iy = (g / sa.nx) % sa.ny; iz = g / plane;
        }
        T sum = (T)0;
        if (sa.nz > 1 && iz > 0) sum = add_rn<T>(sum, mul_rn<T>(cd, X(i - plane)));
        if (iy > 0) sum = add_rn<T>(sum, mul_rn<T>(cs, X(i - sa.nx)));
        if (ix > 0) sum = add_rn<T>(sum, mul_rn<T>(cw, X(i - 1)));
        xi = X(i);
        sum = add_rn<T>(sum, mul_rn<T>(c0, xi));
        if (ix < sa.nx - 1) sum = add_rn<T>(sum, mul_rn<T>(ce, X(i + 1)));
        if (iy < sa.ny - 1) sum = add_rn<T>(sum, mul_rn<T>(cn, X(i + sa.nx)));
        if (sa.nz > 1 && iz < sa.nz - 1) sum = add_rn<T>(sum, mul_rn<T>(cu, X(i + plane)));
        if (shifted) sum = fma(a0, __ldg(x + i), a1 * sum);
        return sum;
    };
    auto finish = [&](int64_t i, T sum, T xi) {
        y[i] = sum;
        if (vout) vout[i] = xi;
        if (want_dot) {
            const T dv = fz.dot_self ? xi : __ldg(dotv + i);
            dacc = fma(dv, dsub ? fma(-dsc, __ldg(dsub + i), sum) : sum, dacc);
        }
    };
    // two grid-strided rows per trip, both evaluated before either is stored (twice the loads in flight per thread;
    // the order in which a thread visits its rows — and with it the fused dot product — is unchanged)
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < sa.n_rows; i += 2 * stride) {
        const int64_t i2 = i + stride;
        const bool two = i2 < sa.n_rows;
        T xa, xb = (T)0;
        const T sa_ = row(i, xa);
        const T sb_ = two ? row(i2, xb) : (T)0;
        finish(i, sa_, xa);
        if (two) finish(i2, sb_, xb);
    }
    if (want_dot) {
        const double sblk = block_sum((double)dacc, red);
        if (threadIdx.x == 0) {
            part[blockIdx.x] = sblk;
            __threadfence();
            const unsigned t = atomicInc(ticket, gridDim.x - 1);
            last = (t == gridDim.x - 1);
        }
        __syncthreads();
        if (last) {
            __threadfence();
            double v2 = 0.0;
            const volatile double* pv = part;
            for (int gidx = threadIdx.x; gidx < (int)gridDim.x; gidx += blockDim.x) v2 += pv[gidx];
            const double tot = block_sum(v2, red);
            if (threadIdx.x == 0) {
                *out = tot;
                if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
            }
        }
    }
}

// Halo push through the peer window: my first send_lo entries go behind rank-1's lo entries (its hi halo), my
// last send_hi entries to the start of rank+1's receive buffer (its lo halo); the last CTA raises the flags.
template <typename T>
__global__ void __launch_bounds__(256)
k_halo_push(const T* __restrict__ x, int64_t n, const __grid_constant__ PeerStep ps, unsigned* __restrict__ ticket,
            const int* __restrict__ stop) {
    __shared__ bool last;
    if (stop && *reinterpret_cast<const volatile int*>(stop)) return;
    const PeerDev& pd = ps.pd;
    T* dn = ps.send_lo ? reinterpret_cast<T*>(pd.win[pd.rank - 1] + ps.dn_off) : nullptr;
    T* up = ps.send_hi ? reinterpret_cast<T*>(pd.win[pd.rank + 1] + ps.up_off) : nullptr;
    const int64_t total = ps.send_lo + ps.send_hi;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < ps.send_lo) dn[i] = x[i];
        else up[i - ps.send_lo] = x[n - ps.send_hi + (i - ps.send_lo)];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicInc(ticket, gridDim.x - 1);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence_system();
        if (dn) st_relaxed_sys_u64(peer_hflag(pd, pd.rank - 1, ps.seq_halo, 1), ps.seq_halo);
        if (up) st_relaxed_sys_u64(peer_hflag(pd, pd.rank + 1, ps.seq_halo, 0), ps.seq_halo);
    }
}

// stencil assembly -------------------------------------------------------------------
struct StencilDesc {
    int64_t nx, ny, nz;
    int64_t row0, nrows;   // global row range assembled here
    double c[7];
};

__device__ __forceinline__ int stencil_count(const StencilDesc& d, int64_t g) {
    const int64_t ix = g % d.nx, iy = (g / d.nx) % d.ny, iz = g / (d.nx * d.ny);
    int cnt = 1;
    cnt += (ix > 0) + (ix < d.nx - 1) + (iy > 0) + (iy < d.ny - 1);
    if (d.nz > 1) cnt += (iz > 0) + (iz < d.nz - 1);
    return cnt;
}

__global__ void k_stencil_count(StencilDesc d, int32_t* __restrict__ counts) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < d.nrows) counts[i] = stencil_count(d, d.row0 + i);
    if (i == d.nrows) counts[i] = 0;
}

template <typename T>
__global__ void k_stencil_fill(StencilDesc d, const int32_t* __restrict__ rowptr,
                               int64_t* __restrict__ gcol, T* __restrict__ vals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.nrows) return;
    const int64_t g = d.row0 + i;
    const int64_t ix = g % d.nx, iy = (g / d.nx) % d.ny, iz = g / (d.nx * d.ny);
    const int64_t plane = d.nx * d.ny;
    int p = rowptr[i];
    if (d.nz > 1 && iz > 0)        { gcol[p] = g - plane; vals[p] = (T)d.c[5]; ++p; }
    if (iy > 0)                    { gcol[p] = g - d.nx;  vals[p] = (T)d.c[3]; ++p; }
    if (ix > 0)                    { gcol[p] = g - 1;     vals[p] = (T)d.c[1]; ++p; }
    gcol[p] = g; vals[p] = (T)d.c[0]; ++p;
    if (ix < d.nx - 1)             { gcol[p] = g + 1;     vals[p] = (T)d.c[2]; ++p; }
    if (iy < d.ny - 1)             { gcol[p] = g + d.nx;  vals[p] = (T)d.c[4]; ++p; }
    if (d.nz > 1 && iz < d.nz - 1) { gcol[p] = g + plane; vals[p] = (T)d.c[6]; ++p; }
}

// global column -> local index (or halo slot)
__global__ void k_localize_cols(const int64_t* __restrict__ gcol, int32_t* __restrict__ col,
                                int64_t nnz, int64_t col0, int64_t n_loc, int64_t halo_lo,
                                int gather_all) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const int64_t g = gcol[i];
    if (gather_all) { col[i] = (int32_t)g; return; }
    int64_t l;
    if (g >= col0 && g < col0 + n_loc) l = g - col0;
    else if (g < col0) l = n_loc + (g - (col0 - halo_lo));
    else l = n_loc + halo_lo + (g - (col0 + n_loc));
    col[i] = (int32_t)l;
}

__global__ void k_minmax_cols(const int64_t* __restrict__ gcol, int64_t nnz,
                              unsigned long long* __restrict__ mn, unsigned long long* __restrict__ mx) {
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nnz;
         i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long g = (unsigned long long)gcol[i];
        lo = g < lo ? g : lo;
        hi = g > hi ? g : hi;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long l2 = __shfl_xor_sync(0xffffffffu, lo, o);
        const unsigned long long h2 = __shfl_xor_sync(0xffffffffu, hi, o);
        lo = l2 < lo ? l2 : lo;
        hi = h2 > hi ? h2 : hi;
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(mn, lo);
        atomicMax(mx, hi);
    }
}

template <typename T>
__global__ void k_dense_fill_splitmix(T* __restrict__ A, int64_t m, int64_t n, int64_t ld,
                                      uint64_t seed, uint64_t row0, uint64_t m_global) {
    const int64_t total = m * n;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = t / m, i = t - j * m;
        A[j * ld + i] = (T)(splitmix_unit(seed, row0 + (uint64_t)i + (uint64_t)j * m_global) - 0.5);
    }
}

// row blocks: greedy runs of rows with <= SP_NNZ nonzeros and <= SP_ROWS rows; a row longer
// than SP_NNZ forms its own block.
void build_rowblocks(const int32_t* rowptr, int64_t n, std::vector<int32_t>* blk) {
    blk->clear();
    blk->push_back(0);
    int64_t r = 0;
    while (r < n) {
        const int64_t start = r;
        const int32_t p0 = rowptr[r];
        if (rowptr[r + 1] - p0 > SP_NNZ) {
            ++r;
        } else {
            while (r < n && rowptr[r + 1] - p0 <= SP_NNZ && (r - start) < SP_ROWS) ++r;
        }
        blk->push_back((int32_t)r);
    }
}

// longest row and monotonicity of rowptr (device): out[0] = max row length, out[1] = #violations
__global__ void k_rowptr_stats(const int32_t* __restrict__ rowptr, int64_t n, int* __restrict__ out) {
    int mx = 0, bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int d = rowptr[i + 1] - rowptr[i];
        mx = d > mx ? d : mx;
        bad += d < 0;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const int m2 = __shfl_xor_sync(0xffffffffu, mx, o);
        mx = m2 > mx ? m2 : mx;
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(out, mx);
        if (bad) atomicAdd(out + 1, bad);
    }
}

// nnz-balanced partition: block b = rows [lower_bound(rowptr, b*T), lower_bound(rowptr, (b+1)*T)).
// With T = SP_NNZ - maxrow + 1 every block holds <= SP_NNZ nonzeros.
__global__ void k_rowblocks(const int32_t* __restrict__ rowptr, int64_t n, int T, int nblk,
                            int32_t* __restrict__ rowblk) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > nblk) return;
    if (b == nblk) { rowblk[b] = (int32_t)n; return; }
    const int64_t target = (int64_t)b * T;
    int64_t lo = 0, hi = n;           // first r in [0, n] with rowptr[r] >= target
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (rowptr[mid] >= target) hi = mid; else lo = mid + 1;
    }
    rowblk[b] = (int32_t)lo;
}

int32_t finish_csr(b2k_ctx* ctx, b2k_op* op) {
    const int64_t n = op->n_rows;
    int* d_stats;
    int h_stats[2] = {0, 0};
    B2K_CUDA(ctx, B2K_DMALLOC(&d_stats, 2 * sizeof(int)));
    B2K_CUDA(ctx, cudaMemsetAsync(d_stats, 0, 2 * sizeof(int), ctx->stream));
    if (n > 0) {
        k_rowptr_stats<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(op->rowptr, n, d_stats);
        B2K_LAUNCH_CHECK(ctx);
    }
    B2K_CUDA(ctx, cudaMemcpyAsync(h_stats, d_stats, sizeof(h_stats), cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    B2K_DFREE(d_stats);
    if (h_stats[1] != 0) return b2k_fail(ctx, B2K_EINVAL, "CSR: rowptr is not non-decreasing");
    const int maxrow = h_stats[0];
    if (maxrow <= SP_NNZ / 2) {
        const int T = SP_NNZ - maxrow + 1;
        op->nblk = (int32_t)std::max<int64_t>(1, (op->nnz + T - 1) / T);
        B2K_CUDA(ctx, B2K_DMALLOC(&op->rowblk, sizeof(int32_t) * (op->nblk + 1)));
        k_rowblocks<<<(op->nblk + 1 + 255) / 256, 256, 0, ctx->stream>>>(op->rowptr, n, T, op->nblk,
                                                                        op->rowblk);
        B2K_LAUNCH_CHECK(ctx);
    } else {
        // irregular matrix with very long rows: greedy partition on the host
        std::vector<int32_t> h_rowptr(n + 1), blk;
        B2K_CUDA(ctx, cudaMemcpyAsync(h_rowptr.data(), op->rowptr, sizeof(int32_t) * (n + 1),
                                      cudaMemcpyDeviceToHost, ctx->stream));
        B2K_TRY(b2k_stream_sync(ctx));
        build_rowblocks(h_rowptr.data(), n, &blk);
        op->nblk = (int32_t)blk.size() - 1;
        B2K_CUDA(ctx, B2K_DMALLOC(&op->rowblk, sizeof(int32_t) * blk.size()));
        B2K_CUDA(ctx, cudaMemcpyAsync(op->rowblk, blk.data(), sizeof(int32_t) * blk.size(),
                                      cudaMemcpyHostToDevice, ctx->stream));
        B2K_TRY(b2k_stream_sync(ctx));
    }
    B2K_CUDA(ctx, B2K_DMALLOC(&op->pblk, sizeof(int32_t) * (op->nblk + 1)));
    k_pblk<<<(op->nblk + 1 + 255) / 256, 256, 0, ctx->stream>>>(op->rowptr, op->rowblk, op->nblk + 1, op->pblk);
    B2K_LAUNCH_CHECK(ctx);
    B2K_CUDA(ctx, B2K_DMALLOC(&op->part, sizeof(double) * std::max(1, op->nblk)));
    return B2K_OK;
}

// raw host index arrays (int32/int64, base 0/1) -> device rowptr (int32) / global columns (int64)
template <typename IT>
__global__ void k_convert_rowptr(const IT* __restrict__ raw, int base, int32_t* __restrict__ out,
                                 int64_t count) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count;
         i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (int32_t)((int64_t)raw[i] - base);
}
template <typename IT>
__global__ void k_convert_cols(const IT* __restrict__ raw, int base, int64_t* __restrict__ out,
                               int64_t count) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count;
         i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (int64_t)raw[i] - base;
}

// Halo plan from the global column range of the local rows (dist only).
int32_t plan_halo(b2k_ctx* ctx, b2k_op* op, const int64_t* d_gcol) {
    op->n_loc_cols = ctx->spaces[0].n;
    op->halo_lo = op->halo_hi = op->send_lo = op->send_hi = 0;
    op->gather_all = 0;
    if (ctx->nranks == 1) return B2K_OK;
    unsigned long long* d_mm;
    B2K_CUDA(ctx, B2K_DMALLOC(&d_mm, 2 * sizeof(unsigned long long)));
    unsigned long long init[2] = {~0ull, 0ull};
    B2K_CUDA(ctx, cudaMemcpyAsync(d_mm, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    if (op->nnz > 0) {
        k_minmax_cols<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(d_gcol, op->nnz, d_mm, d_mm + 1);
        ctx->launches++;
    }
    unsigned long long mm[2];
    B2K_CUDA(ctx, cudaMemcpyAsync(mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    B2K_DFREE(d_mm);
    const int64_t col0 = ctx->row_offset, n_loc = op->n_loc_cols;
    int64_t lo = 0, hi = 0;
    if (op->nnz > 0) {
        lo = std::max<int64_t>(0, col0 - (int64_t)mm[0]);
        hi = std::max<int64_t>(0, (int64_t)mm[1] - (col0 + n_loc - 1));
    }
    // exchange (halo_lo, halo_hi, n_loc) with all ranks over the node-local rendezvous (host side, no NCCL)
    const int R = ctx->nranks;
    double mine[3] = {(double)lo, (double)hi, (double)n_loc};
    std::vector<double> all(3 * R);
    B2K_TRY(b2k_host_allgather(ctx, mine, sizeof(mine), all.data()));
    bool neighbour_ok = true;
    for (int r = 0; r < R; ++r) {
        const int64_t l = (int64_t)all[3 * r], h = (int64_t)all[3 * r + 1];
        if (l > 0 && (r == 0 || l > (int64_t)all[3 * (r - 1) + 2])) neighbour_ok = false;
        if (h > 0 && (r == R - 1 || h > (int64_t)all[3 * (r + 1) + 2])) neighbour_ok = false;
    }
    if (neighbour_ok) {
        op->halo_lo = lo;
        op->halo_hi = hi;
        op->send_hi = ctx->rank + 1 < R ? (int64_t)all[3 * (ctx->rank + 1)] : 0;      // rank+1's halo_lo
        op->send_lo = ctx->rank > 0 ? (int64_t)all[3 * (ctx->rank - 1) + 1] : 0;      // rank-1's halo_hi
        op->dn_lo = ctx->rank > 0 ? (int64_t)all[3 * (ctx->rank - 1)] : 0;
        // receive buffers: in the NVLink peer window when there is one (neighbours store into it directly),
        // at a heap offset that is the same on every rank; else private memory filled by ncclSend/Recv
        int64_t maxtot = 0;
        for (int r = 0; r < R; ++r) maxtot = std::max<int64_t>(maxtot, (int64_t)all[3 * r] + (int64_t)all[3 * r + 1]);
        if (b2k_peer_ok(ctx) && maxtot > 0) {
            const size_t region = (((size_t)maxtot * ctx->esize) + 255) & ~(size_t)255;
            const size_t off = b2k_peer_heap_alloc(ctx, 2 * region);          // same arithmetic on every rank
            if (off != SIZE_MAX) {
                op->peer_halo = 1;
                op->halo_off = off;
                op->halo_region = region;
            }
        }
        if (!op->peer_halo && !b2k_has_nccl(ctx))
            return b2k_fail(ctx, B2K_ENOTSUP, "halo of %lld entries does not fit the peer window (B2K_PEER_WINDOW_MB) "
                                              "and NCCL is disabled", (long long)maxtot);
        if (!op->peer_halo && lo + hi > 0) B2K_CUDA(ctx, B2K_DMALLOC(&op->halo, (size_t)(lo + hi) * ctx->esize));
    } else {
        if (!b2k_has_nccl(ctx))
            return b2k_fail(ctx, B2K_ENOTSUP, "operator couples non-adjacent row shards: needs the NCCL all-gather "
                                              "fallback, but NCCL is disabled");
        for (int r = 0; r < R; ++r)
            if ((int64_t)all[3 * r + 2] != n_loc)
                return b2k_fail(ctx, B2K_ENOTSUP,
                                "operator couples non-adjacent row shards and shards are unequal: "
                                "allgather fallback needs equal n_local");
        op->gather_all = 1;
        B2K_CUDA(ctx, B2K_DMALLOC(&op->xall, (size_t)n_loc * R * ctx->esize));
    }
    return B2K_OK;
}

int32_t localize(b2k_ctx* ctx, b2k_op* op, const int64_t* d_gcol) {
    if (op->nnz == 0) return B2K_OK;
    const int64_t blocks = (op->nnz + 255) / 256;
    k_localize_cols<<<(unsigned)blocks, 256, 0, ctx->stream>>>(d_gcol, op->colidx, op->nnz,
                                                               ctx->row_offset, op->n_loc_cols,
                                                               op->halo_lo, op->gather_all);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

template <typename IT>
void widen(const void* src, int64_t count, int base, std::vector<int64_t>* out) {
    const IT* s = (const IT*)src;
    out->resize(count);
    for (int64_t i = 0; i < count; ++i) (*out)[i] = (int64_t)s[i] - base;
}

}  // namespace

// ------------------------------------------------------------------ creation ----

// Upload raw index arrays and do all conversion / validation / planning on the device:
// host work is O(1), so a host-buffer eigsolve pays only the PCIe copies.
static int32_t create_csr_raw(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                              int64_t nnz, const void* rowptr, const void* colidx,
                              const void* vals, int32_t idx_bytes, int32_t index_base) {
    if (nnz >= (int64_t)1 << 31 || n_rows >= (int64_t)1 << 31)
        return b2k_fail(ctx, B2K_ENOTSUP, "CSR: nnz/rows per GPU must be < 2^31");
    // rows must be the length of a vector space of this context: space 0 in general, any space for a
    // rectangular operator on a single GPU (the (A, A') pair of lssolve / svdsolve)
    bool rows_ok = n_rows == ctx->spaces[0].n;
    if (!rows_ok && ctx->nranks == 1)
        for (const auto& sp : ctx->spaces) rows_ok = rows_ok || sp.n == n_rows;
    if (!rows_ok)
        return b2k_fail(ctx, B2K_EDIM, "CSR: %lld local rows but space 0 holds %lld",
                        (long long)n_rows, (long long)ctx->spaces[0].n);
    const int64_t rp0 = idx_bytes == 8 ? ((const int64_t*)rowptr)[0] : ((const int32_t*)rowptr)[0];
    const int64_t rpn = idx_bytes == 8 ? ((const int64_t*)rowptr)[n_rows] : ((const int32_t*)rowptr)[n_rows];
    if (rp0 - index_base != 0 || rpn - index_base != nnz)
        return b2k_fail(ctx, B2K_EINVAL, "op_create_csr: rowptr does not span [0, nnz]");
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* op = new b2k_op();
    op->kind = 0;
    op->n_rows = n_rows;
    op->n_cols = n_cols;
    op->nnz = nnz;
    int64_t* d_gcol = nullptr;
    void* d_raw = nullptr;
    const int64_t nnz1 = std::max<int64_t>(1, nnz);
    const size_t raw_bytes = (size_t)idx_bytes * std::max<int64_t>(nnz1, n_rows + 1);
    int32_t rc = B2K_OK;
    auto fail = [&](int32_t code) {
        cudaStreamSynchronize(ctx->stream);
        if (d_gcol) B2K_DFREE(d_gcol);
        if (d_raw) B2K_DFREE(d_raw);
        b2k_op_destroy(ctx, op);
        return code;
    };
#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return fail(b2k_fail(ctx, B2K_ECUDA, "op_create_csr: %s -> %s", #call,           \
                                 cudaGetErrorString(e__)));                                  \
    } while (0)
    CK(B2K_DMALLOC(&op->rowptr, sizeof(int32_t) * (n_rows + 1 + 8)));
    CK(B2K_DMALLOC(&op->colidx, sizeof(int32_t) * (nnz1 + 8)));
    CK(B2K_DMALLOC(&op->vals, (size_t)ctx->esize * (nnz1 + 8)));
    CK(B2K_DMALLOC(&d_gcol, sizeof(int64_t) * nnz1));
    CK(B2K_DMALLOC(&d_raw, raw_bytes));
    const int g = ctx->num_sms * 8;
    CK(cudaMemcpyAsync(d_raw, rowptr, (size_t)idx_bytes * (n_rows + 1), cudaMemcpyHostToDevice, ctx->stream));
    if (idx_bytes == 8) k_convert_rowptr<int64_t><<<g, 256, 0, ctx->stream>>>((const int64_t*)d_raw, index_base, op->rowptr, n_rows + 1);
    else k_convert_rowptr<int32_t><<<g, 256, 0, ctx->stream>>>((const int32_t*)d_raw, index_base, op->rowptr, n_rows + 1);
    ctx->launches++;
    if (nnz > 0) {
        CK(cudaMemcpyAsync(d_raw, colidx, (size_t)idx_bytes * nnz, cudaMemcpyHostToDevice, ctx->stream));
        if (idx_bytes == 8) k_convert_cols<int64_t><<<g, 256, 0, ctx->stream>>>((const int64_t*)d_raw, index_base, d_gcol, nnz);
        else k_convert_cols<int32_t><<<g, 256, 0, ctx->stream>>>((const int32_t*)d_raw, index_base, d_gcol, nnz);
        ctx->launches++;
        CK(cudaMemcpyAsync(op->vals, vals, (size_t)ctx->esize * nnz, cudaMemcpyHostToDevice, ctx->stream));
        // validate the column range on the device
        unsigned long long* d_mm;
        CK(B2K_DMALLOC(&d_mm, 2 * sizeof(unsigned long long)));
        unsigned long long init[2] = {~0ull, 0ull}, mm[2];
        CK(cudaMemcpyAsync(d_mm, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        k_minmax_cols<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(d_gcol, nnz, d_mm, d_mm + 1);
        ctx->launches++;
        CK(cudaMemcpyAsync(mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        B2K_DFREE(d_mm);
        const int64_t colmax = ctx->nranks > 1 ? ctx->n_global : n_cols;
        // negative columns wrap to huge unsigned values and are caught by the max test
        if ((int64_t)mm[1] >= colmax || (int64_t)mm[1] < 0)
            return fail(b2k_fail(ctx, B2K_EINVAL, "op_create_csr: column index out of range [0, %lld)",
                                 (long long)colmax));
    }
#undef CK
    rc = plan_halo(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = localize(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = finish_csr(ctx, op);
    if (rc != B2K_OK) return fail(rc);
    cudaStreamSynchronize(ctx->stream);
    B2K_DFREE(d_gcol);
    B2K_DFREE(d_raw);
    ctx->ops.push_back(op);
    *out = op;
    return B2K_OK;
}

extern "C" int32_t b2k_op_create_csr(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                                     int64_t nnz, const void* rowptr, const void* colidx,
                                     const void* vals, int32_t idx_bytes, int32_t index_base) {
    if (!ctx || !out || !rowptr || (nnz > 0 && (!colidx || !vals))) return B2K_EINVAL;
    if ((idx_bytes != 4 && idx_bytes != 8) || (index_base != 0 && index_base != 1))
        return b2k_fail(ctx, B2K_EINVAL, "op_create_csr: idx_bytes must be 4/8, index_base 0/1");
    return create_csr_raw(ctx, out, n_rows, n_cols, nnz, rowptr, colidx, vals, idx_bytes, index_base);
}

extern "C" int32_t b2k_op_create_csc(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                                     int64_t nnz, const void* colptr, const void* rowval,
                                     const void* nzval, int32_t idx_bytes, int32_t index_base) {
    if (!ctx || !out || !colptr || (nnz > 0 && (!rowval || !nzval))) return B2K_EINVAL;
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "op_create_csc: single-GPU contexts only");
    if ((idx_bytes != 4 && idx_bytes != 8) || (index_base != 0 && index_base != 1))
        return b2k_fail(ctx, B2K_EINVAL, "op_create_csc: idx_bytes must be 4/8, index_base 0/1");
    std::vector<int64_t> cp, rv;
    if (idx_bytes == 8) {
        widen<int64_t>(colptr, n_cols + 1, index_base, &cp);
        widen<int64_t>(rowval, nnz, index_base, &rv);
    } else {
        widen<int32_t>(colptr, n_cols + 1, index_base, &cp);
        widen<int32_t>(rowval, nnz, index_base, &rv);
    }
    // counting-sort transpose: CSC(A) -> CSR(A); within a row, columns come out ascending
    std::vector<int64_t> rp(n_rows + 1, 0), gc(nnz);
    for (int64_t i = 0; i < nnz; ++i) {
        if (rv[i] < 0 || rv[i] >= n_rows)
            return b2k_fail(ctx, B2K_EINVAL, "op_create_csc: row index out of range");
        rp[rv[i] + 1]++;
    }
    for (int64_t r = 0; r < n_rows; ++r) rp[r + 1] += rp[r];
    std::vector<int64_t> next(rp.begin(), rp.end() - 1);
    const size_t es = ctx->esize;
    std::vector<char> vv(es * std::max<int64_t>(1, nnz));
    for (int64_t c = 0; c < n_cols; ++c)
        for (int64_t p = cp[c]; p < cp[c + 1]; ++p) {
            const int64_t dst = next[rv[p]]++;
            gc[dst] = c;
            memcpy(vv.data() + es * dst, (const char*)nzval + es * p, es);
        }
    return create_csr_raw(ctx, out, n_rows, n_cols, nnz, rp.data(), gc.data(), vv.data(), 8, 0);
}

extern "C" int32_t b2k_op_create_stencil(b2k_ctx* ctx, b2k_op** out, int64_t nx, int64_t ny,
                                         int64_t nz, const double c[7]) {
    if (!ctx || !out || !c || nx < 1 || ny < 1 || nz < 1) return B2K_EINVAL;
    const int64_t nglob = nx * ny * nz;
    const int64_t n_loc = ctx->spaces[0].n;
    if (ctx->nranks == 1 && nglob != n_loc)
        return b2k_fail(ctx, B2K_EDIM, "stencil: grid has %lld points, space 0 holds %lld",
                        (long long)nglob, (long long)n_loc);
    if (ctx->nranks > 1 && nglob != ctx->n_global)
        return b2k_fail(ctx, B2K_EDIM, "stencil: grid has %lld points, n_global is %lld",
                        (long long)nglob, (long long)ctx->n_global);
    if (n_loc >= ((int64_t)1 << 31) / 8) return b2k_fail(ctx, B2K_ENOTSUP, "stencil: shard too large");
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* op = new b2k_op();
    op->kind = 0;
    op->n_rows = n_loc;
    op->n_cols = nglob;
    StencilDesc d;
    d.nx = nx; d.ny = ny; d.nz = nz; d.row0 = ctx->row_offset; d.nrows = n_loc;
    for (int i = 0; i < 7; ++i) d.c[i] = c[i];
    int32_t* counts = nullptr;
    int64_t* d_gcol = nullptr;
    void* tmp = nullptr;
    int32_t rc = B2K_OK;
    auto fail = [&](int32_t code) {
        if (counts) B2K_DFREE(counts);
        if (d_gcol) B2K_DFREE(d_gcol);
        if (tmp) B2K_DFREE(tmp);
        b2k_op_destroy(ctx, op);
        return code;
    };
#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return fail(b2k_fail(ctx, B2K_ECUDA, "stencil: %s -> %s", #call,                 \
                                 cudaGetErrorString(e__)));                                  \
    } while (0)
    CK(B2K_DMALLOC(&counts, sizeof(int32_t) * (n_loc + 1)));
    CK(B2K_DMALLOC(&op->rowptr, sizeof(int32_t) * (n_loc + 1 + 8)));
    const unsigned blocks = (unsigned)((n_loc + 1 + 255) / 256);
    k_stencil_count<<<blocks, 256, 0, ctx->stream>>>(d, counts);
    ctx->launches++;
    size_t tmp_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, op->rowptr, (int)(n_loc + 1),
                                     ctx->stream));
    CK(B2K_DMALLOC(&tmp, tmp_bytes));
    CK(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, op->rowptr, (int)(n_loc + 1),
                                     ctx->stream));
    int32_t h_nnz = 0;
    CK(cudaMemcpyAsync(&h_nnz, op->rowptr + n_loc, sizeof(int32_t), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    op->nnz = h_nnz;
    CK(B2K_DMALLOC(&op->colidx, sizeof(int32_t) * (std::max<int64_t>(1, op->nnz) + 8)));
    CK(B2K_DMALLOC(&op->vals, (size_t)ctx->esize * (std::max<int64_t>(1, op->nnz) + 8)));
    CK(B2K_DMALLOC(&d_gcol, sizeof(int64_t) * std::max<int64_t>(1, op->nnz)));
    if (n_loc > 0) {
        if (ctx->dtype == B2K_F64)
            k_stencil_fill<double><<<blocks, 256, 0, ctx->stream>>>(d, op->rowptr, d_gcol,
                                                                    (double*)op->vals);
        else
            k_stencil_fill<float><<<blocks, 256, 0, ctx->stream>>>(d, op->rowptr, d_gcol,
                                                                   (float*)op->vals);
        ctx->launches++;
    }
#undef CK
    rc = plan_halo(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = localize(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = finish_csr(ctx, op);
    if (rc != B2K_OK) return fail(rc);
    cudaStreamSynchronize(ctx->stream);
    B2K_DFREE(counts);
    B2K_DFREE(d_gcol);
    B2K_DFREE(tmp);
    ctx->ops.push_back(op);
    *out = op;
    return B2K_OK;
}

// Matrix-free form of b2k_op_create_stencil: nothing is assembled, `apply` evaluates the stencil (k_stencil_apply).
// Row-sharded contexts shard by whole grid lines (2-D) / planes (3-D); the halo is one line / plane per neighbour.
extern "C" int32_t b2k_op_create_stencil_free(b2k_ctx* ctx, b2k_op** out, int64_t nx, int64_t ny, int64_t nz,
                                              const double c[7]) {
    if (!ctx || !out || !c || nx < 1 || ny < 1 || nz < 1) return B2K_EINVAL;
    const int64_t nglob = nx * ny * nz;
    const int64_t n_loc = ctx->spaces[0].n;
    if (ctx->nranks == 1 && nglob != n_loc)
        return b2k_fail(ctx, B2K_EDIM, "stencil: grid has %lld points, space 0 holds %lld", (long long)nglob, (long long)n_loc);
    if (ctx->nranks > 1 && nglob != ctx->n_global)
        return b2k_fail(ctx, B2K_EDIM, "stencil: grid has %lld points, n_global is %lld", (long long)nglob,
                        (long long)ctx->n_global);
    const int64_t unit = nz > 1 ? nx * ny : nx;           // one plane / one line
    if (ctx->nranks > 1 && (ctx->row_offset % unit != 0 || n_loc % unit != 0 || n_loc < unit))
        return b2k_fail(ctx, B2K_ENOTSUP, "matrix-free stencil: shards must be whole grid %s", nz > 1 ? "planes" : "lines");
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* op = new b2k_op();
    op->kind = 2;
    op->n_rows = n_loc;
    op->n_cols = nglob;
    op->nnz = 0;
    op->snx = nx; op->sny = ny; op->snz = nz; op->srow0 = ctx->row_offset;
    for (int i = 0; i < 7; ++i) op->sc[i] = c[i];
    op->n_loc_cols = n_loc;
    op->nblk = 0;
    int32_t rc = B2K_OK;
    if (ctx->nranks > 1) {
        // same halo plan as a CSR operator with this column range: one unit below, one above
        op->halo_lo = ctx->rank > 0 ? unit : 0;
        op->halo_hi = ctx->rank + 1 < ctx->nranks ? unit : 0;
        op->send_lo = op->halo_lo;      // symmetric: what I need from rank-1 is what it needs from me
        op->send_hi = op->halo_hi;
        op->dn_lo = ctx->rank > 1 ? unit : 0;             // rank-1's own lo halo (0 if rank-1 is rank 0)
        const size_t region = (((size_t)2 * unit * ctx->esize) + 255) & ~(size_t)255;
        if (b2k_peer_ok(ctx)) {
            const size_t off = b2k_peer_heap_alloc(ctx, 2 * region);
            if (off != SIZE_MAX) { op->peer_halo = 1; op->halo_off = off; op->halo_region = region; }
        }
        if (!op->peer_halo) {
            if (!b2k_has_nccl(ctx)) rc = b2k_fail(ctx, B2K_ENOTSUP, "stencil halo does not fit the peer window and NCCL is disabled");
            else if (B2K_DMALLOC(&op->halo, (size_t)(op->halo_lo + op->halo_hi) * ctx->esize) != cudaSuccess)
                rc = b2k_fail(ctx, B2K_ENOMEM, "stencil: halo allocation failed");
        }
    }
    if (rc == B2K_OK && B2K_DMALLOC(&op->part, sizeof(double) * 4096) != cudaSuccess)
        rc = b2k_fail(ctx, B2K_ENOMEM, "stencil: partial buffer allocation failed");
    if (rc != B2K_OK) { b2k_op_release(ctx, op); return rc; }
    ctx->ops.push_back(op);
    *out = op;
    return B2K_OK;
}

static int32_t alloc_dense(b2k_ctx* ctx, b2k_op** out, int64_t m_local, int64_t n) {
    if (m_local < 1 || n < 1) return b2k_fail(ctx, B2K_EINVAL, "dense: bad shape");
    if (m_local != ctx->spaces[0].n)
        return b2k_fail(ctx, B2K_EDIM, "dense: %lld local rows but space 0 holds %lld",
                        (long long)m_local, (long long)ctx->spaces[0].n);
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* op = new b2k_op();
    op->kind = 1;
    op->n_rows = m_local;
    op->n_cols = n;
    op->nnz = m_local * n;
    op->ld = ((m_local + 31) / 32) * 32;
    const size_t bytes = (size_t)op->ld * n * ctx->esize;
    cudaError_t e = B2K_DMALLOC(&op->A, bytes);
    if (e != cudaSuccess) {
        delete op;
        return b2k_fail(ctx, B2K_ENOMEM, "dense: B2K_DMALLOC(%zu) failed: %s", bytes,
                        cudaGetErrorString(e));
    }
    cudaMemsetAsync(op->A, 0, bytes, ctx->stream);
    ctx->ops.push_back(op);
    *out = op;
    return B2K_OK;
}

extern "C" int32_t b2k_op_create_dense(b2k_ctx* ctx, b2k_op** out, int64_t m_local, int64_t n,
                                       const void* host_colmajor, int64_t ld) {
    if (!ctx || !out || !host_colmajor || ld < m_local) return B2K_EINVAL;
    B2K_TRY(alloc_dense(ctx, out, m_local, n));
    b2k_op* op = *out;
    B2K_CUDA(ctx, cudaMemcpy2DAsync(op->A, (size_t)op->ld * ctx->esize, host_colmajor,
                                    (size_t)ld * ctx->esize, (size_t)m_local * ctx->esize, n,
                                    cudaMemcpyHostToDevice, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

extern "C" int32_t b2k_op_create_dense_splitmix(b2k_ctx* ctx, b2k_op** out, int64_t m_local,
                                                int64_t n, uint64_t seed) {
    if (!ctx || !out) return B2K_EINVAL;
    B2K_TRY(alloc_dense(ctx, out, m_local, n));
    b2k_op* op = *out;
    const uint64_t mg = ctx->nranks > 1 ? (uint64_t)ctx->n_global : (uint64_t)m_local;
    if (ctx->dtype == B2K_F64)
        k_dense_fill_splitmix<double><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(
            (double*)op->A, m_local, n, op->ld, seed, (uint64_t)ctx->row_offset, mg);
    else
        k_dense_fill_splitmix<float><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(
            (float*)op->A, m_local, n, op->ld, seed, (uint64_t)ctx->row_offset, mg);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

void b2k_op_release(b2k_ctx* ctx, b2k_op* op) {
    cudaStream_t st = ctx ? ctx->stream : nullptr;
    void* ptrs[] = {op->rowptr, op->colidx, op->vals, op->rowblk, op->pblk, op->part, op->halo, op->xall, op->A};
    for (void* p : ptrs) b2k_dfree(p, st);     // stream-ordered: pending kernels finish first
    delete op;
}

extern "C" int32_t b2k_op_destroy(b2k_ctx* ctx, b2k_op* op) {
    if (!op) return B2K_OK;
    if (ctx) {
        cudaSetDevice(ctx->device);
        for (size_t i = 0; i < ctx->ops.size(); ++i)
            if (ctx->ops[i] == op) {
                ctx->ops.erase(ctx->ops.begin() + i);
                break;
            }
    }
    b2k_op_release(ctx, op);
    return B2K_OK;
}

extern "C" int32_t b2k_op_info(const b2k_op* op, int64_t* n_rows, int64_t* n_cols, int64_t* nnz,
                               int32_t* kind) {
    if (!op) return B2K_EINVAL;
    if (n_rows) *n_rows = op->n_rows;
    if (n_cols) *n_cols = op->n_cols;
    if (nnz) *nnz = op->nnz;
    if (kind) *kind = op->kind;
    return B2K_OK;
}

extern "C" int32_t b2k_op_csr_download(b2k_ctx* ctx, const b2k_op* op, int32_t* rowptr,
                                       int32_t* colidx, void* vals) {
    if (!ctx || !op) return B2K_EINVAL;
    if (op->kind != 0) return b2k_fail(ctx, B2K_ENOTSUP, "op_csr_download: not an assembled CSR operator");
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    if (rowptr)
        B2K_CUDA(ctx, cudaMemcpyAsync(rowptr, op->rowptr, sizeof(int32_t) * (op->n_rows + 1),
                                      cudaMemcpyDeviceToHost, ctx->stream));
    if (colidx)
        B2K_CUDA(ctx, cudaMemcpyAsync(colidx, op->colidx, sizeof(int32_t) * op->nnz,
                                      cudaMemcpyDeviceToHost, ctx->stream));
    if (vals)
        B2K_CUDA(ctx, cudaMemcpyAsync(vals, op->vals, (size_t)ctx->esize * op->nnz,
                                      cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

// ------------------------------------------------------------------ transpose ----
// CSR(A') from CSR(A) on the device: a stable radix sort of the nonzeros by column (CUB) keeps, inside each column of
// A, the order of the nonzeros in CSR(A) — rows ascending — so row c of A' lists its columns in ascending order, as
// scipy's A.T.tocsr() with sorted indices does.  The row of a nonzero is found by binary search in rowptr; the row
// pointer of A' by binary search in the sorted columns.  Setup cost: 2 x 12 nnz bytes moved by the sort plus the
// gathers; the matrix never leaves the device.
namespace {

__global__ void k_iota(uint32_t* __restrict__ out, int64_t count) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (uint32_t)i;
}

// nonzero k of A' is nonzero perm[k] of A: its column in A' is the row of perm[k] in A
template <typename T>
__global__ void k_transpose_gather(const int32_t* __restrict__ rowptr, int64_t n_rows, const T* __restrict__ vals,
                                   const uint32_t* __restrict__ perm, int64_t nnz, int32_t* __restrict__ tcol,
                                   T* __restrict__ tvals) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t q = perm[k];
        int64_t lo = 0, hi = n_rows;          // last r with rowptr[r] <= q
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (rowptr[mid] <= q) lo = mid; else hi = mid;
        }
        tcol[k] = (int32_t)lo;
        tvals[k] = vals[q];
    }
}

// trowptr[c] = first k with sorted_col[k] >= c, c = 0 .. n_cols
__global__ void k_transpose_rowptr(const uint32_t* __restrict__ scol, int64_t nnz, int64_t n_cols,
                                   int32_t* __restrict__ trowptr) {
    for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c <= n_cols; c += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = nnz;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)scol[mid] >= c) hi = mid; else lo = mid + 1;
        }
        trowptr[c] = (int32_t)lo;
    }
}

}  // namespace

extern "C" int32_t b2k_op_create_transpose(b2k_ctx* ctx, b2k_op** out, const b2k_op* op) {
    if (!ctx || !out || !op) return B2K_EINVAL;
    if (ctx->nranks > 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "op_create_transpose: row-sharded contexts are not supported; assemble A' "
                                          "on the host and pass (A, At)");
    if (op->kind == 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "op_create_transpose: dense operator; b2k_op_apply_adjoint applies A' "
                                          "directly");
    if (op->kind == 2)
        return b2k_fail(ctx, B2K_ENOTSUP, "op_create_transpose: matrix-free stencil; create the stencil with the "
                                          "west/east, south/north and down/up coefficients swapped");
    const int64_t m = op->n_cols, n = op->n_rows, nnz = op->nnz;
    if (m >= ((int64_t)1 << 31)) return b2k_fail(ctx, B2K_ENOTSUP, "op_create_transpose: A has >= 2^31 columns");
    bool rows_ok = false;
    for (const auto& sp : ctx->spaces) rows_ok = rows_ok || sp.n == m;
    if (!rows_ok)
        return b2k_fail(ctx, B2K_EDIM, "op_create_transpose: A' has %lld rows, but no vector space of the context "
                                       "has that length", (long long)m);
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* t = new b2k_op();
    t->kind = 0;
    t->n_rows = m;
    t->n_cols = n;
    t->nnz = nnz;
    const int64_t nnz1 = std::max<int64_t>(1, nnz);
    uint32_t *iota = nullptr, *perm = nullptr, *scol = nullptr;
    void* tmp = nullptr;
    auto release = [&]() {
        cudaStreamSynchronize(ctx->stream);
        if (iota) B2K_DFREE(iota);
        if (perm) B2K_DFREE(perm);
        if (scol) B2K_DFREE(scol);
        if (tmp) B2K_DFREE(tmp);
    };
    auto fail = [&](int32_t code) {
        release();
        b2k_op_release(ctx, t);
        return code;
    };
#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return fail(b2k_fail(ctx, B2K_ECUDA, "op_create_transpose: %s -> %s", #call,     \
                                 cudaGetErrorString(e__)));                                  \
    } while (0)
    CK(B2K_DMALLOC(&t->rowptr, sizeof(int32_t) * (m + 1 + 8)));
    CK(B2K_DMALLOC(&t->colidx, sizeof(int32_t) * (nnz1 + 8)));
    CK(B2K_DMALLOC(&t->vals, (size_t)ctx->esize * (nnz1 + 8)));
    CK(B2K_DMALLOC(&iota, sizeof(uint32_t) * nnz1));
    CK(B2K_DMALLOC(&perm, sizeof(uint32_t) * nnz1));
    CK(B2K_DMALLOC(&scol, sizeof(uint32_t) * nnz1));
    const int g = ctx->num_sms * 8;
    if (nnz > 0) {
        int end_bit = 1;
        while (end_bit < 32 && ((int64_t)1 << end_bit) < m) ++end_bit;
        k_iota<<<g, 256, 0, ctx->stream>>>(iota, nnz);
        ctx->launches++;
        size_t tmp_bytes = 0;
        const uint32_t* keys = reinterpret_cast<const uint32_t*>(op->colidx);
        CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, scol, iota, perm, (int)nnz, 0, end_bit,
                                           ctx->stream));
        CK(B2K_DMALLOC(&tmp, tmp_bytes));
        CK(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, scol, iota, perm, (int)nnz, 0, end_bit,
                                           ctx->stream));
        if (ctx->dtype == B2K_F64)
            k_transpose_gather<double><<<g, 256, 0, ctx->stream>>>(op->rowptr, n, (const double*)op->vals, perm, nnz,
                                                                   t->colidx, (double*)t->vals);
        else
            k_transpose_gather<float><<<g, 256, 0, ctx->stream>>>(op->rowptr, n, (const float*)op->vals, perm, nnz,
                                                                  t->colidx, (float*)t->vals);
        ctx->launches++;
    }
    k_transpose_rowptr<<<g, 256, 0, ctx->stream>>>(scol, nnz, m, t->rowptr);
    ctx->launches++;
    CK(cudaGetLastError());
#undef CK
    int32_t rc = plan_halo(ctx, t, nullptr);
    if (rc == B2K_OK) rc = finish_csr(ctx, t);
    if (rc != B2K_OK) return fail(rc);
    release();
    ctx->ops.push_back(t);
    *out = t;
    return B2K_OK;
}

// ------------------------------------------------------------------ apply ----

static bool g_spmv_pipe = true;
extern "C" int32_t b2k_debug_set_onepass_variant(int32_t v);     // defined with the one-pass dense step below
static int g_spmv_variant = 1;     // 1 (default): 2 stages x 4 CTAs/SM, 0: 3 stages x 3 CTAs/SM (B2K_SPMV_VARIANT)

extern "C" int32_t b2k_debug_set_spmv_pipe(int32_t on) {
    g_spmv_pipe = on != 0;
    return B2K_OK;
}

extern "C" int32_t b2k_debug_set_spmv_variant(int32_t v) {
    g_spmv_variant = v == 0 ? 0 : 1;
    return B2K_OK;
}

// opt in to > 48 KB dynamic shared memory for the pipelined SpMV (called per context)
int32_t b2k_spmv_init(b2k_ctx* ctx) {
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_spmm_pipe<double>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SpmLayout<double>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_spmm_pipe<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SpmLayout<float>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<double, 3, 3>), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SppLayout<double, 3>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<float, 3, 3>), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SppLayout<float, 3>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<double, 2, 4>), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SppLayout<double, 2>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<float, 2, 4>), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SppLayout<float, 2>::SMEM));
    const char* sv = getenv("B2K_SPMV_VARIANT");
    if (sv) g_spmv_variant = atoi(sv) == 0 ? 0 : 1;
    const char* ov = getenv("B2K_ONEPASS_VARIANT");       // kernel of the flagged one-pass GKL step: 0 = A (default), 1 = B
    if (ov && (ov[0] == '0' || ov[0] == '1')) b2k_debug_set_onepass_variant(ov[0] - '0');
    return B2K_OK;
}

int32_t b2k_enqueue_apply(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y,
                          double a0, double a1, bool shifted, const VecRef* dotv, int dot_slot) {
    return b2k_enqueue_apply_fused(ctx, op, x, y, a0, a1, shifted, dotv,
                                   dotv ? ctx->d_res + dot_slot : nullptr, nullptr);
}

// Halo traffic of one apply through the peer window, for sequence number `seq`: what I send where, what I wait for.
int32_t b2k_op_peer_halo(const b2k_ctx* ctx, const b2k_op* op, unsigned long long seq, PeerStep* ps) {
    if (!op->peer_halo) return B2K_ENOTSUP;
    const size_t par = (size_t)(seq & 1ull) * op->halo_region;
    ps->seq_halo = seq;
    ps->send_lo = op->send_lo;
    ps->send_hi = op->send_hi;
    ps->dn_off = op->halo_off + par + (size_t)op->dn_lo * ctx->esize;     // behind rank-1's lo entries
    ps->up_off = op->halo_off + par;                                      // start of rank+1's buffer
    ps->wait_lo = op->halo_lo > 0;
    ps->wait_hi = op->halo_hi > 0;
    return B2K_OK;
}

bool b2k_op_has_peer_halo(const b2k_op* op) { return op->peer_halo != 0; }

// fz (optional): normalise-on-gather / write the normalised operand / dot with it / skip flag — see SpmvFuse.
int32_t b2k_enqueue_apply_fused(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y,
                                double a0, double a1, bool shifted, const VecRef* dotv, double* dot_out,
                                const SpmvFuse* fzp) {
    SpmvFuse fz;
    memset(&fz, 0, sizeof(fz));
    if (fzp) fz = *fzp;
    if (fzp && op->kind == 1) return b2k_fail(ctx, B2K_ENOTSUP, "fused apply: CSR / stencil operators only");
    if ((fz.vout || fz.dot_self) && (op->n_rows != x.n))
        return b2k_fail(ctx, B2K_EDIM, "fused apply: needs a square operator (row r <-> x[r])");
    if (fz.dot_self && !dot_out) return b2k_fail(ctx, B2K_EINVAL, "fused apply: dot_self without an output slot");
    if (op->kind == 1) {
        if (shifted || dotv) return b2k_fail(ctx, B2K_ENOTSUP, "dense apply: no shift/dot fusion");
        if (x.n != op->n_cols || y.n != op->n_rows)
            return b2k_fail(ctx, B2K_EDIM, "dense apply: x has %lld (want %lld), y has %lld (want %lld)",
                            (long long)x.n, (long long)op->n_cols, (long long)y.n,
                            (long long)op->n_rows);
        return b2k_panel_unproject_dev(ctx, op->A, op->ld, op->n_rows, (int32_t)op->n_cols, y, x.ptr);
    }
    // one GPU: x must span all columns (a rectangular operator takes x from the matching space);
    // row-sharded: x is the local slice and the halo plan supplies the rest
    if (ctx->nranks == 1 ? x.n != op->n_cols : x.n != op->n_loc_cols)
        return b2k_fail(ctx, B2K_EDIM, "apply: x has %lld entries, operator wants %lld",
                        (long long)x.n, (long long)(ctx->nranks == 1 ? op->n_cols : op->n_loc_cols));
    if (y.n != op->n_rows)
        return b2k_fail(ctx, B2K_EDIM, "apply: y has %lld entries, operator has %lld rows",
                        (long long)y.n, (long long)op->n_rows);
    if (x.ptr == y.ptr) return b2k_fail(ctx, B2K_EINVAL, "apply: y must not alias x");
    if (shifted && x.n != y.n) return b2k_fail(ctx, B2K_EDIM, "shifted apply needs a square operator");
    if (op->n_rows == 0) return B2K_OK;
    const void* xsrc = x.ptr;
    int32_t n_loc = (int32_t)x.n;
    const void* halo = op->halo;
    PeerStep ps;
    memset(&ps, 0, sizeof(ps));
    if (ctx->nranks > 1 && b2k_peer_ok(ctx)) {
        ps.pd = *b2k_peer_dev(ctx);
        ps.on = 1;
        ps.seq_alpha = fz.seq_alpha;
    }
    if (ctx->nranks > 1) {
        if (op->peer_halo) {
            // the neighbours store my boundary rows straight into my window; the kernel waits for their flags
            unsigned long long hs = fz.seq_halo;
            if (!hs) {
                hs = b2k_peer_next_seq(ctx, 4);
                B2K_TRY(b2k_op_peer_halo(ctx, op, hs, &ps));
                const int64_t total = ps.send_lo + ps.send_hi;
                if (total > 0) {
                    const int g = (int)std::max<int64_t>(1, std::min<int64_t>((total + 1023) / 1024, ctx->num_sms));
                    if (ctx->dtype == B2K_F64)
                        k_halo_push<double><<<g, 256, 0, ctx->stream>>>((const double*)x.ptr, x.n, ps,
                                                                        ctx->d_sync + B2K_SYNC_HALO, fz.stop);
                    else
                        k_halo_push<float><<<g, 256, 0, ctx->stream>>>((const float*)x.ptr, x.n, ps,
                                                                       ctx->d_sync + B2K_SYNC_HALO, fz.stop);
                    B2K_LAUNCH_CHECK(ctx);
                }
            } else {
                B2K_TRY(b2k_op_peer_halo(ctx, op, hs, &ps));
            }
            halo = b2k_peer_local(ctx) + op->halo_off + (size_t)(hs & 1ull) * op->halo_region;
        } else if (op->gather_all) {
            B2K_TRY(b2k_nccl_allgather(ctx, x.ptr, op->xall, (size_t)x.n * ctx->esize));
            xsrc = op->xall;
            n_loc = 0x7fffffff;
        } else {
            const size_t es = ctx->esize;
            const int up = ctx->rank + 1 < ctx->nranks ? ctx->rank + 1 : -1;
            const int dn = ctx->rank > 0 ? ctx->rank - 1 : -1;
            const char* xp = (const char*)x.ptr;
            char* hl = (char*)op->halo;
            char* hh = hl + (size_t)op->halo_lo * es;
            // one grouped exchange: my last send_hi entries go up (rank+1's lo halo), my
            // first send_lo entries go down (rank-1's hi halo)
            B2K_TRY(b2k_nccl_halo_exchange(ctx, up, dn,
                                           xp + (size_t)(x.n - op->send_hi) * es, op->send_hi * es,
                                           hl, op->halo_lo * es,
                                           xp, op->send_lo * es,
                                           hh, op->halo_hi * es));
        }
    } else if (x.n == op->n_cols) {
        n_loc = 0x7fffffff;
    }
    double* out = (dotv || fz.dot_self) ? dot_out : nullptr;
    if (op->kind == 2) {
        StencilApply sa;
        sa.nx = op->snx; sa.ny = op->sny; sa.nz = op->snz; sa.row0 = op->srow0;
        sa.n_rows = op->n_rows; sa.n_loc = x.n; sa.halo_lo = op->halo_lo;
        for (int i = 0; i < 7; ++i) sa.c[i] = op->sc[i];
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((op->n_rows + 255) / 256, (int64_t)ctx->num_sms * 8));
        const int pr2 = b2k_prof_begin(ctx, 0, 2.0 * ctx->esize * op->n_rows);
        if (ctx->dtype == B2K_F64)
            k_stencil_apply<double><<<grid, 256, 0, ctx->stream>>>(sa, (const double*)xsrc, (const double*)halo, (double*)y.ptr,
                                                                   a0, a1, shifted ? 1 : 0, dotv ? (const double*)dotv->ptr : nullptr,
                                                                   op->part, ctx->d_sync, out, fz, ps);
        else
            k_stencil_apply<float><<<grid, 256, 0, ctx->stream>>>(sa, (const float*)xsrc, (const float*)halo, (float*)y.ptr,
                                                                  (float)a0, (float)a1, shifted ? 1 : 0,
                                                                  dotv ? (const float*)dotv->ptr : nullptr, op->part,
                                                                  ctx->d_sync, out, fz, ps);
        b2k_prof_end(ctx, pr2);
        B2K_LAUNCH_CHECK(ctx);
        return B2K_OK;
    }
    // algorithmic bytes: matrix + x + y, plus the normalised copy of x a chained Lanczos step stores (fz.vout)
    const int pr = b2k_prof_begin(ctx, 0, (double)op->nnz * (ctx->esize + 4) + 4.0 * (op->n_rows + 1) +
                                              (fz.vout ? 3.0 : 2.0) * ctx->esize * op->n_rows);
    if (g_spmv_pipe) {
        const int per_sm = g_spmv_variant == 1 ? 4 : 3;
        const int grid = std::min(op->nblk, per_sm * ctx->num_sms);
#define LAUNCH_V(T, NS, MB)                                                                    \
    k_spmv_pipe<T, NS, MB><<<grid, SPP_THREADS, SppLayout<T, NS>::SMEM, ctx->stream>>>(        \
        op->rowptr, op->colidx, (const T*)op->vals, (const T*)xsrc, (const T*)halo, n_loc,     \
        (T*)y.ptr, op->rowblk, op->pblk, op->nblk, (T)a0, (T)a1, shifted ? 1 : 0,              \
        (const T*)x.ptr, dotv ? (const T*)dotv->ptr : nullptr, op->part, ctx->d_sync, out, fz, ps)
        if (g_spmv_variant == 1) {
            if (ctx->dtype == B2K_F64) LAUNCH_V(double, 2, 4);
            else LAUNCH_V(float, 2, 4);
        } else {
            if (ctx->dtype == B2K_F64) LAUNCH_V(double, 3, 3);
            else LAUNCH_V(float, 3, 3);
        }
#undef LAUNCH_V
    } else {
#define LAUNCH(T)                                                                              \
    k_spmv_stream<T><<<op->nblk, SP_BT, 0, ctx->stream>>>(                                     \
        op->rowptr, op->colidx, (const T*)op->vals, (const T*)xsrc, (const T*)halo, n_loc,     \
        (T*)y.ptr, op->rowblk, (T)a0, (T)a1, shifted ? 1 : 0, (const T*)x.ptr,                 \
        dotv ? (const T*)dotv->ptr : nullptr, op->part, ctx->d_sync, out, fz, ps)
        if (ctx->dtype == B2K_F64) LAUNCH(double);
        else LAUNCH(float);
#undef LAUNCH
    }
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_op_apply(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y) {
    if (!ctx || !op) return B2K_EINVAL;
    VecRef rx, ry;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    return b2k_enqueue_apply(ctx, op, rx, ry, 0.0, 1.0, false, nullptr, -1);
}

extern "C" int32_t b2k_op_apply_shifted(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y,
                                        double a0, double a1) {
    if (!ctx || !op) return B2K_EINVAL;
    VecRef rx, ry;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    // apply.jl:6: the add!! only happens if α₀ != 0 || α₁ != 1
    const bool shifted = (a0 != 0.0) || (a1 != 1.0);
    if (op->kind == 1 && shifted) {
        B2K_TRY(b2k_enqueue_apply(ctx, op, rx, ry, 0.0, 1.0, false, nullptr, -1));
        return b2k_vec_axpby(ctx, y, x, a0, a1);
    }
    return b2k_enqueue_apply(ctx, op, rx, ry, a0, a1, shifted, nullptr, -1);
}

extern "C" int32_t b2k_op_apply_dot(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y, b2k_vec v,
                                    double* dot) {
    if (!ctx || !op || !dot) return B2K_EINVAL;
    VecRef rx, ry, rv;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    B2K_TRY(b2k_resolve(ctx, v, &rv));
    if (rv.n != ry.n) return b2k_fail(ctx, B2K_EDIM, "apply_dot: v/y length mismatch");
    if (op->kind == 1) {
        B2K_TRY(b2k_enqueue_apply(ctx, op, rx, ry, 0.0, 1.0, false, nullptr, -1));
        return b2k_vec_inner(ctx, v, y, dot);
    }
    B2K_TRY(b2k_enqueue_apply(ctx, op, rx, ry, 0.0, 1.0, false, &rv, 0));
    B2K_TRY(b2k_fetch_results(ctx, 1, ry.sharded));
    *dot = ctx->h_res[0];
    return B2K_OK;
}

extern "C" int32_t b2k_op_apply_adjoint(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y) {
    if (!ctx || !op) return B2K_EINVAL;
    VecRef rx, ry;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    if (op->kind != 1)
        return b2k_fail(ctx, B2K_ENOTSUP,
                        "apply_adjoint on a CSR operator: create the operator from the transposed "
                        "matrix (b2k_op_create_csc of A' / CSR of A') instead");
    if (rx.n != op->n_rows || ry.n != op->n_cols)
        return b2k_fail(ctx, B2K_EDIM, "dense adjoint: x has %lld (want %lld), y has %lld (want %lld)",
                        (long long)rx.n, (long long)op->n_rows, (long long)ry.n, (long long)op->n_cols);
    return b2k_panel_project_dev(ctx, op->A, op->ld, op->n_rows, (int32_t)op->n_cols, rx, ry.ptr,
                                 rx.sharded);
}

// ------------------------------------------------------------------------------------------------
// One pass over a dense A for BOTH products of a Golub-Kahan-Lanczos step (SURVEY §8f-4, the flagged
// `onepass` mode of the GKL mirror; the reference's step reads A twice: gkl.jl:308-323 `apply_adjoint` then
// `apply_normal`).  While y = A x is formed, z = A'(A x) is accumulated from the same resident row tile; the
// host recovers A'u_{k+1} = (z - sum_j c_j A'u_j) / beta_k from it (factorizations/gkl.py) without a second
// pass.  The reduction over rows of y = A x is LOCAL to a row tile, so no grid-wide barrier is needed:
//
//   tile   = 32 rows x n columns of the column-major A (n <= 1700 Float32 / 850 Float64), parked in shared
//            memory with a column stride of 33 words: conflict-free both for lane <-> row (the tile stores)
//            and for lane <-> column (phase 2);
//   load   : every thread issues 8 independent 16-byte loads (4 Float32 / 2 Float64 consecutive rows of one
//            column) per batch; its partial y for those rows is accumulated straight from the registers;
//   phase 1: partial y summed over the threads that hold the same rows (shuffles, then the 8 warps in fixed
//            order) -> y[32], written to global memory;
//   phase 2: thread <-> column: z_c += sum_rows tile[c][row] * y[row]  (T per tile, double across tiles);
//   end    : per-CTA partial z (double) -> k_onepass_reduce sums the CTAs in fixed order (deterministic).
//
// Rows [m, ld) of A are zero (alloc_dense memsets, both fills write rows < m only) and ld is a multiple of 32,
// so every tile is loaded without row guards.  Algorithmic traffic: sizeof(T) * (m n + m + n) bytes per call —
// half of the two-pass step.  3 CTAs per SM for n = 512 Float32 (71 KB of shared memory each): the loads of one
// CTA overlap the phases of the others; no asynchronous copies, no spin waits.
namespace {

#include "onepass_kernels.cuh"

int g_onepass_variant = 0;       // 0: 32-row tiles, 3 CTAs per SM (A); 1: 64-row tiles, register-pipelined (B, Float32 n <= 512)

// per-CTA partials -> z (and the sum over the ranks of a row-sharded context)
template <typename T>
int32_t onepass_finish(b2k_ctx* ctx, b2k_op* op, int grid, int n, const VecRef& y, const VecRef& z) {
    const bool reduce_ranks = ctx->nranks > 1 && y.sharded;
    k_onepass_reduce<T><<<(n + 31) / 32, 256, 0, ctx->stream>>>(op->part, grid, n, ctx->d_res,
                                                                reduce_ranks ? nullptr : (T*)z.ptr);
    B2K_LAUNCH_CHECK(ctx);
    if (reduce_ranks) {
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res, n, 1));
        k_onepass_store<T><<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_res, (T*)z.ptr, n);
        B2K_LAUNCH_CHECK(ctx);
    }
    return B2K_OK;
}

int32_t onepass_part(b2k_ctx* ctx, b2k_op* op, size_t need) {
    if (op->part_bytes < need) {
        if (op->part) B2K_DFREE(op->part);
        op->part = nullptr;
        op->part_bytes = 0;
        B2K_CUDA(ctx, B2K_DMALLOC(&op->part, need));
        op->part_bytes = need;
    }
    return B2K_OK;
}

int32_t onepass_w(b2k_ctx* ctx, b2k_op* op, const VecRef& x, const VecRef& y, const VecRef& z) {
    const int n = (int)op->n_cols;
    const size_t smem = ((size_t)n * OPW_PAD + n + (OPW_T / 32) * OPW_ROWS + OPW_ROWS) * sizeof(float);
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_dense_onepass_w, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t ntiles = (op->ld + OPW_ROWS - 1) / OPW_ROWS;
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)ctx->num_sms);
    B2K_TRY(onepass_part(ctx, op, (size_t)grid * n * sizeof(double)));
    const int pr = b2k_prof_begin(ctx, 8, 4.0 * ((double)op->n_rows * n + (double)op->n_rows + n));
    k_dense_onepass_w<<<grid, OPW_T, smem, ctx->stream>>>((const float*)op->A, op->ld, op->n_rows, n, (const float*)x.ptr,
                                                         (float*)y.ptr, op->part, ntiles);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    return onepass_finish<float>(ctx, op, grid, n, y, z);
}

template <typename T>
int32_t onepass_t(b2k_ctx* ctx, b2k_op* op, const VecRef& x, const VecRef& y, const VecRef& z) {
    const int n = (int)op->n_cols;
    const size_t smem = ((size_t)n * OP_PAD + n + (OP_T / 32) * OP_ROWS + OP_ROWS) * sizeof(T);
    if (smem > 227u * 1024u)
        return b2k_fail(ctx, B2K_ENOTSUP, "one-pass dense step: a 32 x %d tile needs %zu bytes of shared memory", n, smem);
    if (sizeof(T) == 4 && g_onepass_variant == 1 && n <= OPW_LD * (OPW_T / (OPW_ROWS / 4)))
        return onepass_w(ctx, op, x, y, z);
    void (*kern)(const T*, int64_t, int64_t, int32_t, const T*, T*, double*, int64_t) =
        n <= OP_T ? k_dense_onepass<T, 1> : n <= 2 * OP_T ? k_dense_onepass<T, 2> :
        n <= 4 * OP_T ? k_dense_onepass<T, 4> : k_dense_onepass<T, OP_ZMAX>;
    B2K_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    B2K_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, OP_T, smem));
    if (occ < 1) return b2k_fail(ctx, B2K_ENOTSUP, "one-pass dense step: a %d-column tile does not fit an SM", n);
    const int64_t ntiles = op->ld / OP_ROWS;
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)occ * ctx->num_sms);
    B2K_TRY(onepass_part(ctx, op, (size_t)grid * n * sizeof(double)));
    const int pr = b2k_prof_begin(ctx, 8, (double)sizeof(T) * ((double)op->n_rows * n + (double)op->n_rows + n));
    kern<<<grid, OP_T, smem, ctx->stream>>>((const T*)op->A, op->ld, op->n_rows, n, (const T*)x.ptr,
                                                           (T*)y.ptr, op->part, ntiles);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    return onepass_finish<T>(ctx, op, grid, n, y, z);
}

}  // namespace

// y = A x and z = A'(A x) from ONE pass over the dense A (see k_dense_onepass).  x, z: length n_cols (the
// operator's input space); y: length n_rows (space 0).  Dense operators only; everything else is B2K_ENOTSUP.
extern "C" int32_t b2k_op_apply_normal_gram(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y, b2k_vec z) {
    if (!ctx || !op) return B2K_EINVAL;
    VecRef rx, ry, rz;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    B2K_TRY(b2k_resolve(ctx, z, &rz));
    if (op->kind != 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "apply_normal_gram: dense operators only (the one-pass GKL step)");
    if (rx.n != op->n_cols || rz.n != op->n_cols || ry.n != op->n_rows)
        return b2k_fail(ctx, B2K_EDIM, "apply_normal_gram: x has %lld, z has %lld (want %lld), y has %lld (want %lld)",
                        (long long)rx.n, (long long)rz.n, (long long)op->n_cols, (long long)ry.n, (long long)op->n_rows);
    if (rx.ptr == rz.ptr || rx.ptr == ry.ptr || ry.ptr == rz.ptr)
        return b2k_fail(ctx, B2K_EINVAL, "apply_normal_gram: x, y and z must be three different vectors");
    if (op->n_cols > OP_ZMAX * OP_T || op->n_cols > B2K_RES_DOUBLES)
        return b2k_fail(ctx, B2K_ENOTSUP, "apply_normal_gram: more than %d columns", OP_ZMAX * OP_T);
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    b2k_op* mop = const_cast<b2k_op*>(op);          // the per-CTA partial buffer is allocated on first use
    if (ctx->dtype == B2K_F64) return onepass_t<double>(ctx, mop, rx, ry, rz);
    return onepass_t<float>(ctx, mop, rx, ry, rz);
}

// A/B switch of the one-pass dense step (tools / tests / bench.py's c4o child): 0 = variant A, 1 = variant B
extern "C" int32_t b2k_debug_set_onepass_variant(int32_t v) {
    if (v < 0 || v > 1) return B2K_EINVAL;
    g_onepass_variant = v;
    return B2K_OK;
}

// apply(A, X::Block) — blocklanczos.jl:38: Y[i] = A X[i] for the p vectors of a block.  Single-GPU CSR operators
// read the matrix once per 8 vectors (k_spmm_pipe); everything else is the loop of single applies the
// reference runs.  Same bits either way.
extern "C" int32_t b2k_op_apply_block(b2k_ctx* ctx, const b2k_op* op, const b2k_vec* X, const b2k_vec* Y, int32_t p) {
    if (!ctx || !op || !X || !Y || p < 1) return B2K_EINVAL;
    for (int i = 0; i < p; ++i)
        for (int j = 0; j < p; ++j)
            if (X[i] == Y[j]) return b2k_fail(ctx, B2K_EINVAL, "apply_block: Y[%d] aliases X[%d]", j, i);
    bool fast = op->kind == 0 && ctx->nranks == 1 && g_spmv_pipe && p > 1 &&   // (stencil: the loop of applies)
                b2k_block_kernels_enabled();
    int32_t sx = -1, sy = -1;
    std::vector<int32_t> ix, iy;
    B2K_TRY(b2k_resolve_cols(ctx, X, p, &sx, &ix));
    B2K_TRY(b2k_resolve_cols(ctx, Y, p, &sy, &iy));
    fast = fast && sx == sy && ctx->spaces[sx].n == op->n_rows && op->n_rows == op->n_cols;
    if (!fast) {
        for (int i = 0; i < p; ++i) B2K_TRY(b2k_op_apply(ctx, op, X[i], Y[i]));
        return B2K_OK;
    }
    const B2kSpace& sp = ctx->spaces[sx];
    const int grid = std::min(op->nblk, 3 * ctx->num_sms);
    for (int i0 = 0; i0 < p; i0 += SPM_PMAX) {
        const int np = std::min(SPM_PMAX, p - i0);
        SpmmCols cols;
        for (int i = 0; i < SPM_PMAX; ++i) { cols.x[i] = ix[i0 + (i < np ? i : 0)]; cols.y[i] = iy[i0 + (i < np ? i : 0)]; }
        const int pr = b2k_prof_begin(ctx, 7, (double)op->nnz * (ctx->esize + 4) + 4.0 * (op->n_rows + 1) +
                                                  2.0 * np * ctx->esize * op->n_rows);
        if (ctx->dtype == B2K_F64)
            k_spmm_pipe<double><<<grid, SPP_THREADS, SpmLayout<double>::SMEM, ctx->stream>>>(
                op->rowptr, op->colidx, (const double*)op->vals, (double*)sp.base, sp.ld, cols, np, op->rowblk,
                op->pblk, op->nblk);
        else
            k_spmm_pipe<float><<<grid, SPP_THREADS, SpmLayout<float>::SMEM, ctx->stream>>>(
                op->rowptr, op->colidx, (const float*)op->vals, (float*)sp.base, sp.ld, cols, np, op->rowblk,
                op->pblk, op->nblk);
        b2k_prof_end(ctx, pr);
        B2K_LAUNCH_CHECK(ctx);
    }
    return B2K_OK;
}
