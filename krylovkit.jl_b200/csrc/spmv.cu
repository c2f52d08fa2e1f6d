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
    // compact copy of the CSR stream read by k_spmv_compact (build_compact; single-GPU CSR operators).  Each part is
    // allocated only when it compressed losslessly; k_spmv_compact reads the plain array in place of a missing one.
    // crp is null when neither values nor columns compressed: the operator then has no compact view.
    float*    cvals = nullptr;    // Float64 contexts: every value as float (each one round-trips exactly)
    int16_t*  ccol = nullptr;     // colidx - rowblk[tile] for every nonzero of every tile of <= SP_NNZ nonzeros
    uint16_t* crp = nullptr;      // low 16 bits of rowptr
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
            if (shifted) s = fma(a0, xs[r] * sc, a1 * s);      // the shift acts on the normalised operand
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
            if (shifted) s = fma(a0, xs[r0] * sc, a1 * s);
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
        finish_sums<1>({block_sum((double)dacc, red)}, part, ticket, red, &last, SP_BT, [&](int, double tot) {
            *out = tot;
            if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
        });
    }
}


// ---------------------------------------------------------------------------------------
// Pipelined CSR-stream SpMV (the default): persistent CTAs (3 per SM), a producer warp
// streams each row block's nonzeros (vals, colidx) and its rowptr segment into a 3-stage
// shared-memory ring with 1-D TMA bulk copies (UBLKCP) signalled on mbarriers; the 8
// consumer warps gather x, multiply in place, and sum rows out of shared memory while the
// next blocks are already in flight.  Same arithmetic (products rounded, summed in CSR
// order) as k_spmv_stream, which remains as the reference implementation for tests.
constexpr int SPP_RMAX = 1024;            // rowptr entries staged per block
constexpr int SPP_TV = SP_NNZ + 8;        // staged nonzeros (block + alignment slack)
constexpr int SPP_CONS = 256;
constexpr int SPP_THREADS = SPP_CONS + 32;

// A tile's bulk copies into ring stage st, completing on the stage's full barrier.
struct TileCopy {
    uint32_t st, bar;
    int lane;
    bool hints;                  // L2 evict_first: the CSR arrays are read once per apply
    // lane 0 announces the tile's bytes before any of its copies is issued
    __device__ __forceinline__ void expect(uint32_t bytes) const {
        if (lane == 0) mbar_expect_tx(bar, bytes);
        __syncwarp();
    }
    // lane l copies `bytes` bytes from src to stage offset off
    __device__ __forceinline__ void operator()(int l, int off, const void* src, uint32_t bytes) const {
        if (lane != l || bytes == 0) return;
        if (hints) bulk_g2s_hint(st + off, src, bytes, bar, l2_policy_evict_first());
        else bulk_g2s(st + off, src, bytes, bar);
    }
};

// The TMA tile ring of the warp-specialised CSR kernels (k_spmv_pipe, k_spmv_compact, k_spmv_pencil, k_spmm_pipe).
// Shared memory: NSTG stages of STAGE bytes, EXTRA bytes of the kernel's own, the stages' full and empty mbarriers,
// then the consumers' reduction scratch red (32 doubles) and flag.  CTA b takes tiles b, b + G, ...  Per tile the
// producer warp waits for the stage to be empty and issues the tile's copies; a tile of more than SP_NNZ nonzeros (one
// long row) copies nothing, lane 0 arrives instead and the consumers read global memory.  The consumers wait for the
// stage to be full, read it, and release it with one arrival per warp.
template <int NSTG_, int STAGE_, int EXTRA = 0>
struct TileRing {
    static constexpr int NSTG = NSTG_, STAGE = STAGE_;
    static constexpr int OFF_EXTRA = NSTG * STAGE;
    static constexpr int OFF_BAR = OFF_EXTRA + EXTRA;
    static constexpr int OFF_RED = OFF_BAR + 2 * NSTG * 8 + 16;
    static constexpr int SMEM = OFF_RED + 32 * 8 + 16;

    uint8_t* smem;
    const int32_t* rowblk;
    const int32_t* pblk;
    int nblk;
    uint32_t s = 0, ph = 0;              // consumers: the current tile's stage and its phase parity
    int4 dn = make_int4(0, 0, 0, 0);     // consumers: (r0, r1, p0, p1) of the next tile

    __device__ __forceinline__ uint8_t* stage(uint32_t i) const { return smem + i * STAGE; }
    __device__ __forceinline__ uint32_t full(uint32_t i) const { return smem_u32(smem + OFF_BAR) + 8 * i; }
    __device__ __forceinline__ uint32_t empty(uint32_t i) const { return full(NSTG + i); }
    __device__ __forceinline__ double* red() const { return reinterpret_cast<double*>(smem + OFF_RED); }
    __device__ __forceinline__ int* flag() const { return reinterpret_cast<int*>(smem + OFF_RED + 32 * 8); }
    __device__ __forceinline__ int4 desc(int t) const {
        return make_int4(rowblk[t], rowblk[t + 1], pblk[t], pblk[t + 1]);
    }

    // every thread of the CTA
    __device__ __forceinline__ void init() const {
        if (threadIdx.x == 0) {
            for (int i = 0; i < NSTG; ++i) {
                mbar_init(full(i), 1);
                mbar_init(empty(i), SPP_CONS / 32);
            }
            fence_mbar_init();
        }
        __syncthreads();
    }

    // The producer warp: issue(copy, r0, r1, p0, p1) stages a tile of <= SP_NNZ nonzeros through copy.expect and copy.
    template <typename Issue>
    __device__ __forceinline__ void produce(bool hints, Issue issue) const {
        const int lane = threadIdx.x & 31;
        uint32_t ps = 0, pph = 0;
        int tile = blockIdx.x;
        int d = 0;   // lanes 0..3 hold r0, r1, p0, p1 of the current tile
        if (tile < nblk && lane < 4) d = (lane < 2) ? rowblk[tile + lane] : pblk[tile + lane - 2];
        for (; tile < nblk; tile += gridDim.x) {
            const int r0 = __shfl_sync(0xffffffffu, d, 0), r1 = __shfl_sync(0xffffffffu, d, 1);
            const int p0 = __shfl_sync(0xffffffffu, d, 2), p1 = __shfl_sync(0xffffffffu, d, 3);
            const int nt = tile + gridDim.x;      // prefetch the next descriptor before blocking
            if (nt < nblk && lane < 4) d = (lane < 2) ? rowblk[nt + lane] : pblk[nt + lane - 2];
            mbar_wait(empty(ps), pph ^ 1);
            if (p1 - p0 <= SP_NNZ) issue(TileCopy{smem_u32(stage(ps)), full(ps), lane, hints}, r0, r1, p0, p1);
            else if (lane == 0) mbar_arrive(full(ps));
            if (++ps == NSTG) { ps = 0; pph ^= 1; }
        }
    }

    // The consumers: start() before the tile loop, then per tile next(tile) gives its descriptor (and loads the next
    // one's into dn), wait() waits for its stage, release() hands the stage back and moves to the next.
    __device__ __forceinline__ void start() {
        if ((int)blockIdx.x < nblk) dn = desc(blockIdx.x);
    }
    __device__ __forceinline__ int4 next(int tile) {
        const int4 d = dn;
        const int nt = tile + gridDim.x;
        if (nt < nblk) dn = desc(nt);
        return d;
    }
    __device__ __forceinline__ void wait() const { mbar_wait(full(s), ph); }
    // the next tile's stage, and a wait for it while the current one is still held
    __device__ __forceinline__ uint32_t s_next() const { return s + 1 == NSTG ? 0 : s + 1; }
    __device__ __forceinline__ void wait_next() const { mbar_wait(full(s_next()), s + 1 == NSTG ? ph ^ 1 : ph); }
    // wrote: the consumers wrote the stage; their generic-proxy writes must precede its reuse by the TMA unit
    __device__ __forceinline__ void release(bool wrote = true) {
        if (wrote) fence_proxy_async();
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(empty(s));
        if (++s == NSTG) { s = 0; ph ^= 1; }
    }
};

// A ring stage of k_spmv_pipe and k_spmm_pipe (NV = 1) and k_spmv_pencil (NV = 2: A's values, then B's): NV value
// arrays, the columns and the row pointers of a tile, each with room for the 16-byte alignment of its copy.
template <typename T, int NV> struct CsrStage {
    static constexpr int VAL_BYTES = SPP_TV * (int)sizeof(T);
    static constexpr int OFF_COL = NV * VAL_BYTES;
    static constexpr int OFF_RP = OFF_COL + SPP_TV * 4;
    static constexpr int BYTES = OFF_RP + (SPP_RMAX + 8) * 4;
};
template <typename T, int NSTG, int EXTRA = 0> using SppRing = TileRing<NSTG, CsrStage<T, 1>::BYTES, EXTRA>;

// A CsrStage's copies of tile (r0, r1, p0, p1): lane v copies value array v, lane NV the columns and lane NV + 1 the
// row pointers (none for a tile of more than SPP_RMAX rows, whose consumers read rowptr from global memory).
template <typename T, int NV>
__device__ __forceinline__ void copy_csr_tile(const TileCopy& c, const T* const (&vals)[NV], const int32_t* colidx,
                                              const int32_t* rowptr, int r0, int r1, int p0, int p1) {
    using SG = CsrStage<T, NV>;
    const int p0a = p0 & ~3, cnt = ((p1 + 3) & ~3) - p0a;
    const int r0a = r0 & ~3;
    const int rcnt = (r1 - r0 <= SPP_RMAX) ? (((r1 + 1 + 3) & ~3) - r0a) : 0;
    const uint32_t vb = (uint32_t)cnt * (uint32_t)sizeof(T), cb = (uint32_t)cnt * 4u, rb = (uint32_t)rcnt * 4u;
    c.expect(NV * vb + cb + rb);
#pragma unroll
    for (int v = 0; v < NV; ++v) c(v, v * SG::VAL_BYTES, vals[v] + p0a, vb);
    c(NV, SG::OFF_COL, colidx + p0a, cb);
    c(NV + 1, SG::OFF_RP, rowptr + r0a, rb);
}

// The fused dots of the TMA kernels, summed by their SPP_CONS consumer threads (named barrier 1): per sum k, each
// warp's butterfly of its threads' v[k] and the warps added in order from 0.0 give the CTA partial part[k G + b]; the
// last CTA to take a ticket has thread t add partials t, t + SPP_CONS, ... from 0.0, reduces those the same way, and
// its thread 0 calls fin(k, total_k) for k = 0 .. NRED-1.  red and flag: the ring's scratch.
template <int NRED, typename Fin>
__device__ __forceinline__ void consumer_sums(const double (&v)[NRED], double* __restrict__ part,
                                              unsigned* __restrict__ ticket, double* red, int* flag, Fin fin) {
    constexpr int NW = SPP_CONS / 32;
    static_assert(NRED * NW <= 32, "red holds 32 doubles");
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    // thread 0 gets each x[k] summed over the consumers
    auto cta_sums = [&](double (&x)[NRED]) {
#pragma unroll
        for (int k = 0; k < NRED; ++k) x[k] = warp_sum(x[k]);
        named_bar_sync(1, SPP_CONS);                    // red's last reader is done with it
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NRED; ++k) red[k * NW + w] = x[k];
        }
        named_bar_sync(1, SPP_CONS);
        if (tid == 0) {
#pragma unroll
            for (int k = 0; k < NRED; ++k) {
                double tot = 0.0;
                for (int i = 0; i < NW; ++i) tot += red[k * NW + i];
                x[k] = tot;
            }
        }
    };
    double s[NRED];
#pragma unroll
    for (int k = 0; k < NRED; ++k) s[k] = v[k];
    cta_sums(s);
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < NRED; ++k) part[(size_t)k * gridDim.x + blockIdx.x] = s[k];
        __threadfence();
        const unsigned t = atomicInc(ticket, gridDim.x - 1);
        *flag = (t == gridDim.x - 1);
    }
    named_bar_sync(1, SPP_CONS);
    if (!*flag) return;
    __threadfence();
    const volatile double* pv = part;
#pragma unroll
    for (int k = 0; k < NRED; ++k) s[k] = 0.0;
    for (int g = tid; g < (int)gridDim.x; g += SPP_CONS) {
#pragma unroll
        for (int k = 0; k < NRED; ++k) s[k] += pv[(size_t)k * gridDim.x + g];
    }
    cta_sums(s);
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < NRED; ++k) fin(k, s[k]);
    }
}

// The GKL epilogue's norm (SpmvFuse::nrm_out): the CTA-ordered sum of the threads' y_r^2 chains, as the fused dot; the
// last CTA stores {sqrt(s), 1/sqrt(s), s} and raises the chain's stop flag when the norm is not finite.
__device__ __forceinline__ void gkl_norm_sums(double v, double* __restrict__ part, unsigned* __restrict__ ticket,
                                              double* red, int* flag, const SpmvFuse& fz) {
    consumer_sums<1>({v}, part, ticket, red, flag, [&](int, double tot) {
        const double a = sqrt(tot);
        fz.nrm_out[0] = a;
        fz.nrm_out[1] = 1.0 / a;
        fz.nrm_out[2] = tot;
        if (fz.stop && !isfinite(a)) *const_cast<int*>(fz.stop) = 1;
    });
}

__global__ void k_pblk(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ rowblk, int count,
                       int32_t* __restrict__ pblk) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < count) pblk[b] = rowptr[rowblk[b]];
}

// Row epilogue of the single-operator TMA kernels (k_spmv_pipe, k_spmv_compact): y_r = a0 xs_r + a1 (A x)_r with the
// shift acting on the normalised operand, vout_r = the normalised x_r, and the dot chain dacc = fma(dv_r, y_r - dsc
// dsub_r, dacc) over the thread's rows, dv = dotv or the normalised x (fz.dot_self).  load(r) issues a row's global
// loads, before its sum so that they overlap it; row(r, loads, sum) finishes it.
// GK (the instances b2k_gkl_expand_many launches): after the sum, p_r = rn(pvec_r * pscale) is stored to pout,
// y_r = fma(-acoef, p_r, sum) is stored instead of the sum, and nacc = fma(y_r, y_r, nacc) when nrm_out is set
// (SpmvFuse).  Off, none of it is compiled.
template <typename T, bool GK = false>
struct RowEpilogue {
    struct Loads { T dv, xself, xsr, dsv, pv; };
    const SpmvFuse fz;
    const T* x;
    T* y;
    const T* xs;
    const T* dotv;
    T a0, a1;
    int shifted;
    bool scaled = fz.xscale != nullptr;
    T sc = scaled ? (T)(*fz.xscale) : (T)1;
    T* vout = reinterpret_cast<T*>(fz.vout);
    bool self = (vout != nullptr) || fz.dot_self;
    bool want_dot = (dotv != nullptr) || fz.dot_self;
    uint64_t pol_last = fz.l2_hints ? l2_policy_evict_last() : 0;
    const T* dsub = reinterpret_cast<const T*>(fz.dot_sub_vec);
    T dsc = dsub ? (T)(*fz.dot_sub_scale) : (T)0;
    T dacc = (T)0;
    const T* pvec = GK ? reinterpret_cast<const T*>(fz.pvec) : nullptr;
    T* pout = GK ? reinterpret_cast<T*>(fz.pout) : nullptr;
    bool pscaled = GK && fz.pscale != nullptr;
    T psc = pscaled ? (T)(*fz.pscale) : (T)1;
    T nac = GK ? -(T)(*fz.acoef) : (T)0;
    bool want_nrm = GK && fz.nrm_out != nullptr;

    __device__ __forceinline__ Loads load(int r) const {
        return {(dotv && !fz.dot_self) ? __ldg(dotv + r) : (T)0, self ? __ldg(x + r) : (T)0,
                shifted ? __ldg(xs + r) : (T)0, dsub ? __ldg(dsub + r) : (T)0, GK ? pvec[r] : (T)0};
    }
    // the GKL step's finish of row r: the previous vector normalised and stored, the axpy, the norm chain
    __device__ __forceinline__ T gkl_row(int r, T pv, T sum) {
        const T p = pscaled ? mul_rn<T>(pv, psc) : pv;
        if (pout) pout[r] = p;
        sum = fma(nac, p, sum);
        if (want_nrm) dacc = fma(sum, sum, dacc);
        return sum;
    }
    __device__ __forceinline__ void row(int r, const Loads& l, T sum) {
        if constexpr (GK) {
            y[r] = gkl_row(r, l.pv, sum);
            return;
        }
        if (shifted) sum = fma(a0, l.xsr * sc, a1 * sum);      // the shift acts on the normalised operand
        if (fz.l2_hints) st_hint(y + r, sum, pol_last);
        else y[r] = sum;
        T dv = l.dv;
        if (self) {
            const T vn = l.xself * sc;
            if (vout) vout[r] = vn;
            if (fz.dot_self) dv = vn;
        }
        dacc = fma(dv, dsub ? fma(-dsc, l.dsv, sum) : sum, dacc);
    }
    // A row of more than SP_NNZ nonzeros, the CTA's only one: a double sum of the rounded products, thread i taking
    // nonzeros i, i + SPP_CONS, ..., then warp butterflies and the warps in order, rounded to T once.  xg(c) = x_c.
    template <typename G>
    __device__ __forceinline__ void long_row(int r0, const T* vals, const int32_t* colidx, int p0, int nnzb,
                                             double* red, G xg) {
        const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
        double acc = 0.0;
        for (int i = tid; i < nnzb; i += SPP_CONS) {
            T xv = xg(colidx[p0 + i]);
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
            if constexpr (GK) {
                y[r0] = gkl_row(r0, pvec[r0], sum);
            } else {
                if (shifted) sum = fma(a0, xs[r0] * sc, a1 * sum);
                y[r0] = sum;
                T dv = (dotv && !fz.dot_self) ? dotv[r0] : (T)0;
                if (self) {
                    const T vn = __ldg(x + r0) * sc;
                    if (vout) vout[r0] = vn;
                    if (fz.dot_self) dv = vn;
                }
                if (want_dot) dacc = fma(dv, dsub ? fma(-dsc, dsub[r0], sum) : sum, dacc);
            }
        }
        named_bar_sync(1, SPP_CONS);
    }
};

// NSTG ring stages, MINB CTAs per SM (variants: (3, 3); (2, 4): fewer stages, more resident warps to hide the
// latency of the x gather)
template <typename T, int NSTG, int MINB, bool GK = false>
__global__ void __launch_bounds__(SPP_THREADS, MINB)
k_spmv_pipe(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
            const T* __restrict__ vals, const T* __restrict__ x, const T* __restrict__ halo,
            int32_t n_loc, T* __restrict__ y, const int32_t* __restrict__ rowblk,
            const int32_t* __restrict__ pblk, int nblk, T a0, T a1, int shifted,
            const T* __restrict__ xs, const T* __restrict__ dotv, double* __restrict__ part,
            unsigned* __restrict__ ticket, double* __restrict__ out, const SpmvFuse fz,
            const __grid_constant__ PeerStep ps) {
    using SG = CsrStage<T, 1>;
    extern __shared__ __align__(128) uint8_t smem[];
    if (fz.stop && *reinterpret_cast<const volatile int*>(fz.stop)) return;
    SppRing<T, NSTG> ring{smem, rowblk, pblk, nblk};
    ring.init();
    if (threadIdx.x >= SPP_CONS) {
        ring.produce(fz.l2_hints, [&](const TileCopy& c, int r0, int r1, int p0, int p1) {
            copy_csr_tile<T, 1>(c, {vals}, colidx, rowptr, r0, r1, p0, p1);
        });
        return;
    }
    // ---------------------------------- consumers ----------------------------------
    const int tid = threadIdx.x;
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
    RowEpilogue<T, GK> ep{fz, x, y, xs, dotv, a0, a1, shifted};
    ring.start();
    for (int tile = blockIdx.x; tile < nblk; tile += gridDim.x) {
        const int4 d = ring.next(tile);
        const int r0 = d.x, r1 = d.y, p0 = d.z, p1 = d.w;
        const int nnzb = p1 - p0, nrows = r1 - r0;
        ring.wait();
        if (nnzb <= SP_NNZ) {
            uint8_t* const st = ring.stage(ring.s);
            T* vs = reinterpret_cast<T*>(st);
            const int32_t* cs = reinterpret_cast<const int32_t*>(st + SG::OFF_COL);
            const int32_t* rs = reinterpret_cast<const int32_t*>(st + SG::OFF_RP);
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
            if (ep.scaled) {
#pragma unroll
                for (int u = 0; u < U; ++u) xv[u] *= ep.sc;      // v_j = r_j * (1/β), rounded like scale!!
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) vs[off + i] *= xv[u];
            }
            named_bar_sync(1, SPP_CONS);
            const bool rp_staged = nrows <= SPP_RMAX;
            for (int r = r0 + tid; r < r1; r += SPP_CONS) {
                const auto ld = ep.load(r);
                int a, b;
                if (rp_staged) { a = rs[r - r0a]; b = rs[r + 1 - r0a]; }
                else { a = rowptr[r]; b = rowptr[r + 1]; }
                a -= p0a; b -= p0a;
                T sum = (T)0;
                for (int p = a; p < b; ++p) sum += vs[p];
                ep.row(r, ld, sum);
            }
        } else {
            ep.long_row(r0, vals, colidx, p0, nnzb, ring.red(),
                        [&](int32_t cc) { return (cc < n_loc) ? __ldg(x + cc) : __ldg(halo + (cc - n_loc)); });
        }
        ring.release();
    }
    if (tr0) b2k_trace(fz.trace, 3);
    if constexpr (GK) {
        if (ep.want_nrm) gkl_norm_sums((double)ep.dacc, part, ticket, ring.red(), ring.flag(), fz);
    } else if (ep.want_dot) {
        consumer_sums<1>({(double)ep.dacc}, part, ticket, ring.red(), ring.flag(), [&](int, double tot) {
            *out = tot;
            if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
            if (fz.trace) b2k_trace(fz.trace, 4);
        });
    }
}

// ---------------------------------------------------------------------------------------
// k_spmv_pipe on the compact copy of the matrix (finish_csr / build_compact, single-GPU operators):
//   values   VS = float in a Float64 context when every value round-trips exactly ((double)(float)v bit-identical,
//            no NaN), else T;
//   columns  IS = int16 offsets col - rowblk[tile] when they fit for every nonzero of every tile of <= SP_NNZ
//            nonzeros, else the int32 columns;
//   rowptr   the low 16 bits of rowptr: inside a tile the offset rowptr[r] - pblk[tile] <= SP_NNZ is exact mod 2^16.
// Each consumer rebuilds (T)value and the column and then does exactly what k_spmv_pipe does: the same products
// (rounded in T), summed in the same CSR order by the same thread, the same dacc chain and CTA partials, so y, vout and
// the dot are bit-identical to k_spmv_pipe at the same grid.  Long rows and tiles of more than SPP_RMAX rows read the
// plain global arrays, as there.  With VS = float the products need T slots of their own: one buffer per CTA, so the
// consumers meet once more per tile (before overwriting it) instead of growing every stage by SP_NNZ * 8 bytes.
// The stages are half the size of k_spmv_pipe's, so the ring takes as many as fit beside 4 CTAs per SM.
constexpr int SPC_TV = SP_NNZ + 16;          // staged entries of a 2- or 4-byte nonzero array (16-byte alignment slack)
constexpr int SPC_CTAS = 4;
constexpr int SPC_SMEM_MAX = 233472 / SPC_CTAS - 1024;     // 228 KB per SM, 1 KB reserved per CTA
template <typename X> __device__ __forceinline__ int al_dn(int i) { return i & ~(16 / (int)sizeof(X) - 1); }
template <typename X> __device__ __forceinline__ int al_up(int i) { return al_dn<X>(i + 16 / (int)sizeof(X) - 1); }
template <typename T, typename VS, typename IS> struct SpcLayout {
    static constexpr bool PROD = sizeof(VS) < sizeof(T);
    static constexpr int VAL_BYTES = SPC_TV * (int)sizeof(VS);
    static constexpr int COL_BYTES = SPC_TV * (int)sizeof(IS);
    static constexpr int RP_BYTES = (SPP_RMAX + 16) * 2;
    static constexpr int STAGE = VAL_BYTES + COL_BYTES + RP_BYTES;
    static constexpr int PROD_BYTES = PROD ? SP_NNZ * (int)sizeof(T) : 0;       // the ring's EXTRA bytes
    static constexpr int NSTG = std::min(4, (SPC_SMEM_MAX - PROD_BYTES - TileRing<4, 0>::SMEM) / STAGE);
    using Ring = TileRing<NSTG, STAGE, PROD_BYTES>;
    static_assert(NSTG >= 2 && Ring::SMEM <= SPC_SMEM_MAX, "compact SpMV stage ring does not fit 4 CTAs per SM");
    static_assert(VAL_BYTES % 16 == 0 && COL_BYTES % 16 == 0 && RP_BYTES % 16 == 0, "TMA needs 16-byte offsets");
};

template <typename T, typename VS, typename IS, bool GK = false>
__global__ void __launch_bounds__(SPP_THREADS, SPC_CTAS)
k_spmv_compact(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const T* __restrict__ vals,
               const VS* __restrict__ cvals, const IS* __restrict__ ccol, const uint16_t* __restrict__ crp,
               const T* __restrict__ x, T* __restrict__ y, const int32_t* __restrict__ rowblk,
               const int32_t* __restrict__ pblk, int nblk, T a0, T a1, int shifted, const T* __restrict__ xs,
               const T* __restrict__ dotv, double* __restrict__ part, unsigned* __restrict__ ticket,
               double* __restrict__ out, const SpmvFuse fz) {
    using LY = SpcLayout<T, VS, IS>;
    constexpr bool OFFS = sizeof(IS) == 2;     // columns staged as offsets from the tile's first row
    extern __shared__ __align__(128) uint8_t smem[];
    if (fz.stop && *reinterpret_cast<const volatile int*>(fz.stop)) return;
    typename LY::Ring ring{smem, rowblk, pblk, nblk};
    ring.init();
    if (threadIdx.x >= SPP_CONS) {
        ring.produce(fz.l2_hints, [&](const TileCopy& c, int r0, int r1, int p0, int p1) {
            const int pv = al_dn<VS>(p0), pc = al_dn<IS>(p0), r0a = al_dn<uint16_t>(r0);
            const uint32_t vb = (uint32_t)(al_up<VS>(p1) - pv) * (uint32_t)sizeof(VS);
            const uint32_t cb = (uint32_t)(al_up<IS>(p1) - pc) * (uint32_t)sizeof(IS);
            const uint32_t rb = r1 - r0 <= SPP_RMAX ? (uint32_t)(al_up<uint16_t>(r1 + 1) - r0a) * 2u : 0u;
            c.expect(vb + cb + rb);
            c(0, 0, cvals + pv, vb);
            c(1, LY::VAL_BYTES, ccol + pc, cb);
            c(2, LY::VAL_BYTES + LY::COL_BYTES, crp + r0a, rb);
        });
        return;
    }
    // ---------------------------------- consumers ----------------------------------
    const int tid = threadIdx.x;
    const bool tr0 = fz.trace && blockIdx.x == 0 && tid == 0;
    if (tr0) b2k_trace(fz.trace, 1);
    if (tr0) b2k_trace(fz.trace, 2);
    RowEpilogue<T, GK> ep{fz, x, y, xs, dotv, a0, a1, shifted};
    // The x gather of the next tile is issued before the row sums of this one, so its latency (the first touch of an
    // entry of x misses L2) overlaps them instead of stalling the CTA once per tile.
    constexpr int U = SP_NNZ / SPP_CONS;
    T xv[U];
    auto gather = [&](uint32_t sg, int4 d) {
        if (d.w - d.z > SP_NNZ) return;
        const IS* cg = reinterpret_cast<const IS*>(ring.stage(sg) + LY::VAL_BYTES);
        const int og = d.z - al_dn<IS>(d.z);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = tid + u * SPP_CONS;
            if (i < d.w - d.z) xv[u] = __ldg(x + (OFFS ? d.x + (int)cg[og + i] : (int)cg[og + i]));
        }
    };
    ring.start();
    if ((int)blockIdx.x < nblk) {
        ring.wait();
        gather(ring.s, ring.dn);
    }
    for (int tile = blockIdx.x; tile < nblk; tile += gridDim.x) {
        const int4 d = ring.next(tile);
        const int r0 = d.x, r1 = d.y, p0 = d.z, p1 = d.w;
        const int nnzb = p1 - p0, nrows = r1 - r0;
        auto prefetch_next = [&]() {
            if (tile + (int)gridDim.x < nblk) {
                ring.wait_next();
                gather(ring.s_next(), ring.dn);
            }
        };
        if (nnzb <= SP_NNZ) {
            uint8_t* const st = ring.stage(ring.s);
            VS* vs = reinterpret_cast<VS*>(st);
            const uint16_t* rs = reinterpret_cast<const uint16_t*>(st + LY::VAL_BYTES + LY::COL_BYTES);
            const int offv = p0 - al_dn<VS>(p0), r0a = al_dn<uint16_t>(r0);
            if (ep.scaled) {
#pragma unroll
                for (int u = 0; u < U; ++u) xv[u] *= ep.sc;      // v_j = r_j * (1/β), rounded like scale!!
            }
            T* pr;
            if constexpr (LY::PROD) {
                pr = reinterpret_cast<T*>(smem + LY::Ring::OFF_EXTRA);
                named_bar_sync(1, SPP_CONS);                   // every row sum of the previous tile has read it
            } else {
                pr = reinterpret_cast<T*>(vs) + offv;          // in place, as k_spmv_pipe
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) pr[i] = (T)vs[offv + i] * xv[u];
            }
            named_bar_sync(1, SPP_CONS);
            prefetch_next();
            const bool rp_staged = nrows <= SPP_RMAX;
            for (int r = r0 + tid; r < r1; r += SPP_CONS) {
                const auto ld = ep.load(r);
                int a, b;
                if (rp_staged) {
                    a = (uint16_t)(rs[r - r0a] - (uint16_t)p0);
                    b = (uint16_t)(rs[r + 1 - r0a] - (uint16_t)p0);
                } else {
                    a = rowptr[r] - p0;
                    b = rowptr[r + 1] - p0;
                }
                T sum = (T)0;
                for (int p = a; p < b; ++p) sum += pr[p];
                ep.row(r, ld, sum);
            }
        } else {
            ep.long_row(r0, vals, colidx, p0, nnzb, ring.red(), [&](int32_t c) { return __ldg(x + c); });
            prefetch_next();
        }
        ring.release();
    }
    if (tr0) b2k_trace(fz.trace, 3);
    if constexpr (GK) {
        if (ep.want_nrm) gkl_norm_sums((double)ep.dacc, part, ticket, ring.red(), ring.flag(), fz);
    } else if (ep.want_dot) {
        consumer_sums<1>({(double)ep.dacc}, part, ticket, ring.red(), ring.flag(), [&](int, double tot) {
            *out = tot;
            if (fz.trace) b2k_trace(fz.trace, 4);
        });
    }
}

// One CTA per tile: the compact copy of the tile's nonzeros and row pointers (k_spmv_compact), speculatively, and
// bad |= 1 if a value does not round-trip through float (Float64 only), |= 2 if a column offset does not fit int16.
template <typename T>
__global__ void k_csr_compact(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                              const T* __restrict__ vals, const int32_t* __restrict__ rowblk,
                              const int32_t* __restrict__ pblk, int nblk, float* __restrict__ cvals,
                              int16_t* __restrict__ ccol, uint16_t* __restrict__ crp, int* __restrict__ bad) {
    const int t = blockIdx.x;
    const int r0 = rowblk[t], r1 = rowblk[t + 1], p0 = pblk[t], p1 = pblk[t + 1];
    const bool normal = p1 - p0 <= SP_NNZ;
    bool vbad = false, cbad = false;
    for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
        if (cvals) {
            const double v = (double)vals[p];
            const float f = (float)v;
            vbad |= isnan(v) || __double_as_longlong((double)f) != __double_as_longlong(v);
            cvals[p] = f;
        }
        if (normal) {
            const int o = colidx[p] - r0;
            cbad |= o < -32768 || o > 32767;
            ccol[p] = (int16_t)o;
        }
    }
    const int rend = r1 + (t == nblk - 1);
    for (int r = r0 + threadIdx.x; r < rend; r += blockDim.x) crp[r] = (uint16_t)rowptr[r];
    vbad = __syncthreads_or(vbad);
    cbad = __syncthreads_or(cbad);
    if (threadIdx.x == 0 && (vbad || cbad)) atomicOr(bad, (vbad ? 1 : 0) | (cbad ? 2 : 0));
}

// ---------------------------------------------------------------------------------------
// Fused two-operator SpMV of a pencil (A, B) whose CSR patterns are equal (b2k_pencil_apply / b2k_pencil_rayleigh):
// golubyerecurrence's product `av, bv = genapply(f, v); w = add!!(av, bv, -ρ)` (golubye.jl:198-199, plus
// `add!!(w, V[end-1], -β)` of :202/:211) and the genapply of the Ritz loop (:112-114).  k_spmv_pipe's TileRing with
// B's values staged next to A's in every stage (CsrStage<T, 2>): rowptr and colidx are streamed once, x[c] is gathered once per
// nonzero for both products, and only the outputs are written — 2 (sizeof(T) + 2) nnz + 4 (n + 1) + 3 sizeof(T) n
// bytes instead of 2 (sizeof(T) + 4) nnz + 8 (n + 1) + ... for the composition.
//
// Rounding contract: every row of A x and of B x is formed exactly as k_spmv_pipe forms it — products rounded in T and
// summed in CSR order in T; a long row (> SP_NNZ nonzeros in its tile) as a double sum of rounded products, thread i
// taking nonzeros i, i + 256, ..., then warp butterflies, then the 8 warps in order, rounded to T once.  Then
//   MODE 0: bx = B x;  w = fma(-rho, bx, A x);  w = fma(-beta, vprev, w) when vprev is given;
//   MODE 1: ax = A x;  bx = B x;
// so ax, bx and w are bit-identical to b2k_op_apply with A and with B followed by b2k_vec_axpby(w, bx, -rho, 1) and
// b2k_vec_axpby(w, vprev, -beta, 1).  The dots (<x, w>; <x, ax> and <x, bx>) are fma chains in T over each thread's
// rows, summed by consumer_sums as k_spmv_pipe's dot is: per CTA in double (warp butterflies, then the warps in order),
// then the last CTA to take a ticket adds the CTA partials in CTA order (no FP atomics).  They may differ from b2k_vec_inner in
// the last bits.
//
// A stage holds both value arrays: 35008 B in Float64 (22656 B in Float32), so two stages are 70 KB (45 KB) per CTA.
// Float64 runs 3 CTAs per SM (210 KB; four would need 280 KB of the 227 KB), Float32 4 CTAs per SM (181 KB), the
// shape of the default single-operator variant.  -Xptxas -v: no spills for either.
constexpr int PEN_NSTG = 2;
template <typename T> using PenRing = TileRing<PEN_NSTG, CsrStage<T, 2>::BYTES>;
template <typename T> struct PenCtas { static constexpr int N = sizeof(T) == 8 ? 3 : 4; };

template <typename T, int MODE>
__device__ __forceinline__ void pencil_row(int r, T sa, T sb, T xr, T vp, T nrho, T nbeta, bool has_prev, T* y0,
                                           T* y1, bool hints, uint64_t pol, T& d0, T& d1) {
    if (MODE == 0) {
        T wv = fma(nrho, sb, sa);                       // add!!(av, bv, -ρ): k_axpby MODE 1
        if (has_prev) wv = fma(nbeta, vp, wv);          // add!!(w, V[end-1], -β)
        sa = wv;
    } else {
        d1 = fma(xr, sb, d1);
    }
    d0 = fma(xr, sa, d0);
    if (hints) {
        st_hint(y0 + r, sa, pol);
        st_hint(y1 + r, sb, pol);
    } else {
        y0[r] = sa;
        y1[r] = sb;
    }
}

template <typename T, int NSTG, int MINB, int MODE>
__global__ void __launch_bounds__(SPP_THREADS, MINB)
k_spmv_pencil(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const T* __restrict__ va,
              const T* __restrict__ vb, const T* __restrict__ x, T* __restrict__ y0, T* __restrict__ y1,
              const int32_t* __restrict__ rowblk, const int32_t* __restrict__ pblk, int nblk, T nrho,
              const T* __restrict__ vprev, T nbeta, int want_dot, int l2_hints, double* __restrict__ part,
              unsigned* __restrict__ ticket, double* __restrict__ out) {
    using SG = CsrStage<T, 2>;
    extern __shared__ __align__(128) uint8_t smem[];
    TileRing<NSTG, SG::BYTES> ring{smem, rowblk, pblk, nblk};
    ring.init();
    if (threadIdx.x >= SPP_CONS) {
        ring.produce(l2_hints != 0, [&](const TileCopy& c, int r0, int r1, int p0, int p1) {
            copy_csr_tile<T, 2>(c, {va, vb}, colidx, rowptr, r0, r1, p0, p1);
        });
        return;
    }
    // ---------------------------------- consumers ----------------------------------
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const bool has_prev = MODE == 0 && vprev != nullptr;
    const bool hints = l2_hints != 0;
    const uint64_t pol_last = hints ? l2_policy_evict_last() : 0;
    double* red = ring.red();
    T d0 = (T)0, d1 = (T)0;
    ring.start();
    for (int tile = blockIdx.x; tile < nblk; tile += gridDim.x) {
        const int4 d = ring.next(tile);
        const int r0 = d.x, r1 = d.y, p0 = d.z, p1 = d.w;
        const int nnzb = p1 - p0, nrows = r1 - r0;
        ring.wait();
        if (nnzb <= SP_NNZ) {
            uint8_t* const st = ring.stage(ring.s);
            T* as = reinterpret_cast<T*>(st);
            T* bs = reinterpret_cast<T*>(st + SG::VAL_BYTES);
            const int32_t* cs = reinterpret_cast<const int32_t*>(st + SG::OFF_COL);
            const int32_t* rs = reinterpret_cast<const int32_t*>(st + SG::OFF_RP);
            const int p0a = p0 & ~3, r0a = r0 & ~3, off = p0 - p0a;
            constexpr int U = SP_NNZ / SPP_CONS;
            T xv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) xv[u] = __ldg(x + cs[off + i]);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = tid + u * SPP_CONS;
                if (i < nnzb) {
                    as[off + i] *= xv[u];
                    bs[off + i] *= xv[u];
                }
            }
            named_bar_sync(1, SPP_CONS);
            const bool rp_staged = nrows <= SPP_RMAX;
            for (int r = r0 + tid; r < r1; r += SPP_CONS) {
                const T xr = want_dot ? __ldg(x + r) : (T)0;
                const T vp = has_prev ? __ldg(vprev + r) : (T)0;
                int a, b;
                if (rp_staged) { a = rs[r - r0a]; b = rs[r + 1 - r0a]; }
                else { a = rowptr[r]; b = rowptr[r + 1]; }
                a -= p0a; b -= p0a;
                T sa = (T)0, sb = (T)0;
                for (int p = a; p < b; ++p) {
                    sa += as[p];
                    sb += bs[p];
                }
                pencil_row<T, MODE>(r, sa, sb, xr, vp, nrho, nbeta, has_prev, y0, y1, hints, pol_last, d0, d1);
            }
        } else {
            double acca = 0.0, accb = 0.0;
            for (int i = tid; i < nnzb; i += SPP_CONS) {
                const T xv = __ldg(x + colidx[p0 + i]);
                acca += (double)mul_rn<T>(va[p0 + i], xv);
                accb += (double)mul_rn<T>(vb[p0 + i], xv);
            }
            acca = warp_sum(acca);
            accb = warp_sum(accb);
            if (lane == 0) {
                red[w] = acca;
                red[8 + w] = accb;
            }
            named_bar_sync(1, SPP_CONS);
            if (tid == 0) {
                double ta = 0.0, tb = 0.0;
                for (int i = 0; i < SPP_CONS / 32; ++i) ta += red[i];
                for (int i = 0; i < SPP_CONS / 32; ++i) tb += red[8 + i];
                const T xr = want_dot ? x[r0] : (T)0;
                const T vp = has_prev ? vprev[r0] : (T)0;
                pencil_row<T, MODE>(r0, (T)ta, (T)tb, xr, vp, nrho, nbeta, has_prev, y0, y1, hints, pol_last, d0, d1);
            }
            named_bar_sync(1, SPP_CONS);
        }
        ring.release();
    }
    if (want_dot) {
        consumer_sums<2>({(double)d0, (double)d1}, part, ticket, red, ring.flag(),
                         [&](int k, double tot) { out[k] = tot; });
    }
}

__global__ void k_pattern_diff(const int32_t* __restrict__ a, const int32_t* __restrict__ b, int64_t n,
                               int* __restrict__ diff) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (a[i] != b[i]) {
            *diff = 1;
            return;
        }
}

// SpMM for apply(A, ::Block) (blocklanczos.jl:38): the nonzero stream of a row block is staged ONCE (k_spmv_pipe's
// stage in a 2-stage TileRing, copied without L2 hints) and used for all p <= 8 vectors of the block: 12*nnz + p*16n bytes instead of
// p*(12*nnz + 16n).  Per vector the consumers do what k_spmv_pipe does — thread <-> nonzero gathers x_i and writes the
// rounded product into a product buffer (two of them, alternating, so one barrier per vector), thread <-> row sums
// its products in CSR order — bit-identical to p single-vector applies.  (The first version let one thread per row
// walk its nonzeros for all p vectors: a fifth of the gathers in flight — slower than four SpMVs.)
constexpr int SPM_NSTG = 2;
template <typename T> using SpmRing = SppRing<T, SPM_NSTG, 2 * CsrStage<T, 1>::VAL_BYTES>;    // two product buffers
constexpr int SPM_PMAX = 8;
struct SpmmCols {
    int32_t x[SPM_PMAX], y[SPM_PMAX];
};

template <typename T>
__global__ void __launch_bounds__(SPP_THREADS, 3)
k_spmm_pipe(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const T* __restrict__ vals,
            T* __restrict__ base, int64_t ld, const __grid_constant__ SpmmCols cols, int np,
            const int32_t* __restrict__ rowblk, const int32_t* __restrict__ pblk, int nblk) {
    using SG = CsrStage<T, 1>;
    extern __shared__ __align__(128) uint8_t smem[];
    SpmRing<T> ring{smem, rowblk, pblk, nblk};
    ring.init();
    if (threadIdx.x >= SPP_CONS) {
        ring.produce(false, [&](const TileCopy& c, int r0, int r1, int p0, int p1) {
            copy_csr_tile<T, 1>(c, {vals}, colidx, rowptr, r0, r1, p0, p1);
        });
        return;
    }
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    double* red = ring.red();
    auto xcol = [&](int i) -> const T* { return base + (int64_t)cols.x[i] * ld; };
    auto ycol = [&](int i) -> T* { return base + (int64_t)cols.y[i] * ld; };
    ring.start();
    for (int tile = blockIdx.x; tile < nblk; tile += gridDim.x) {
        const int4 d = ring.next(tile);
        const int r0 = d.x, r1 = d.y, p0 = d.z, p1 = d.w;
        const int nnzb = p1 - p0, nrows = r1 - r0;
        ring.wait();
        if (nnzb <= SP_NNZ) {
            const uint8_t* const st = ring.stage(ring.s);
            const T* vs = reinterpret_cast<const T*>(st);
            const int32_t* cs = reinterpret_cast<const int32_t*>(st + SG::OFF_COL);
            const int32_t* rs = reinterpret_cast<const int32_t*>(st + SG::OFF_RP);
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
                T* prod = reinterpret_cast<T*>(smem + SpmRing<T>::OFF_EXTRA + (iv & 1) * SG::VAL_BYTES);
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
        ring.release(false);
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
        if (shifted) sum = fma(a0, xi, a1 * sum);      // xi = x_i, normalised when the operand is
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
        finish_sums<1>({block_sum((double)dacc, red)}, part, ticket, red, &last, blockDim.x, [&](int, double tot) {
            *out = tot;
            if (ps.on && ps.seq_alpha) peer_publish1(ps.pd, PEER_CH_ALPHA, ps.seq_alpha, tot);
        });
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

// The compact copy of a CSR operator (k_spmv_compact): one pass writes every part and finds which ones are lossless,
// then the parts that are not are freed.  Allocations are padded for the TMA segments, which round the end of a
// tile up to 16 bytes.
int32_t build_compact(b2k_ctx* ctx, b2k_op* op) {
    const bool f64 = ctx->dtype == B2K_F64;
    int* d_bad;
    int h_bad = 0;
    B2K_CUDA(ctx, B2K_DMALLOC(&d_bad, sizeof(int)));
    B2K_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(int), ctx->stream));
    B2K_CUDA(ctx, B2K_DMALLOC(&op->crp, sizeof(uint16_t) * (op->n_rows + 1 + 16)));
    B2K_CUDA(ctx, B2K_DMALLOC(&op->ccol, sizeof(int16_t) * (op->nnz + 16)));
    if (f64) B2K_CUDA(ctx, B2K_DMALLOC(&op->cvals, sizeof(float) * (op->nnz + 16)));
    if (f64)
        k_csr_compact<double><<<op->nblk, 256, 0, ctx->stream>>>(op->rowptr, op->colidx, (const double*)op->vals,
                                                                 op->rowblk, op->pblk, op->nblk, op->cvals, op->ccol,
                                                                 op->crp, d_bad);
    else
        k_csr_compact<float><<<op->nblk, 256, 0, ctx->stream>>>(op->rowptr, op->colidx, (const float*)op->vals,
                                                                op->rowblk, op->pblk, op->nblk, nullptr, op->ccol,
                                                                op->crp, d_bad);
    B2K_LAUNCH_CHECK(ctx);
    B2K_CUDA(ctx, cudaMemcpyAsync(&h_bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    B2K_DFREE(d_bad);
    auto drop = [&](auto*& p) {
        B2K_DFREE(p);
        p = nullptr;
    };
    if (op->cvals && (h_bad & 1)) drop(op->cvals);
    if (h_bad & 2) drop(op->ccol);
    if (!op->cvals && !op->ccol) drop(op->crp);
    return B2K_OK;
}

// rowptr_bad: k_convert_rowptr's out-of-range flag when nothing has read it back yet (an operator without nonzeros
// has no column check); it comes back with the stats, so such an operator pays no synchronisation of its own.
int32_t finish_csr(b2k_ctx* ctx, b2k_op* op, const unsigned long long* rowptr_bad = nullptr) {
    const int64_t n = op->n_rows;
    int* d_stats;
    int h_stats[2] = {0, 0};
    unsigned long long h_bad = 0;
    B2K_CUDA(ctx, B2K_DMALLOC(&d_stats, 2 * sizeof(int)));
    B2K_CUDA(ctx, cudaMemsetAsync(d_stats, 0, 2 * sizeof(int), ctx->stream));
    if (n > 0) {
        k_rowptr_stats<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(op->rowptr, n, d_stats);
        B2K_LAUNCH_CHECK(ctx);
    }
    B2K_CUDA(ctx, cudaMemcpyAsync(h_stats, d_stats, sizeof(h_stats), cudaMemcpyDeviceToHost, ctx->stream));
    if (rowptr_bad)
        B2K_CUDA(ctx, cudaMemcpyAsync(&h_bad, rowptr_bad, sizeof(h_bad), cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    B2K_DFREE(d_stats);
    if (h_bad != 0) return b2k_fail(ctx, B2K_EINVAL, "op_create_csr: rowptr entry outside [base, nnz + base]");
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
    // row-sharded operators keep the plain arrays: their halo columns (n_loc + j) do not fit 16-bit offsets
    if (ctx->nranks == 1 && op->nnz > 0) return build_compact(ctx, op);
    return B2K_OK;
}

// raw host index arrays (int32/int64, base 0/1) -> device rowptr (int32) / global columns (int64).  A row pointer
// outside [base, nnz + base] sets *bad: the test runs on the raw value, as the int32 cast can make an int64 entry
// look in range and monotone.
template <typename IT>
__global__ void k_convert_rowptr(const IT* __restrict__ raw, int base, int32_t* __restrict__ out,
                                 int64_t count, int64_t nnz, unsigned long long* __restrict__ bad) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t v = (int64_t)raw[i];
        if (v < base || v > nnz + base) *bad = 1ull;
        out[i] = (int32_t)(v - base);
    }
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
// Shapes of an operator built from index arrays: no negative size; rows and nnz per GPU below 2^31 (the device
// indices are int32), and so the columns on one GPU, where k_localize_cols stores the column itself (a row shard's
// columns are global, and become local or halo indices that fit); the rows the length of a vector space of this
// context: space 0 in general, any space for a rectangular operator on a single GPU (the (A, A') pair of lssolve /
// svdsolve).
static int32_t check_index_shape(b2k_ctx* ctx, const char* who, int64_t n_rows, int64_t n_cols, int64_t nnz) {
    if (n_rows < 0 || n_cols < 0 || nnz < 0)
        return b2k_fail(ctx, B2K_EINVAL, "%s: negative size (%lld rows, %lld columns, nnz %lld)", who,
                        (long long)n_rows, (long long)n_cols, (long long)nnz);
    const int64_t lim = (int64_t)1 << 31;
    if (n_rows >= lim || nnz >= lim)
        return b2k_fail(ctx, B2K_ENOTSUP, "%s: rows and nnz per GPU must be < 2^31", who);
    if (ctx->nranks == 1 && n_cols >= lim)
        return b2k_fail(ctx, B2K_ENOTSUP, "%s: columns on one GPU must be < 2^31", who);
    bool rows_ok = n_rows == ctx->spaces[0].n;
    if (!rows_ok && ctx->nranks == 1)
        for (const auto& sp : ctx->spaces) rows_ok = rows_ok || sp.n == n_rows;
    if (!rows_ok)
        return b2k_fail(ctx, B2K_EDIM, "%s: %lld local rows but space 0 holds %lld", who,
                        (long long)n_rows, (long long)ctx->spaces[0].n);
    return B2K_OK;
}

static int32_t create_csr_raw(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                              int64_t nnz, const void* rowptr, const void* colidx,
                              const void* vals, int32_t idx_bytes, int32_t index_base) {
    B2K_TRY(check_index_shape(ctx, "op_create_csr", n_rows, n_cols, nnz));
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
    unsigned long long* d_chk = nullptr;      // {min column, max column, a row pointer out of range}
    const int64_t nnz1 = std::max<int64_t>(1, nnz);
    const size_t raw_bytes = (size_t)idx_bytes * std::max<int64_t>(nnz1, n_rows + 1);
    int32_t rc = B2K_OK;
    auto fail = [&](int32_t code) {
        cudaStreamSynchronize(ctx->stream);
        if (d_gcol) B2K_DFREE(d_gcol);
        if (d_raw) B2K_DFREE(d_raw);
        if (d_chk) B2K_DFREE(d_chk);
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
    CK(B2K_DMALLOC(&d_chk, 3 * sizeof(unsigned long long)));
    unsigned long long chk[3] = {~0ull, 0ull, 0ull};
    CK(cudaMemcpyAsync(d_chk, chk, sizeof(chk), cudaMemcpyHostToDevice, ctx->stream));
    const int g = ctx->num_sms * 8;
    CK(cudaMemcpyAsync(d_raw, rowptr, (size_t)idx_bytes * (n_rows + 1), cudaMemcpyHostToDevice, ctx->stream));
    if (idx_bytes == 8) k_convert_rowptr<int64_t><<<g, 256, 0, ctx->stream>>>((const int64_t*)d_raw, index_base, op->rowptr, n_rows + 1, nnz, d_chk + 2);
    else k_convert_rowptr<int32_t><<<g, 256, 0, ctx->stream>>>((const int32_t*)d_raw, index_base, op->rowptr, n_rows + 1, nnz, d_chk + 2);
    ctx->launches++;
    if (nnz > 0) {
        CK(cudaMemcpyAsync(d_raw, colidx, (size_t)idx_bytes * nnz, cudaMemcpyHostToDevice, ctx->stream));
        if (idx_bytes == 8) k_convert_cols<int64_t><<<g, 256, 0, ctx->stream>>>((const int64_t*)d_raw, index_base, d_gcol, nnz);
        else k_convert_cols<int32_t><<<g, 256, 0, ctx->stream>>>((const int32_t*)d_raw, index_base, d_gcol, nnz);
        ctx->launches++;
        CK(cudaMemcpyAsync(op->vals, vals, (size_t)ctx->esize * nnz, cudaMemcpyHostToDevice, ctx->stream));
        // validate the column range on the device
        k_minmax_cols<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(d_gcol, nnz, d_chk, d_chk + 1);
        ctx->launches++;
        // one read-back for both checks; nothing that indexes with these arrays has run yet
        CK(cudaMemcpyAsync(chk, d_chk, sizeof(chk), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (chk[2] != 0)
            return fail(b2k_fail(ctx, B2K_EINVAL, "op_create_csr: rowptr entry outside [%d, nnz + %d]", index_base,
                                 index_base));
        const int64_t colmax = ctx->nranks > 1 ? ctx->n_global : n_cols;
        // negative columns wrap to huge unsigned values and are caught by the max test
        if ((int64_t)chk[1] >= colmax || (int64_t)chk[1] < 0)
            return fail(b2k_fail(ctx, B2K_EINVAL, "op_create_csr: column index out of range [0, %lld)",
                                 (long long)colmax));
    }
#undef CK
    // without nonzeros, plan_halo and localize read no index array, and finish_csr reads the flag back before it
    // uses rowptr for anything but its stats (which read in bounds whatever the values)
    rc = plan_halo(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = localize(ctx, op, d_gcol);
    if (rc == B2K_OK) rc = finish_csr(ctx, op, nnz > 0 ? nullptr : d_chk + 2);
    if (rc != B2K_OK) return fail(rc);
    cudaStreamSynchronize(ctx->stream);
    B2K_DFREE(d_gcol);
    B2K_DFREE(d_raw);
    B2K_DFREE(d_chk);
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
    B2K_TRY(check_index_shape(ctx, "op_create_csc", n_rows, n_cols, nnz));
    std::vector<int64_t> cp, rv;
    if (idx_bytes == 8) widen<int64_t>(colptr, n_cols + 1, index_base, &cp);
    else widen<int32_t>(colptr, n_cols + 1, index_base, &cp);
    // the loops below index rowval / nzval and the rows' fill positions through colptr: check it first
    bool cp_ok = cp[0] == 0 && cp[n_cols] == nnz;
    for (int64_t c = 0; c < n_cols && cp_ok; ++c) cp_ok = cp[c] <= cp[c + 1];
    if (!cp_ok)
        return b2k_fail(ctx, B2K_EINVAL, "op_create_csc: colptr must rise from %d to nnz + %d", index_base,
                        index_base);
    if (idx_bytes == 8) widen<int64_t>(rowval, nnz, index_base, &rv);
    else widen<int32_t>(rowval, nnz, index_base, &rv);
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
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_stencil_fill<T><<<blocks, 256, 0, ctx->stream>>>(d, op->rowptr, d_gcol, (T*)op->vals);
        });
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
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_dense_fill_splitmix<T><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>((T*)op->A, m_local, n, op->ld, seed,
                                                                            (uint64_t)ctx->row_offset, mg);
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

void b2k_op_release(b2k_ctx* ctx, b2k_op* op) {
    cudaStream_t st = ctx ? ctx->stream : nullptr;
    void* ptrs[] = {op->rowptr, op->colidx, op->vals, op->rowblk, op->pblk, op->part, op->halo, op->xall, op->A,
                    op->cvals, op->ccol, op->crp};
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
        b2k_dispatch(ctx, [&](auto tt) {
            using T = decltype(tt);
            k_transpose_gather<T><<<g, 256, 0, ctx->stream>>>(op->rowptr, n, (const T*)op->vals, perm, nnz, t->colidx,
                                                              (T*)t->vals);
        });
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
// L2 eviction hints of the fused pencil SpMV, on the terms of the chained single-operator step (basis.cu): on unless
// B2K_L2_HINTS=0
static bool g_pencil_l2_hints = true;
extern "C" int32_t b2k_debug_set_onepass_variant(int32_t v);     // defined with the one-pass dense step below
static int g_spmv_variant = 1;     // 1 (default): 2 stages x 4 CTAs/SM, 0: 3 stages x 3 CTAs/SM (B2K_SPMV_VARIANT)

extern "C" int32_t b2k_debug_set_spmv_pipe(int32_t on) {
    g_spmv_pipe = on != 0;
    return B2K_OK;
}

// is the SpMV of this process one of the TMA kernels (the ones that carry the GKL epilogue)?
bool b2k_spmv_tma_on() { return g_spmv_pipe; }

extern "C" int32_t b2k_debug_set_spmv_variant(int32_t v) {
    g_spmv_variant = v == 0 ? 0 : 1;
    return B2K_OK;
}

// k_spmv_compact in place of k_spmv_pipe for operators with a compact view: on unless B2K_CSR_COMPACT=0
static bool g_csr_compact = true;
// the CSR SpMV kernel the last apply launched (b2k_debug_spmv_kernel): 0 = none yet, 1 = k_spmv_stream,
// 2 = k_spmv_pipe, 3 = k_spmv_compact
static int g_spmv_kernel = 0;
// the last single-operator SpMV launch that passed its checks (b2k_debug_spmv_launch): {kernel (1 = k_spmv_stream,
// 2 = k_spmv_pipe, 3 = k_spmv_compact, 4 = k_stencil_apply), instance, grid, nblk}.  instance: k_spmv_pipe's variant
// (g_spmv_variant), k_spmv_compact's <VS, IS> as 1 (VS = float) | 2 (IS = int16_t), else 0.
static int32_t g_spmv_launch[4] = {0, 0, 0, 0};

extern "C" int32_t b2k_debug_set_csr_compact(int32_t on) {
    g_csr_compact = on != 0;
    return B2K_OK;
}

extern "C" int32_t b2k_debug_spmv_kernel(void) { return g_spmv_kernel; }

// the compact view of an operator: 0 = none, else 4 (16-bit row pointers) | 2 (16-bit column offsets) | 1 (Float32
// values in a Float64 context)
extern "C" int32_t b2k_debug_csr_format(const b2k_op* op) {
    if (!op || !op->crp) return 0;
    return 4 | (op->ccol ? 2 : 0) | (op->cvals ? 1 : 0);
}

extern "C" int32_t b2k_debug_spmv_launch(int32_t* out) {
    if (!out) return B2K_EINVAL;
    for (int i = 0; i < 4; ++i) out[i] = g_spmv_launch[i];
    return B2K_OK;
}

// The tile boundaries of a CSR operator: *nblk, and rowblk[0 .. nblk] when rowblk is given (nblk = 0 for a matrix-free
// stencil).
extern "C" int32_t b2k_debug_op_tiles(b2k_ctx* ctx, const b2k_op* op, int32_t* rowblk, int32_t* nblk) {
    if (!ctx || !op || !nblk) return B2K_EINVAL;
    *nblk = op->nblk;
    if (rowblk && op->rowblk) {
        B2K_CUDA(ctx, cudaMemcpyAsync(rowblk, op->rowblk, sizeof(int32_t) * (op->nblk + 1), cudaMemcpyDeviceToHost,
                                      ctx->stream));
        B2K_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return B2K_OK;
}

// b2k_enqueue_apply_fused with a SpmvFuse built from host arguments, through the production checks.  Vectors < 0 are
// absent; xscale (null: none) and dsub_scale are copied to device scratch of their own, and the stop flag is a private
// device int set to `stop`.  The dot goes to a scratch slot prefilled with *dot (no slot at all when no_slot is set);
// on return *dot is what the slot holds, so a launch that did not write it returns the value passed in.
extern "C" int32_t b2k_debug_apply_fused(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y, double a0, double a1,
                                         int32_t shifted, b2k_vec dotv, const double* xscale, b2k_vec vout,
                                         int32_t dot_self, b2k_vec dsub, double dsub_scale, int32_t l2_hints,
                                         int32_t stop, int32_t no_slot, double* dot) {
    if (!ctx || !op || !dot) return B2K_EINVAL;
    VecRef rx, ry, rd, rv, rs;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    if (dotv >= 0) B2K_TRY(b2k_resolve(ctx, dotv, &rd));
    if (vout >= 0) B2K_TRY(b2k_resolve(ctx, vout, &rv));
    if (dsub >= 0) B2K_TRY(b2k_resolve(ctx, dsub, &rs));
    double h[4] = {*dot, xscale ? *xscale : 0.0, dsub_scale, 0.0};     // slot, xscale, dot_sub_scale, stop
    const int32_t hstop = stop;
    memcpy(&h[3], &hstop, sizeof(hstop));
    double* d = nullptr;
    B2K_CUDA(ctx, B2K_DMALLOC(&d, sizeof(h)));
    cudaError_t e = cudaMemcpyAsync(d, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream);
    int32_t rc = B2K_OK;
    if (e == cudaSuccess) {
        SpmvFuse fz;
        memset(&fz, 0, sizeof(fz));
        fz.xscale = xscale ? d + 1 : nullptr;
        fz.vout = vout >= 0 ? rv.ptr : nullptr;
        fz.stop = reinterpret_cast<const int*>(d + 3);
        fz.dot_self = dot_self;
        fz.l2_hints = l2_hints;
        fz.dot_sub_vec = dsub >= 0 ? rs.ptr : nullptr;
        fz.dot_sub_scale = dsub >= 0 ? d + 2 : nullptr;
        rc = b2k_enqueue_apply_fused(ctx, op, rx, ry, a0, a1, shifted != 0, dotv >= 0 ? &rd : nullptr,
                                     no_slot ? nullptr : d, &fz);
        e = cudaMemcpyAsync(dot, d, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    B2K_DFREE(d);
    B2K_TRY(rc);
    B2K_CUDA(ctx, e);
    return B2K_OK;
}

// opt in to > 48 KB dynamic shared memory for the pipelined SpMV (called per context)
int32_t b2k_spmv_init(b2k_ctx* ctx) {
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_spmm_pipe<double>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SpmRing<double>::SMEM));
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_spmm_pipe<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SpmRing<float>::SMEM));
    // every instance, with and without the GKL epilogue
#define SPP_ATTR(T, NS, MB)                                                                                    \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<T, NS, MB>), cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                       SppRing<T, NS>::SMEM));                                                 \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pipe<T, NS, MB, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       SppRing<T, NS>::SMEM))
    SPP_ATTR(double, 3, 3);
    SPP_ATTR(float, 3, 3);
    SPP_ATTR(double, 2, 4);
    SPP_ATTR(float, 2, 4);
#undef SPP_ATTR
#define SPC_ATTR(T, VS, IS)                                                                                    \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_compact<T, VS, IS>), cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       SpcLayout<T, VS, IS>::Ring::SMEM));                                     \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_compact<T, VS, IS, true>),                                      \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, SpcLayout<T, VS, IS>::Ring::SMEM))
    SPC_ATTR(double, float, int16_t);
    SPC_ATTR(double, float, int32_t);
    SPC_ATTR(double, double, int16_t);
    SPC_ATTR(float, float, int16_t);
#undef SPC_ATTR
    if (const char* e = getenv("B2K_CSR_COMPACT")) g_csr_compact = e[0] != '0';
#define PEN_ATTR(T, MODE)                                                                                      \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_spmv_pencil<T, PEN_NSTG, PenCtas<T>::N, MODE>),                     \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, PenRing<T>::SMEM))
    PEN_ATTR(double, 0);
    PEN_ATTR(double, 1);
    PEN_ATTR(float, 0);
    PEN_ATTR(float, 1);
#undef PEN_ATTR
    if (const char* e = getenv("B2K_L2_HINTS")) g_pencil_l2_hints = e[0] != '0';
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
    const bool gk = fz.pvec != nullptr;
    if (gk && (op->kind != 0 || !g_spmv_pipe || ctx->nranks > 1 || !fz.acoef || fz.vout || fz.dot_self || dotv || shifted))
        return b2k_fail(ctx, B2K_ENOTSUP, "fused apply: the GKL epilogue needs a single-GPU CSR operator and a TMA kernel");
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
                    b2k_dispatch(ctx, [&](auto t) {
                        using T = decltype(t);
                        k_halo_push<T><<<g, 256, 0, ctx->stream>>>((const T*)x.ptr, x.n, ps, ctx->d_sync + B2K_SYNC_HALO,
                                                                   fz.stop);
                    });
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
        g_spmv_launch[0] = 4; g_spmv_launch[1] = 0; g_spmv_launch[2] = grid; g_spmv_launch[3] = 0;
        const int pr2 = b2k_prof_begin(ctx, 0, 2.0 * ctx->esize * op->n_rows);
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_stencil_apply<T><<<grid, 256, 0, ctx->stream>>>(sa, (const T*)xsrc, (const T*)halo, (T*)y.ptr, T(a0), T(a1),
                                                              shifted ? 1 : 0, dotv ? (const T*)dotv->ptr : nullptr,
                                                              op->part, ctx->d_sync, out, fz, ps);
        });
        b2k_prof_end(ctx, pr2);
        B2K_LAUNCH_CHECK(ctx);
        return B2K_OK;
    }
    // algorithmic bytes: matrix (as streamed) + x + y, plus the normalised copy of x a chained Lanczos step stores
    // (fz.vout), or the previous vector the GKL epilogue reads and stores (fz.pvec, fz.pout)
    const bool compact = g_spmv_pipe && g_csr_compact && op->crp != nullptr;
    const double vbytes = (compact && op->cvals) ? 4.0 : (double)ctx->esize, cbytes = (compact && op->ccol) ? 2.0 : 4.0;
    const int pr = b2k_prof_begin(ctx, 0, (double)op->nnz * (vbytes + cbytes) + (compact ? 2.0 : 4.0) * (op->n_rows + 1) +
                                              (2.0 + (fz.vout ? 1.0 : 0.0) + (gk ? 1.0 : 0.0) + (fz.pout ? 1.0 : 0.0)) *
                                                  ctx->esize * op->n_rows);
    g_spmv_kernel = compact ? 3 : (g_spmv_pipe ? 2 : 1);
    if (compact) {
        // the grid of k_spmv_pipe's variant: the CTA partials of the dot, and so its rounding, stay the same
        const int per_sm = g_spmv_variant == 1 ? 4 : 3;
        const int grid = std::min(op->nblk, per_sm * ctx->num_sms);
        g_spmv_launch[0] = 3; g_spmv_launch[2] = grid; g_spmv_launch[3] = op->nblk;
        g_spmv_launch[1] = (ctx->dtype == B2K_F32 || op->cvals ? 1 : 0) | (op->ccol ? 2 : 0);
#define LAUNCH_CG(T, VS, IS, GK, cv, cc)                                                                       \
    k_spmv_compact<T, VS, IS, GK><<<grid, SPP_THREADS, SpcLayout<T, VS, IS>::Ring::SMEM, ctx->stream>>>(             \
        op->rowptr, op->colidx, (const T*)op->vals, (const VS*)(cv), (const IS*)(cc), op->crp, (const T*)xsrc, \
        (T*)y.ptr, op->rowblk, op->pblk, op->nblk, (T)a0, (T)a1, shifted ? 1 : 0, (const T*)x.ptr,            \
        dotv ? (const T*)dotv->ptr : nullptr, op->part, ctx->d_sync, out, fz)
#define LAUNCH_C(T, VS, IS, cv, cc)                                                                            \
    do {                                                                                                       \
        if (gk) LAUNCH_CG(T, VS, IS, true, cv, cc);                                                            \
        else LAUNCH_CG(T, VS, IS, false, cv, cc);                                                              \
    } while (0)
        if (ctx->dtype == B2K_F64) {
            if (op->cvals && op->ccol) LAUNCH_C(double, float, int16_t, op->cvals, op->ccol);
            else if (op->cvals) LAUNCH_C(double, float, int32_t, op->cvals, op->colidx);
            else LAUNCH_C(double, double, int16_t, op->vals, op->ccol);
        } else {
            LAUNCH_C(float, float, int16_t, op->vals, op->ccol);
        }
#undef LAUNCH_C
#undef LAUNCH_CG
    } else if (g_spmv_pipe) {
        const int per_sm = g_spmv_variant == 1 ? 4 : 3;
        const int grid = std::min(op->nblk, per_sm * ctx->num_sms);
        g_spmv_launch[0] = 2; g_spmv_launch[1] = g_spmv_variant; g_spmv_launch[2] = grid; g_spmv_launch[3] = op->nblk;
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            b2k_flag(gk, [&](auto GK) {
                b2k_flag(g_spmv_variant == 1, [&](auto v1) {      // variant 1: two stages of 4 row blocks, else 3 of 3
                    constexpr int NS = v1 ? 2 : 3, MB = v1 ? 4 : 3;
                    k_spmv_pipe<T, NS, MB, GK><<<grid, SPP_THREADS, SppRing<T, NS>::SMEM, ctx->stream>>>(
                        op->rowptr, op->colidx, (const T*)op->vals, (const T*)xsrc, (const T*)halo, n_loc, (T*)y.ptr,
                        op->rowblk, op->pblk, op->nblk, T(a0), T(a1), shifted ? 1 : 0, (const T*)x.ptr,
                        dotv ? (const T*)dotv->ptr : nullptr, op->part, ctx->d_sync, out, fz, ps);
                });
            });
        });
    } else {
        g_spmv_launch[0] = 1; g_spmv_launch[1] = 0; g_spmv_launch[2] = op->nblk; g_spmv_launch[3] = op->nblk;
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_spmv_stream<T><<<op->nblk, SP_BT, 0, ctx->stream>>>(
                op->rowptr, op->colidx, (const T*)op->vals, (const T*)xsrc, (const T*)halo, n_loc, (T*)y.ptr, op->rowblk,
                T(a0), T(a1), shifted ? 1 : 0, (const T*)x.ptr, dotv ? (const T*)dotv->ptr : nullptr, op->part,
                ctx->d_sync, out, fz, ps);
        });
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
// Pencils (A, B) for geneigsolve / Golub-Ye (golubye.jl).  A pencil is a host-side pairing: it owns no device memory,
// and keeps A and B, which must outlive it.  Same-pattern CSR pairs take k_spmv_pencil (one launch per call), every
// other pair the composition of b2k_op_apply / b2k_vec_axpby / b2k_vec_inner.

struct b2k_pencil {
    b2k_ctx* ctx;
    const b2k_op* A;
    const b2k_op* B;
    int64_t n;
    int32_t fused;
};

static int32_t g_pencil_path = 0;    // path of the last pencil call that passed its checks: 0 composed, 1 fused

extern "C" int32_t b2k_debug_pencil_path(void) { return g_pencil_path; }

extern "C" int32_t b2k_pencil_create(b2k_ctx* ctx, void** out, const b2k_op* A, const b2k_op* B) {
    if (!ctx || !out || !A || !B) return B2K_EINVAL;
    if (A == B) return b2k_fail(ctx, B2K_EINVAL, "pencil_create: A and B are the same operator");
    for (const b2k_op* op : {A, B})
        if (std::find(ctx->ops.begin(), ctx->ops.end(), op) == ctx->ops.end())
            return b2k_fail(ctx, B2K_EINVAL, "pencil_create: an operator of another context");
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "pencil_create: row-sharded contexts are not supported");
    if (A->n_rows != A->n_cols || B->n_rows != B->n_cols || A->n_rows != B->n_rows)
        return b2k_fail(ctx, B2K_EDIM, "pencil_create: A (%lld x %lld) and B (%lld x %lld) must be square of one size",
                        (long long)A->n_rows, (long long)A->n_cols, (long long)B->n_rows, (long long)B->n_cols);
    int32_t fused = 0;
    if (A->kind == 0 && B->kind == 0 && A->nnz == B->nnz && A->n_rows > 0) {
        int* d_diff;
        int h_diff = 0;
        B2K_CUDA(ctx, B2K_DMALLOC(&d_diff, sizeof(int)));
        B2K_CUDA(ctx, cudaMemsetAsync(d_diff, 0, sizeof(int), ctx->stream));
        const int g = ctx->num_sms * 4;
        k_pattern_diff<<<g, 256, 0, ctx->stream>>>(A->rowptr, B->rowptr, A->n_rows + 1, d_diff);
        B2K_LAUNCH_CHECK(ctx);
        if (A->nnz > 0) {
            k_pattern_diff<<<g, 256, 0, ctx->stream>>>(A->colidx, B->colidx, A->nnz, d_diff);
            B2K_LAUNCH_CHECK(ctx);
        }
        B2K_CUDA(ctx, cudaMemcpyAsync(&h_diff, d_diff, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        B2K_TRY(b2k_stream_sync(ctx));
        B2K_DFREE(d_diff);
        fused = h_diff == 0;
    }
    *out = new b2k_pencil{ctx, A, B, A->n_rows, fused};
    return B2K_OK;
}

extern "C" int32_t b2k_pencil_destroy(b2k_ctx* ctx, void* Pv) {
    if (!ctx || !Pv) return B2K_EINVAL;
    b2k_pencil* P = static_cast<b2k_pencil*>(Pv);
    if (P->ctx != ctx) return b2k_fail(ctx, B2K_EINVAL, "pencil_destroy: the pencil belongs to another context");
    delete P;
    return B2K_OK;
}

// checks shared by both calls: resolves the handles (v[i] < 0 with opt[i]: absent), lengths, pairwise distinct
static int32_t pencil_check(b2k_ctx* ctx, const b2k_pencil* P, const char* who, const b2k_vec* v, const bool* opt,
                            int cnt, VecRef* r) {
    if (P->ctx != ctx) return b2k_fail(ctx, B2K_EINVAL, "%s: the pencil belongs to another context", who);
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "%s: row-sharded contexts are not supported", who);
    for (int i = 0; i < cnt; ++i) {
        r[i].ptr = nullptr;
        if (opt[i] && v[i] < 0) continue;
        B2K_TRY(b2k_resolve(ctx, v[i], &r[i]));
        if (r[i].n != P->n)
            return b2k_fail(ctx, B2K_EDIM, "%s: vector %d has %lld entries, the pencil %lld", who, i,
                            (long long)r[i].n, (long long)P->n);
        for (int j = 0; j < i; ++j)
            if (r[j].ptr && r[j].ptr == r[i].ptr)
                return b2k_fail(ctx, B2K_EINVAL, "%s: vectors %d and %d are the same", who, j, i);
    }
    return B2K_OK;
}

template <typename T, int MODE>
static int32_t pencil_launch(b2k_ctx* ctx, const b2k_pencil* P, const VecRef& x, const VecRef& y0, const VecRef& y1,
                             double rho, const VecRef* vprev, double beta, bool want_dot, double bytes) {
    const b2k_op* A = P->A;
    const int grid = std::min(A->nblk, PenCtas<T>::N * ctx->num_sms);
    const int pr = b2k_prof_begin(ctx, 0, bytes);
    k_spmv_pencil<T, PEN_NSTG, PenCtas<T>::N, MODE><<<grid, SPP_THREADS, PenRing<T>::SMEM, ctx->stream>>>(
        A->rowptr, A->colidx, (const T*)A->vals, (const T*)P->B->vals, (const T*)x.ptr, (T*)y0.ptr, (T*)y1.ptr,
        A->rowblk, A->pblk, A->nblk, (T)(-rho), vprev ? (const T*)vprev->ptr : nullptr, (T)(-beta), want_dot ? 1 : 0,
        g_pencil_l2_hints ? 1 : 0, ctx->d_part_s, ctx->d_sync, ctx->d_res);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_pencil_apply(b2k_ctx* ctx, const void* Pv, b2k_vec x, b2k_vec w, b2k_vec bx, double rho,
                                    b2k_vec vprev, double beta, double* dot) {
    if (!ctx || !Pv) return B2K_EINVAL;
    const b2k_pencil* P = static_cast<const b2k_pencil*>(Pv);
    const b2k_vec v[4] = {x, w, bx, vprev};
    const bool opt[4] = {false, false, false, true};
    VecRef r[4];
    B2K_TRY(pencil_check(ctx, P, "pencil_apply", v, opt, 4, r));
    const bool has_prev = r[3].ptr != nullptr;
    g_pencil_path = P->fused;
    if (!P->fused) {
        B2K_TRY(b2k_op_apply(ctx, P->A, x, w));
        B2K_TRY(b2k_op_apply(ctx, P->B, x, bx));
        B2K_TRY(b2k_vec_axpby(ctx, w, bx, -rho, 1.0));
        if (has_prev) B2K_TRY(b2k_vec_axpby(ctx, w, vprev, -beta, 1.0));
        return dot ? b2k_vec_inner(ctx, x, w, dot) : B2K_OK;
    }
    if (P->n == 0) {
        if (dot) *dot = 0.0;
        return B2K_OK;
    }
    const double es = ctx->esize, n = (double)P->n;
    const double bytes = (double)P->A->nnz * (2 * es + 4) + 4.0 * (n + 1) + (has_prev ? 4.0 : 3.0) * es * n;
    B2K_TRY(b2k_dispatch(ctx, [&](auto t) {
        return pencil_launch<decltype(t), 0>(ctx, P, r[0], r[1], r[2], rho, has_prev ? &r[3] : nullptr, beta, dot, bytes);
    }));
    if (!dot) return B2K_OK;
    B2K_TRY(b2k_fetch_results(ctx, 1, 0));
    *dot = ctx->h_res[0];
    return B2K_OK;
}

extern "C" int32_t b2k_pencil_rayleigh(b2k_ctx* ctx, const void* Pv, b2k_vec x, b2k_vec ax, b2k_vec bx,
                                       double* xax, double* xbx) {
    if (!ctx || !Pv) return B2K_EINVAL;
    const b2k_pencil* P = static_cast<const b2k_pencil*>(Pv);
    const b2k_vec v[3] = {x, ax, bx};
    const bool opt[3] = {false, false, false};
    VecRef r[3];
    B2K_TRY(pencil_check(ctx, P, "pencil_rayleigh", v, opt, 3, r));
    g_pencil_path = P->fused;
    const bool want_dot = xax || xbx;
    if (!P->fused) {
        B2K_TRY(b2k_op_apply(ctx, P->A, x, ax));
        B2K_TRY(b2k_op_apply(ctx, P->B, x, bx));
        if (xax) B2K_TRY(b2k_vec_inner(ctx, x, ax, xax));
        if (xbx) B2K_TRY(b2k_vec_inner(ctx, x, bx, xbx));
        return B2K_OK;
    }
    if (P->n == 0) {
        if (xax) *xax = 0.0;
        if (xbx) *xbx = 0.0;
        return B2K_OK;
    }
    const double es = ctx->esize, n = (double)P->n;
    const double bytes = (double)P->A->nnz * (2 * es + 4) + 4.0 * (n + 1) + 3.0 * es * n;
    B2K_TRY(b2k_dispatch(ctx, [&](auto t) {
        return pencil_launch<decltype(t), 1>(ctx, P, r[0], r[1], r[2], 0.0, nullptr, 0.0, want_dot, bytes);
    }));
    if (!want_dot) return B2K_OK;
    B2K_TRY(b2k_fetch_results(ctx, 2, 0));
    if (xax) *xax = ctx->h_res[0];
    if (xbx) *xbx = ctx->h_res[1];
    return B2K_OK;
}

// ------------------------------------------------------------------------------------------------
// One pass over a dense A for BOTH products of a Golub-Kahan-Lanczos step (SURVEY §8f-4, the flagged
// `onepass` mode of the GKL mirror; the reference's step reads A twice: gkl.jl:308-323 `apply_adjoint` then
// `apply_normal`).  While y = A x is formed, z = A'(A x) is accumulated from the same resident row tile; the
// host recovers A'u_{k+1} = (z - sum_j c_j A'u_j) / beta_k from it (factorizations/gkl.py) without a second
// pass.  The reduction over rows of y = A x is LOCAL to a row tile, so no grid-wide barrier is needed:
//
//   tile   = 32 rows x n columns of the column-major A (n <= 1700 Float32 / 846 Float64), parked in shared
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
int32_t g_onepass_launch[4] = {-1, 0, 0, 0};     // {variant, NZ, grid, ntiles} of the last launch (b2k_debug_onepass_launch)

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
    g_onepass_launch[0] = 1; g_onepass_launch[1] = 0; g_onepass_launch[2] = grid; g_onepass_launch[3] = (int32_t)ntiles;
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
    g_onepass_launch[0] = 0;
    g_onepass_launch[1] = n <= OP_T ? 1 : n <= 2 * OP_T ? 2 : n <= 4 * OP_T ? 4 : OP_ZMAX;
    g_onepass_launch[2] = grid;
    g_onepass_launch[3] = (int32_t)ntiles;
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
    return b2k_dispatch(ctx, [&](auto t) { return onepass_t<decltype(t)>(ctx, mop, rx, ry, rz); });
}

// A/B switch of the one-pass dense step (tools / tests / bench.py's c4o child): 0 = variant A, 1 = variant B
extern "C" int32_t b2k_debug_set_onepass_variant(int32_t v) {
    if (v < 0 || v > 1) return B2K_EINVAL;
    g_onepass_variant = v;
    return B2K_OK;
}

// the last one-pass launch that passed its checks: {variant (0 = A, 1 = B, -1 = none yet), NZ (variant A's template
// instance, 0 for B), grid, ntiles} — the grid depends on the occupancy, which a test of the summation order needs
extern "C" int32_t b2k_debug_onepass_launch(int32_t* out) {
    if (!out) return B2K_EINVAL;
    for (int i = 0; i < 4; ++i) out[i] = g_onepass_launch[i];
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
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_spmm_pipe<T><<<grid, SPP_THREADS, SpmRing<T>::SMEM, ctx->stream>>>(
                op->rowptr, op->colidx, (const T*)op->vals, (T*)sp.base, sp.ld, cols, np, op->rowblk, op->pblk, op->nblk);
        });
        b2k_prof_end(ctx, pr);
        B2K_LAUNCH_CHECK(ctx);
    }
    return B2K_OK;
}
