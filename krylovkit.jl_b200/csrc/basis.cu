// basis.cu — OrthonormalBasis operations on the device slab: project!!, unproject!!,
// the orthogonalize!! family (fused CGS / CGS2, pipelined MGS), basistransform!,
// rank1update!, Householder, block products, and the fused Lanczos expansion step.
// Reference semantics: KrylovKit.jl src/orthonormal.jl, src/factorizations/lanczos.jl.
#include "tsk.cuh"
#include <cmath>
#include <algorithm>

// blas1.cu
int32_t b2k_enqueue_dot(b2k_ctx* ctx, const void* q, void* x, int64_t n, const void* qprev,
                        int sprev_slot, int slot, int accum_slot);
int32_t b2k_enqueue_axpy_dev(b2k_ctx* ctx, void* x, const void* q, int s_slot, int64_t n);
// spmv.cu
int32_t b2k_enqueue_apply(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y,
                          double a0, double a1, bool shifted, const VecRef* dotv, int dot_slot);
bool b2k_spmv_tma_on();

using namespace tsk;

namespace {

// ---------------------------------------------------------------- kernels ----

template <typename T, bool UPDATE, bool PROJECT>
__global__ void __launch_bounds__(NTHREADS, 1)
k_phase(const __grid_constant__ PhaseParams<T> p, const __grid_constant__ ColList cl) {
    extern __shared__ __align__(128) uint8_t smem[];
    SmemView sm(smem);
    const int64_t ntiles = (p.n + Cfg<T>::R - 1) / Cfg<T>::R;
    const bool ragged = (p.n % Cfg<T>::R) != 0 && ((ntiles - 1) % gridDim.x) == blockIdx.x;
    pipe_setup(sm, ragged);
    Pipe st;
    if (threadIdx.x >= NCONS) producer_phase<T>(p, cl, sm, st);
    else if (p.prologue) consumer_phase<T, UPDATE, PROJECT, true>(p, sm, st);
    else consumer_phase<T, UPDATE, PROJECT, false>(p, sm, st);
}

// Cooperative fused Gram-Schmidt kernel: up to three phases in one launch, separated by
// grid barriers.  kind: 0 = project, 1 = update+project, 2 = update (+norm).
template <typename T>
struct FusedParams {
    PhaseParams<T> ph[3];
    int32_t kind[3];
    int32_t nph;
    int32_t run_ahead[2];    // boundary i (after phase i): producers skip it (boundary_sync), set by launch_fused
    unsigned* barrier;
    unsigned barrier_base;   // counter value before this launch
    const int* stop;         // device flag: when set, the launch does nothing (see FinalizeParams)
    FinalizeParams fin;      // optional in-kernel finalisation by the last CTA
    PeerStep ps;             // row-sharded contexts: cross-GPU exchanges of this launch (ps.on == 0: one GPU)
    unsigned long long* trace;   // optional event trace
};

// Phase boundary of a row-sharded launch.  The local grid barrier and the cross-GPU sum of the projection
// coefficients are one step: the last CTA of this rank to arrive reduces the rank's per-CTA partials (same
// fixed order as on one GPU) and stores them into EVERY rank's window; every CTA of every rank then waits, in
// its own window, for the nranks contributions — which also proves that all local CTAs have arrived.  One
// NVLink store latency instead of a kernel boundary + ncclAllReduce + a kernel boundary.
// Like grid_barrier, called by the consumer threads only when the boundary is run-ahead.
template <typename T>
__device__ __forceinline__ void peer_boundary(const FusedParams<T>& fp, int i, uint8_t* smem) {
    const bool ra = fp.run_ahead[i] != 0;
    __threadfence();
    if (!ra) asm volatile("fence.proxy.async;" ::: "memory");
    boundary_sync(ra);
    int* flag = reinterpret_cast<int*>(smem + OFF_RED + 256);
    if (threadIdx.x == 0) {
        const unsigned old = atomicAdd(fp.barrier, 1u);
        *flag = (old == fp.barrier_base + (unsigned)(i + 1) * gridDim.x - 1u);
    }
    boundary_sync(ra);
    const PeerDev& pd = fp.ps.pd;
    const int tid = threadIdx.x;
    const unsigned long long seq = fp.ps.seq_coef[i];
    if (*flag && tid < NCONS) {
        __threadfence();
        const int k = fp.ph[i].k;
        const int L = coef_lanes(k);
        const int j = tid / L, l = tid % L;
        const bool valid = j < k;
        const double a = coef_colsum(fp.ph[i].part_h, gridDim.x, B2K_KSTRIDE, j, l, L, valid);
        if (valid && l == 0)
            for (int p = 0; p < pd.nranks; ++p) peer_slot(pd, p, PEER_CH_COEF, seq, pd.rank)[j] = a;
        __threadfence_system();
        named_bar_sync(1, NCONS);
        if (tid < pd.nranks) st_release_sys_u64(peer_flag(pd, tid, PEER_CH_COEF, seq, pd.rank), seq);
    }
    peer_wait(pd, PEER_CH_COEF, seq, tid);
    boundary_sync(ra);
}

template <typename T>
__global__ void __launch_bounds__(NTHREADS, 1)
k_gs_fused(const __grid_constant__ FusedParams<T> fp, const __grid_constant__ ColList cl) {
    extern __shared__ __align__(128) uint8_t smem[];
    if (fp.stop && *reinterpret_cast<const volatile int*>(fp.stop)) {   // uniform over the grid
        // keep the monotone barrier counter in step with the host's bookkeeping (launch_fused)
        if (threadIdx.x == 0 && fp.nph > 1) atomicAdd(fp.barrier, (unsigned)(fp.nph - 1));
        return;
    }
    SmemView sm(smem);
    const bool tr0 = fp.trace && blockIdx.x == 0 && threadIdx.x == 0;
    if (tr0) b2k_trace(fp.trace, 10);
    const int64_t n = fp.ph[0].n;
    const int64_t ntiles = (n + Cfg<T>::R - 1) / Cfg<T>::R;
    const bool ragged = (n % Cfg<T>::R) != 0 && ((ntiles - 1) % gridDim.x) == blockIdx.x;
    pipe_setup(sm, ragged);
    Pipe st;
    const bool prod = threadIdx.x >= NCONS;
    if (fp.ps.on && fp.ps.seq_alpha && !prod) {
        // <v, A v>: every rank's partial must be in my window before the prologue; the producer warps do not
        // wait — they fill the ring with the first basis tiles meanwhile
        peer_wait(fp.ps.pd, PEER_CH_ALPHA, fp.ps.seq_alpha, threadIdx.x);
        named_bar_sync(1, NCONS);
    }
    if (tr0) b2k_trace(fp.trace, 11);
    for (int i = 0; i < fp.nph; ++i) {
        if (prod) {
            producer_phase<T>(fp.ph[i], cl, sm, st);
        } else {
            const PhaseParams<T>& p = fp.ph[i];
            if (fp.kind[i] == 0) {
                if (p.prologue) consumer_phase<T, false, true, true>(p, sm, st);
                else consumer_phase<T, false, true, false>(p, sm, st);
            } else if (fp.kind[i] == 1) {
                if (p.prologue) consumer_phase<T, true, true, true>(p, sm, st);
                else consumer_phase<T, true, true, false>(p, sm, st);
            } else {
                if (p.prologue) consumer_phase<T, true, false, true>(p, sm, st);
                else consumer_phase<T, true, false, false>(p, sm, st);
            }
        }
        if (tr0) b2k_trace(fp.trace, 12 + i);           // CTA 0 has finished the phase's tiles
        if (i + 1 < fp.nph && !(prod && fp.run_ahead[i])) {
            if (fp.ps.on) peer_boundary<T>(fp, i, smem);
            else grid_barrier(fp.barrier, fp.barrier_base + (unsigned)(i + 1) * gridDim.x, fp.run_ahead[i] != 0);
            if (tr0) b2k_trace(fp.trace, 15 + i);       // ... and left the boundary
        }
    }
    if (fp.fin.enabled && !prod) {
        // the last CTA to finish (ticket) reduces the per-CTA partials and publishes the step's scalars
        double* sh = reinterpret_cast<double*>(smem + OFF_RED);
        int* flag = reinterpret_cast<int*>(smem + OFF_RED + 256);
        if (fp.ps.on) __threadfence_system();      // halo rows stored into the neighbours' windows
        else __threadfence();
        named_bar_sync(1, NCONS);
        if (threadIdx.x == 0) {
            const unsigned t = atomicInc(fp.fin.ticket, gridDim.x - 1);
            *flag = (t == gridDim.x - 1);
        }
        named_bar_sync(1, NCONS);
        if (*flag) {
            __threadfence();
            if (fp.trace && threadIdx.x == 0) b2k_trace(fp.trace, 18);      // last CTA enters the finaliser
            finalize_block(fp.fin, threadIdx.x, sh, fp.ps.on ? &fp.ps : nullptr);
            if (fp.trace && threadIdx.x == 0) b2k_trace(fp.trace, 19);
        }
    }
}

// one block of NCONS threads: the stand-alone form of finalize_block
__global__ void __launch_bounds__(NCONS)
k_finalize(const double* __restrict__ A, const double* __restrict__ B, const double* __restrict__ N, int G,
           int stride, int k, double* __restrict__ res, int off, int noff) {
    __shared__ double sh[2];
    FinalizeParams f;
    f.A = A; f.B = B; f.N = N; f.G = G; f.stride = stride; f.k = k; f.res = res; f.off = off; f.noff = noff;
    f.rec = nullptr; f.alpha_col = -1; f.tol = 0.0; f.stop = nullptr; f.ticket = nullptr; f.enabled = 1;
    f.peer = 0; f.G_local = G; f.stop_nonfinite = 0;
    finalize_block(f, threadIdx.x, sh);
}

// rec[2] = beta, rec[3] = 1/beta (start of a batch of device-chained Lanczos steps); *stop = 0
__global__ void k_lanczos_seed(double* rec, double beta, int* stop) {
    rec[2] = beta;
    rec[3] = 1.0 / beta;
    rec[4] = beta * beta;
    *stop = 0;
}

// Records of a chained GKL step i (b2k_gkl_expand_many), rec_i = d_steps + B2K_REC (i + 1), rec_{-1} the seed:
//   [2] beta_i  [3] 1/beta_i  [4] beta_i^2          (the U sweep's finaliser; [0], [1] unused)
//   [5] alpha_i [6] 1/alpha_i [7] alpha_i^2         (the A' SpMV's norm epilogue, or the V sweep's finaliser at rec + 3)
// Step i ran and was the last one to run when alpha_i or beta_i is not finite or beta_i <= tol: the flags the kernels
// raise, read back from the records.
__device__ __host__ inline bool gkl_step_stops(const double* rec, double tol) {
    return !isfinite(rec[5]) || !isfinite(rec[2]) || rec[2] <= tol;
}

struct GklFlush {
    const double* rec0;
    double tol;
    int nsteps;
    int64_t ld, n;
    int32_t col[B2K_MAX_CHAIN];     // V column of step i
};

// The flush launch of a chained GKL batch: the last step that ran leaves its v~ unnormalised (the next step's A'
// SpMV would have normalised it), so v = rn(v~ * (1/alpha)) here, whether or not the chain stopped early.
template <typename T>
__global__ void __launch_bounds__(256) k_gkl_flush(T* base, const __grid_constant__ GklFlush f) {
    __shared__ int last;
    if (threadIdx.x == 0) {
        int i = 0;
        while (i + 1 < f.nsteps && !gkl_step_stops(f.rec0 + (size_t)B2K_REC * (i + 1), f.tol)) ++i;
        last = i;
    }
    __syncthreads();
    const T s = (T)f.rec0[(size_t)B2K_REC * (last + 1) + 6];
    T* v = base + (int64_t)f.col[last] * f.ld;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < f.n; r += (int64_t)gridDim.x * blockDim.x)
        v[r] = v[r] * s;
}

// out[j] = (T) res[j]  (dense adjoint: projection coefficients become a device vector)
template <typename T>
__global__ void k_res_to_vec(const double* __restrict__ res, T* __restrict__ out, int k,
                             T alpha) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < k) out[j] = alpha * (T)res[j];
}

// basistransform!: cols[0..keep) <- Q[:, cols[0..m)] * U, in place, tile resident in the ring
struct TransformParams {
    void* base;
    int64_t ld, n;
    int32_t m, keep, ldu;
    const double* U;     // device, column-major m x keep
    int32_t u_in_smem;
};

constexpr int TR_OFF_U = NS * SLOT_BYTES;                 // after the ring
constexpr int TR_U_BYTES = 232448 - TR_OFF_U - 256;       // bytes available for U
constexpr int TR_OFF_BAR = TR_OFF_U + TR_U_BYTES;
constexpr int TR_SMEM = TR_OFF_BAR + 2 * NS * 8;
constexpr int TJ = 36;
constexpr int TR_THREADS = NCONS + 32;   // 8 consumer warps + ONE producer warp (compute-bound kernel)   // output columns accumulated in registers per pass over the resident tile

// Consumers: thread <-> row, TJ accumulators per thread; U row-major in shared memory
// (Us[i*pitch + j]), read as broadcast 128-bit loads: 0.5 LDS per FMA, Q read once per pass.
template <typename T, bool USM>
__global__ void __launch_bounds__(TR_THREADS, 1)
k_transform(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    using CF = Cfg<T>;
    using V16 = typename CF::V16;
    constexpr int R = CF::R, C = CF::C, VEC = CF::VEC;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TR_OFF_BAR), empty = full + NS * 8;
    T* Us = reinterpret_cast<T*>(smem + TR_OFF_U);
    const int pitch = ((p.keep + VEC - 1) / VEC) * VEC;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, NCONS / 32);
        }
        fence_mbar_init();
    }
    if (USM)
        for (int idx = threadIdx.x; idx < p.m * pitch; idx += blockDim.x) {
            const int i = idx / pitch, j = idx - i * pitch;
            Us[idx] = (j < p.keep) ? (T)p.U[(size_t)j * p.ldu + i] : (T)0;
        }
    __syncthreads();
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    T* base = reinterpret_cast<T*>(p.base);
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= NCONS) {
        const int lane = threadIdx.x & 31;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t bytes = (uint32_t)((rt * sizeof(T) + 15) & ~(size_t)15);
            for (int c = 0; c < nch; ++c) {
                mbar_wait(empty + 8 * s, ph ^ 1);
                const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
                if (lane == 0) mbar_expect_tx(full + 8 * s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol)
                    bulk_g2s(ring + s * SLOT_BYTES + lane * R * (int)sizeof(T),
                             base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes, full + 8 * s);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        }
    } else {
        const int tid = threadIdx.x, lane = tid & 31;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t s0 = s;
            for (int c = 0; c < nch; ++c) {   // the whole row tile must be resident
                mbar_wait(full + 8 * s, ph);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
            // thread -> two rows (rp, rp + R/2) x one half of the TJ outputs of this pass: each
            // U value fetched from shared memory feeds two FMAs (22 instead of 38 smem
            // wavefronts per basis vector and warp)
            constexpr int TJT = (sizeof(T) == 8) ? TJ : 40;   // outputs per pass; TJT/2 % VEC == 0
            constexpr int TH = TJT / 2;
            static_assert(TH % VEC == 0, "half-pass width must keep the 128-bit U loads aligned");
            const int half = tid >> 7, rp = tid & 127;
            for (int jb = 0; jb < p.keep; jb += TJT) {
                const int nj = (p.keep - jb) < TJT ? (p.keep - jb) : TJT;
                const int njh = nj - half * TH;          // valid outputs of my half (may be <= 0)
                T acc0[TH], acc1[TH];
#pragma unroll
                for (int t = 0; t < TH; ++t) { acc0[t] = (T)0; acc1[t] = (T)0; }
                uint32_t ss = s0;
                for (int c = 0; c < nch; ++c) {
                    const T* slot = reinterpret_cast<const T*>(smem + ss * SLOT_BYTES);
                    const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
                    for (int jj = 0; jj < ncol; ++jj) {
                        const T q0 = slot[jj * R + rp], q1 = slot[jj * R + rp + R / 2];
                        const int i = c * C + jj;
                        if (USM) {
                            const T* urow = Us + i * pitch + jb + half * TH;
#pragma unroll
                            for (int t = 0; t < TH; t += VEC) {
                                if (t < njh) {
                                    T u[VEC];
                                    CF::unpack(*reinterpret_cast<const V16*>(urow + t), u);
#pragma unroll
                                    for (int e = 0; e < VEC; ++e) {
                                        acc0[t + e] = fma(q0, u[e], acc0[t + e]);
                                        acc1[t + e] = fma(q1, u[e], acc1[t + e]);
                                    }
                                }
                            }
                        } else {
#pragma unroll
                            for (int t = 0; t < TH; ++t)
                                if (t < njh) {
                                    const T u = (T)__ldg(p.U + (size_t)(jb + half * TH + t) * p.ldu + i);
                                    acc0[t] = fma(q0, u, acc0[t]);
                                    acc1[t] = fma(q1, u, acc1[t]);
                                }
                        }
                    }
                    if (++ss == NS) ss = 0;
                }
#pragma unroll
                for (int t = 0; t < TH; ++t)
                    if (t < njh) {
                        T* col = base + (int64_t)cl.c[jb + half * TH + t] * p.ld + r0;
                        if (rp < rt) col[rp] = acc0[t];
                        if (rp + R / 2 < rt) col[rp + R / 2] = acc1[t];
                    }
            }
            // release the tile
            uint32_t ss = s0;
            __syncwarp();
            for (int c = 0; c < nch; ++c) {
                if (lane == 0) mbar_arrive(empty + 8 * ss);
                if (++ss == NS) ss = 0;
            }
        }
    }
}

// basistransform! for bases wider than the resident ring (NS*C < m <= 256; the BlockLanczos default
// krylovdim = 100 lands here).  Still one pass over the basis and in place: a TB_ROWS-row tile of all m
// columns is staged in shared memory with plain coalesced loads, every thread then owns one row and
// TB_J outputs per sweep, reading U (L1-resident, warp-uniform address) straight from global memory.
// Sums run over i in increasing order with fma, like k_transform.
constexpr int TB_ROWS = 64;
constexpr int TB_THREADS = 256;
constexpr int TB_J = 8;                                   // outputs per thread and sweep
constexpr int TB_GROUPS = TB_THREADS / TB_ROWS;           // 4 output groups -> 32 outputs per sweep
constexpr int TB_SMEM_MAX = TB_ROWS * 256 * 8;            // 128 KB at m = 256, f64

template <typename T>
__global__ void __launch_bounds__(TB_THREADS)
k_transform_big(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    extern __shared__ __align__(16) uint8_t smem[];
    T* Qs = reinterpret_cast<T*>(smem);                   // Qs[i * TB_ROWS + r]
    T* base = reinterpret_cast<T*>(p.base);
    const int64_t ntiles = (p.n + TB_ROWS - 1) / TB_ROWS;
    const int r = threadIdx.x % TB_ROWS, g = threadIdx.x / TB_ROWS;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * TB_ROWS;
        for (int idx = threadIdx.x; idx < p.m * TB_ROWS; idx += TB_THREADS) {
            const int i = idx / TB_ROWS, rr = idx - i * TB_ROWS;
            Qs[idx] = (r0 + rr < p.n) ? base[(int64_t)cl.c[i] * p.ld + r0 + rr] : (T)0;
        }
        __syncthreads();
        for (int jb = g * TB_J; jb < p.keep; jb += TB_GROUPS * TB_J) {
            const double* ucol[TB_J];
#pragma unroll
            for (int t = 0; t < TB_J; ++t) {
                const int j = (jb + t < p.keep) ? (jb + t) : (p.keep - 1);   // clamp: no branch in the i loop
                ucol[t] = p.U + (size_t)j * p.ldu;
            }
            T acc[TB_J];
#pragma unroll
            for (int t = 0; t < TB_J; ++t) acc[t] = (T)0;
            for (int i = 0; i < p.m; ++i) {
                const T q = Qs[i * TB_ROWS + r];
#pragma unroll
                for (int t = 0; t < TB_J; ++t) acc[t] = fma(q, (T)__ldg(ucol[t] + i), acc[t]);
            }
            if (r0 + r < p.n) {
#pragma unroll
                for (int t = 0; t < TB_J; ++t)
                    if (jb + t < p.keep) base[(int64_t)cl.c[jb + t] * p.ld + r0 + r] = acc[t];
            }
        }
        __syncthreads();                                  // tile fully consumed before it is overwritten
    }
}

// FP64 tensor-core variant of the restart GEMM (double, U resident in shared memory):
// mma.sync.aligned.m8n8k4.f64 (DMMA).  Warp w owns rows [32w, 32w+32) of the resident tile as
// four 8-row blocks; outputs are produced 40 columns (five 8-column blocks) per pass; the k loop
// walks the basis vectors 4 at a time.  Per k-step a warp loads 4 A fragments + 5 B fragments
// (9 LDS.64) for 20 DMMAs = 5120 FMAs: shared-memory traffic per FMA drops 5x vs the FMA kernel,
// which is bound by the shared-memory broadcast loads of U (two wavefronts per double).
// Column pitch in the ring is R+8 doubles (== 64 mod 128 bytes) so the four columns of an A
// fragment hit two disjoint bank halves: 2 wavefronts per LDS.64, the minimum.
constexpr int TD_PITCH = 256 + 8;                         // doubles per staged column
constexpr int TD_SLOT = 8 * TD_PITCH * 8;                 // 16896 bytes per ring slot
constexpr int TD_OFF_U = NS * TD_SLOT;                    // 202752
constexpr int TD_U_BYTES = 232448 - TD_OFF_U - 256;       // 29440
constexpr int TD_OFF_BAR = TD_OFF_U + TD_U_BYTES;
constexpr int TD_SMEM = TD_OFF_BAR + 2 * NS * 8;
constexpr int TD_NCB = 5;                                 // 8-column output blocks per pass

__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(TR_THREADS, 1)
k_transform_dmma(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    constexpr int R = 256, C = 8;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TD_OFF_BAR), empty = full + NS * 8;
    double* Us = reinterpret_cast<double*>(smem + TD_OFF_U);
    const int pitch = ((p.keep + 7) / 8) * 8;             // zero-padded to whole 8-column blocks
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, NCONS / 32);
        }
        fence_mbar_init();
    }
    for (int idx = threadIdx.x; idx < p.m * pitch; idx += blockDim.x) {
        const int i = idx / pitch, j = idx - i * pitch;
        Us[idx] = (j < p.keep) ? p.U[(size_t)j * p.ldu + i] : 0.0;
    }
    __syncthreads();
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    double* base = reinterpret_cast<double*>(p.base);
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= NCONS) {
        const int lane = threadIdx.x & 31;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t bytes = (uint32_t)((rt * sizeof(double) + 15) & ~(size_t)15);
            for (int c = 0; c < nch; ++c) {
                mbar_wait(empty + 8 * s, ph ^ 1);
                const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
                if (lane == 0) mbar_expect_tx(full + 8 * s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol)
                    bulk_g2s(ring + s * TD_SLOT + lane * TD_PITCH * 8,
                             base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes, full + 8 * s);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        const bool streaming = p.keep <= 8 * TD_NCB;   // one pass: consume and release chunks as they land
        const uint32_t s0 = s;
        if (!streaming) {
            for (int c = 0; c < nch; ++c) {   // several passes: the whole row tile must be resident
                mbar_wait(full + 8 * s, ph);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        }
        for (int jb = 0; jb < p.keep; jb += 8 * TD_NCB) {
            const int ncb = ((p.keep - jb + 7) / 8) < TD_NCB ? ((p.keep - jb + 7) / 8) : TD_NCB;
            double acc[4][TD_NCB][2];
#pragma unroll
            for (int rb = 0; rb < 4; ++rb)
#pragma unroll
                for (int cb = 0; cb < TD_NCB; ++cb) { acc[rb][cb][0] = 0.0; acc[rb][cb][1] = 0.0; }
            uint32_t ss = s0;
            for (int c = 0; c < nch; ++c) {
                if (streaming) {
                    mbar_wait(full + 8 * s, ph);
                    ss = s;
                }
                const double* slot = reinterpret_cast<const double*>(smem + ss * TD_SLOT);
                const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) {
                    const int k0 = ks * 4;
                    if (k0 < ncol) {
                        const bool kv = (k0 + t) < ncol;          // tail of the last chunk: zero operands
                        double a[4], b[TD_NCB];
#pragma unroll
                        for (int rb = 0; rb < 4; ++rb) {
                            const int row = 32 * w + 8 * rb + g;
                            // rows >= rt hold stale (possibly non-finite) data: zero them
                            a[rb] = (kv && row < rt) ? slot[(k0 + t) * TD_PITCH + row] : 0.0;
                        }
                        const double* urow = Us + (size_t)(c * C + k0 + t) * pitch + jb + g;
#pragma unroll
                        for (int cb = 0; cb < TD_NCB; ++cb) b[cb] = (kv && cb < ncb) ? urow[cb * 8] : 0.0;
#pragma unroll
                        for (int rb = 0; rb < 4; ++rb)
#pragma unroll
                            for (int cb = 0; cb < TD_NCB; ++cb)
                                if (cb < ncb) dmma884(acc[rb][cb][0], acc[rb][cb][1], a[rb], b[cb]);
                    }
                }
                if (streaming) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty + 8 * s);
                    if (++s == NS) { s = 0; ph ^= 1; }
                } else if (++ss == NS) ss = 0;
            }
#pragma unroll
            for (int rb = 0; rb < 4; ++rb) {
                const int row = 32 * w + 8 * rb + g;
#pragma unroll
                for (int cb = 0; cb < TD_NCB; ++cb) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = jb + cb * 8 + 2 * t + e;
                        if (cb < ncb && col < p.keep && row < rt)
                            base[(int64_t)cl.c[col] * p.ld + r0 + row] = acc[rb][cb][e];
                    }
                }
            }
        }
        if (streaming) continue;
        uint32_t ss = s0;
        __syncwarp();
        for (int c = 0; c < nch; ++c) {
            if (lane == 0) mbar_arrive(empty + 8 * ss);
            if (++ss == NS) ss = 0;
        }
    }
}

// Pure-DFMA restart GEMM with an 8 x 9 register tile: the alternative to the DMMA kernel that feeds the FP64 FMA
// pipe instead of the tensor cores, for which the rate of each pipe is not what decides — the operands must be
// delivered fast enough.  Which of the two is faster on a given part is an A/B of B2K_TRANSFORM_HYB.  The operand costs are
// LSU cycles: a row value is an LDS.128 per two rows (2 cycles per double), a U value a broadcast (2 cycles per
// double).  thread <-> 8 rows x 9 outputs: 16 + 18 = 34 LSU cycles per 72 warp-DFMAs (144 pipe cycles) and warp, where
// k_transform's 2 x 18 tile spent 40 per 36.  U sits in shared memory as [group][i][10] (9 outputs + pad: 16-byte
// aligned rows for the broadcast LDS.128).  keep <= 36: one pass, chunks consumed and released as they land.
//
// Warps: a 256-row tile is covered by FOUR warps (32 lanes x 8 rows, 4 column groups).  The first version ran those
// four + a producer warp per CTA and was issue-bound (`stall_wait` dominant): ONE warp per scheduler cannot issue
// DFMAs back to back.
// Registers are granted per four warps (8 x 32 x 255 = the whole file), so a ninth (producer) warp is not affordable:
// here EIGHT consumer warps work as two sets on alternate tiles of the SAME FIFO ring (set 1 trails set 0 by half a
// tile), and the TMA refill of a slot is issued by the first warp of the set that just consumed it (chunk g + NS goes
// into the slot of chunk g; dependencies only point backwards in g, so the two sets cannot deadlock each other).
constexpr int F89_G = 4, F89_TH = 9, F89_UP = 10;         // column groups, outputs per group, padded row of U
constexpr int F89_THREADS = 256;                          // two sets of four warps

__global__ void __launch_bounds__(F89_THREADS, 1)
k_transform_f89(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    constexpr int R = 256, C = 8;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TR_OFF_BAR), empty = full + NS * 8;
    double* Us = reinterpret_cast<double*>(smem + TR_OFF_U);
    // uses[s] = how many loads have been posted to slot s.  A set skips the uses of a slot that belong to the other
    // set's tiles, and an mbarrier wait only knows a phase PARITY: waiting for use u while use u - 1 has not landed
    // yet would return at once (parity of the unfinished phase u - 1 != parity u).  So a consumer first waits until
    // the load of ITS use has been posted (the barrier is then in phase u or beyond) and only then on the parity.
    volatile int* uses = reinterpret_cast<volatile int*>(smem + TR_OFF_U + TR_U_BYTES - 64);
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, F89_G);              // the four warps of the set that consumes the chunk
            uses[i] = 0;
        }
        fence_mbar_init();
    }
    for (int idx = threadIdx.x; idx < F89_G * p.m * F89_UP; idx += blockDim.x) {
        const int gq = idx / (p.m * F89_UP), rem = idx - gq * p.m * F89_UP;
        const int i = rem / F89_UP, t = rem - i * F89_UP;
        const int j = gq * F89_TH + t;
        Us[idx] = (t < F89_TH && j < p.keep) ? p.U[(size_t)j * p.ldu + i] : 0.0;
    }
    __syncthreads();
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    const int64_t my_tiles = (int64_t)blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total_chunks = my_tiles * nch;
    double* base = reinterpret_cast<double*>(p.base);
    const int tid = threadIdx.x, lane = tid & 31, cg = (tid >> 5) & 3, set = tid >> 7;
    // chunk g (tile g / nch of this CTA, columns 8 (g % nch) ...) -> ring slot g % NS; issued by one whole warp
    auto issue = [&](int64_t g) {
        const int64_t tl = g / nch;
        const int c = (int)(g - tl * nch);
        const int64_t r0 = ((int64_t)blockIdx.x + tl * gridDim.x) * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        const uint32_t bytes = (uint32_t)((rt * sizeof(double) + 15) & ~(size_t)15);
        const uint32_t sl = (uint32_t)(g % NS);
        const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
        if (lane == 0) {
            mbar_expect_tx(full + 8 * sl, bytes * (uint32_t)ncol);
            __threadfence_block();
            uses[sl] = (int)(g / NS) + 1;
        }
        __syncwarp();
        if (lane < ncol)
            bulk_g2s(ring + sl * SLOT_BYTES + lane * R * 8, base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes,
                     full + 8 * sl);
    };
    if (tid < 32)
        for (int64_t g = 0; g < NS && g < total_chunks; ++g) issue(g);
    const double* ug = Us + (size_t)cg * p.m * F89_UP;    // my group's U rows
    for (int64_t tl = set; tl < my_tiles; tl += 2) {
        const int64_t r0 = ((int64_t)blockIdx.x + tl * gridDim.x) * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        double acc[8][F89_TH];
#pragma unroll
        for (int e = 0; e < 8; ++e)
#pragma unroll
            for (int t = 0; t < F89_TH; ++t) acc[e][t] = 0.0;
        for (int c = 0; c < nch; ++c) {
            const int64_t g = tl * nch + c;
            const uint32_t sl = (uint32_t)(g % NS), ph = (uint32_t)((g / NS) & 1);
            while (uses[sl] < (int)(g / NS) + 1) {}       // my use of the slot has been posted (see `uses`)
            mbar_wait(full + 8 * sl, ph);
            const double* slot = reinterpret_cast<const double*>(smem + sl * SLOT_BYTES) + 2 * lane;
            const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
            const double* urow = ug + (size_t)c * C * F89_UP;
#pragma unroll 2
            for (int jj = 0; jj < ncol; ++jj) {
                double q[8];
#pragma unroll
                for (int e = 0; e < 4; ++e) {             // rows 2 lane, 2 lane + 1 (+ 64 e)
                    const double2 v = *reinterpret_cast<const double2*>(slot + jj * R + 64 * e);
                    q[2 * e] = v.x; q[2 * e + 1] = v.y;
                }
                double u[F89_UP];
#pragma unroll
                for (int t = 0; t < F89_UP; t += 2) {
                    const double2 v = *reinterpret_cast<const double2*>(urow + jj * F89_UP + t);
                    u[t] = v.x; u[t + 1] = v.y;
                }
#pragma unroll
                for (int t = 0; t < F89_TH; ++t)
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[e][t] = fma(q[e], u[t], acc[e][t]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + 8 * sl);
            if (cg == 0 && g + NS < total_chunks) {       // refill the slot this set has just consumed
                mbar_wait(empty + 8 * sl, ph);
                issue(g + NS);
            }
        }
#pragma unroll
        for (int t = 0; t < F89_TH; ++t) {
            const int j = cg * F89_TH + t;
            if (j < p.keep) {
                double* col = base + (int64_t)cl.c[j] * p.ld + r0 + 2 * lane;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int row = 2 * lane + 64 * e;
                    if (row + 1 < rt) *reinterpret_cast<double2*>(col + 64 * e) = make_double2(acc[2 * e][t], acc[2 * e + 1][t]);
                    else if (row < rt) col[64 * e] = acc[2 * e][t];
                }
            }
        }
    }
}

// The 8 x 9 DFMA tile on 512-row tiles: both warp sets consume the SAME chunk (4 basis columns x 512 rows, still one
// 16 KB slot; set 0 takes rows 0..255, set 1 rows 256..511), so every load keeps the full 12-slot lead of the FIFO.
// (With the sets on alternate 256-row tiles the lead at a tile switch is only 3-4 chunks of that set's time, and the
// consumers wait on the `full` barrier.)
constexpr int F89W_R = 512, F89W_C = 4;

__global__ void __launch_bounds__(F89_THREADS, 1)
k_transform_f89w(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    constexpr int R = F89W_R, C = F89W_C;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TR_OFF_BAR), empty = full + NS * 8;
    double* Us = reinterpret_cast<double*>(smem + TR_OFF_U);
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, F89_THREADS / 32);   // all eight warps consume every chunk
        }
        fence_mbar_init();
    }
    for (int idx = threadIdx.x; idx < F89_G * p.m * F89_UP; idx += blockDim.x) {
        const int gq = idx / (p.m * F89_UP), rem = idx - gq * p.m * F89_UP;
        const int i = rem / F89_UP, t = rem - i * F89_UP;
        const int j = gq * F89_TH + t;
        Us[idx] = (t < F89_TH && j < p.keep) ? p.U[(size_t)j * p.ldu + i] : 0.0;
    }
    __syncthreads();
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    const int64_t my_tiles = (int64_t)blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total_chunks = my_tiles * nch;
    double* base = reinterpret_cast<double*>(p.base);
    const int tid = threadIdx.x, lane = tid & 31, cg = (tid >> 5) & 3, set = tid >> 7;
    auto issue = [&](int64_t g) {                         // one whole warp
        const int64_t tl = g / nch;
        const int c = (int)(g - tl * nch);
        const int64_t r0 = ((int64_t)blockIdx.x + tl * gridDim.x) * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        const uint32_t bytes = (uint32_t)((rt * sizeof(double) + 15) & ~(size_t)15);
        const uint32_t sl = (uint32_t)(g % NS);
        const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
        if (lane == 0) mbar_expect_tx(full + 8 * sl, bytes * (uint32_t)ncol);
        __syncwarp();
        if (lane < ncol)
            bulk_g2s(ring + sl * SLOT_BYTES + lane * R * 8, base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes,
                     full + 8 * sl);
    };
    if (tid < 32)
        for (int64_t g = 0; g < NS && g < total_chunks; ++g) issue(g);
    const double* ug = Us + (size_t)cg * p.m * F89_UP;
    int64_t g = 0;
    for (int64_t tl = 0; tl < my_tiles; ++tl) {
        const int64_t r0 = ((int64_t)blockIdx.x + tl * gridDim.x) * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        double acc[8][F89_TH];
#pragma unroll
        for (int e = 0; e < 8; ++e)
#pragma unroll
            for (int t = 0; t < F89_TH; ++t) acc[e][t] = 0.0;
        for (int c = 0; c < nch; ++c, ++g) {
            const uint32_t sl = (uint32_t)(g % NS), ph = (uint32_t)((g / NS) & 1);
            mbar_wait(full + 8 * sl, ph);
            const double* slot = reinterpret_cast<const double*>(smem + sl * SLOT_BYTES) + 256 * set + 2 * lane;
            const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
            const double* urow = ug + (size_t)c * C * F89_UP;
#pragma unroll 2
            for (int jj = 0; jj < ncol; ++jj) {
                double q[8];
#pragma unroll
                for (int e = 0; e < 4; ++e) {             // rows 256 set + 2 lane, + 1 (+ 64 e)
                    const double2 v = *reinterpret_cast<const double2*>(slot + jj * R + 64 * e);
                    q[2 * e] = v.x; q[2 * e + 1] = v.y;
                }
                double u[F89_UP];
#pragma unroll
                for (int t = 0; t < F89_UP; t += 2) {
                    const double2 v = *reinterpret_cast<const double2*>(urow + jj * F89_UP + t);
                    u[t] = v.x; u[t + 1] = v.y;
                }
#pragma unroll
                for (int t = 0; t < F89_TH; ++t)
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[e][t] = fma(q[e], u[t], acc[e][t]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + 8 * sl);
            if (tid < 32 && g + NS < total_chunks) {      // warp 0 refills the slot once all eight warps are done with it
                mbar_wait(empty + 8 * sl, ph);
                issue(g + NS);
            }
        }
#pragma unroll
        for (int t = 0; t < F89_TH; ++t) {
            const int j = cg * F89_TH + t;
            if (j < p.keep) {
                double* col = base + (int64_t)cl.c[j] * p.ld + r0 + 256 * set + 2 * lane;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int row = 256 * set + 2 * lane + 64 * e;
                    if (row + 1 < rt) *reinterpret_cast<double2*>(col + 64 * e) = make_double2(acc[2 * e][t], acc[2 * e + 1][t]);
                    else if (row < rt) col[64 * e] = acc[2 * e][t];
                }
            }
        }
    }
}

// Hybrid restart GEMM: DMMA and DFMA at once.  k_transform_dmma keeps only the pipe `DMMA.8x8x4` issues through busy
// while the DFMA pipe idles; a DFMA-only kernel is bound by the
// shared-memory broadcast of U (2 LSU cycles per double).  Here every consumer warp does both per staged chunk: output
// columns [0, 24) as three 8-column DMMA blocks for its 32 rows (14 smem wavefronts per 3072 FMA), columns [24, 36) as
// register-blocked DFMA — warp <-> 64 rows x 6 columns, lane <-> 2 rows, 12 accumulators, 16 wavefronts per 384 FMA.
// Budget per 256-row tile (60 -> 36): DMMA 12 300 clk, DFMA 2 900 clk/SMSP, LSU 9 400 wavefronts, HBM 8 500 clk.
// keep <= 36 only (one pass, chunks consumed and released as they land); wider restarts use k_transform_dmma.
constexpr int TH_DCB = 3;                                 // DMMA column blocks: columns [0, 24)
constexpr int TH_DF0 = 8 * TH_DCB;                        // first DFMA column
constexpr int TH_DFW = 6;                                 // DFMA columns per warp (two warp groups: 12 columns)
constexpr int TH_MAXKEEP = TH_DF0 + 2 * TH_DFW;           // 36

__global__ void __launch_bounds__(TR_THREADS, 1)
k_transform_hyb(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl) {
    constexpr int R = 256, C = 8;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TD_OFF_BAR), empty = full + NS * 8;
    double* Us = reinterpret_cast<double*>(smem + TD_OFF_U);
    constexpr int pitch = 40;                             // U rows zero-padded to 40 columns
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, NCONS / 32);
        }
        fence_mbar_init();
    }
    for (int idx = threadIdx.x; idx < p.m * pitch; idx += blockDim.x) {
        const int i = idx / pitch, j = idx - i * pitch;
        Us[idx] = (j < p.keep) ? p.U[(size_t)j * p.ldu + i] : 0.0;
    }
    __syncthreads();
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    double* base = reinterpret_cast<double*>(p.base);
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= NCONS) {
        const int lane = threadIdx.x & 31;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t bytes = (uint32_t)((rt * sizeof(double) + 15) & ~(size_t)15);
            for (int c = 0; c < nch; ++c) {
                mbar_wait(empty + 8 * s, ph ^ 1);
                const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
                if (lane == 0) mbar_expect_tx(full + 8 * s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol)
                    bulk_g2s(ring + s * TD_SLOT + lane * TD_PITCH * 8,
                             base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes, full + 8 * s);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int ncb = ((p.keep + 7) / 8) < TH_DCB ? ((p.keep + 7) / 8) : TH_DCB;
    const int frow = 64 * (w & 3) + lane;                 // DFMA rows frow, frow + 32
    const int fcol = TH_DF0 + TH_DFW * (w >> 2);          // DFMA columns fcol .. fcol + 5
    const bool df_on = fcol < p.keep;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        double acc[4][TH_DCB][2];
        double fa[2][TH_DFW];
#pragma unroll
        for (int rb = 0; rb < 4; ++rb)
#pragma unroll
            for (int cb = 0; cb < TH_DCB; ++cb) { acc[rb][cb][0] = 0.0; acc[rb][cb][1] = 0.0; }
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int u = 0; u < TH_DFW; ++u) fa[e][u] = 0.0;
        for (int c = 0; c < nch; ++c) {
            mbar_wait(full + 8 * s, ph);
            const double* slot = reinterpret_cast<const double*>(smem + s * TD_SLOT);
            const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const int k0 = ks * 4;
                if (k0 < ncol) {
                    const bool kv = (k0 + t) < ncol;          // tail of the last chunk: zero operands
                    double a[4], b[TH_DCB];
#pragma unroll
                    for (int rb = 0; rb < 4; ++rb) {
                        const int row = 32 * w + 8 * rb + g;
                        a[rb] = (kv && row < rt) ? slot[(k0 + t) * TD_PITCH + row] : 0.0;   // stale rows: zero
                    }
                    const double* urow = Us + (size_t)(c * C + k0 + t) * pitch + g;
#pragma unroll
                    for (int cb = 0; cb < TH_DCB; ++cb) b[cb] = (kv && cb < ncb) ? urow[cb * 8] : 0.0;
#pragma unroll
                    for (int rb = 0; rb < 4; ++rb)
#pragma unroll
                        for (int cb = 0; cb < TH_DCB; ++cb)
                            if (cb < ncb) dmma884(acc[rb][cb][0], acc[rb][cb][1], a[rb], b[cb]);
                    // the DFMA share of the same four basis vectors (sums over i in increasing order)
                    if (df_on) {
#pragma unroll
                        for (int kk = 0; kk < 4; ++kk) {
                            if (k0 + kk < ncol) {
                                const double q0 = slot[(k0 + kk) * TD_PITCH + frow];
                                const double q1 = slot[(k0 + kk) * TD_PITCH + frow + 32];
                                const double2* uf = reinterpret_cast<const double2*>(
                                    Us + (size_t)(c * C + k0 + kk) * pitch + fcol);
#pragma unroll
                                for (int u = 0; u < TH_DFW / 2; ++u) {
                                    const double2 uu = uf[u];
                                    fa[0][2 * u] = fma(q0, uu.x, fa[0][2 * u]);
                                    fa[1][2 * u] = fma(q1, uu.x, fa[1][2 * u]);
                                    fa[0][2 * u + 1] = fma(q0, uu.y, fa[0][2 * u + 1]);
                                    fa[1][2 * u + 1] = fma(q1, uu.y, fa[1][2 * u + 1]);
                                }
                            }
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + 8 * s);
            if (++s == NS) { s = 0; ph ^= 1; }
        }
#pragma unroll
        for (int rb = 0; rb < 4; ++rb) {
            const int row = 32 * w + 8 * rb + g;
#pragma unroll
            for (int cb = 0; cb < TH_DCB; ++cb) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = cb * 8 + 2 * t + e;
                    if (cb < ncb && col < p.keep && row < rt)
                        base[(int64_t)cl.c[col] * p.ld + r0 + row] = acc[rb][cb][e];
                }
            }
        }
        if (df_on) {
#pragma unroll
            for (int u = 0; u < TH_DFW; ++u) {
                if (fcol + u < p.keep) {
                    double* col = base + (int64_t)cl.c[fcol + u] * p.ld + r0;
                    if (frow < rt) col[frow] = fa[0][u];
                    if (frow + 32 < rt) col[frow + 32] = fa[1][u];
                }
            }
        }
    }
}

// FP64 restart GEMM on the DFMA pipe with U in the constant bank (an alternative to the DMMA kernel).  The FMA
// kernel above starves the DFMA pipe on the shared-memory broadcast of U (two wavefronts per double).  Here U travels as
// a kernel parameter: a warp-uniform constant index compiles to `LDCU.64 URx, c[0x0][UR+imm]` + `DFMA R, R, URx, R`
// (cuobjdump -sass), so U costs no LSU wavefront at all and shared memory only serves the ROWS LDS.64 of Q per
// basis vector.  thread <-> ROWS rows x TH outputs; keep <= 36 is one pass, so chunks are consumed and released as
// they land (TMA overlaps the arithmetic).  Sums run over i in increasing order with fma: the same bits as
// k_transform.
constexpr int UR_J = 36;                                  // outputs per pass == row pitch of U in the parameter
constexpr int UR_MAXM = 96;                               // NS * 8 basis vectors
struct UPar {
    double u[UR_MAXM * UR_J];                             // u[i * UR_J + j], zero-padded to UR_J columns (27 KB)
};

template <int ROWS, int TH, int HOFF>
__device__ __forceinline__ void ur_consume(const UPar& U, const TransformParams& p, const ColList& cl,
                                           const uint8_t* smem, uint32_t full, uint32_t empty, uint32_t& s,
                                           uint32_t& ph, int rp, int lane) {
    constexpr int R = 256, C = 8, RS = R / ROWS;
    const int nch = (p.m + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    double* base = reinterpret_cast<double*>(p.base);
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        double acc[ROWS][TH];
#pragma unroll
        for (int e = 0; e < ROWS; ++e)
#pragma unroll
            for (int t = 0; t < TH; ++t) acc[e][t] = 0.0;
        for (int c = 0; c < nch; ++c) {
            mbar_wait(full + 8 * s, ph);
            const double* slot = reinterpret_cast<const double*>(smem + s * SLOT_BYTES) + rp;
            const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
            const double* urow = U.u + c * C * UR_J + HOFF;
            if (ncol == C) {
#pragma unroll
                for (int jj = 0; jj < C; ++jj) {
                    double q[ROWS];
#pragma unroll
                    for (int e = 0; e < ROWS; ++e) q[e] = slot[jj * R + e * RS];
#pragma unroll
                    for (int t = 0; t < TH; ++t) {
                        const double u = urow[jj * UR_J + t];
#pragma unroll
                        for (int e = 0; e < ROWS; ++e) acc[e][t] = fma(q[e], u, acc[e][t]);
                    }
                }
            } else {
                for (int jj = 0; jj < ncol; ++jj) {
                    double q[ROWS];
#pragma unroll
                    for (int e = 0; e < ROWS; ++e) q[e] = slot[jj * R + e * RS];
#pragma unroll
                    for (int t = 0; t < TH; ++t) {
                        const double u = urow[jj * UR_J + t];
#pragma unroll
                        for (int e = 0; e < ROWS; ++e) acc[e][t] = fma(q[e], u, acc[e][t]);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + 8 * s);
            if (++s == NS) { s = 0; ph ^= 1; }
        }
#pragma unroll
        for (int t = 0; t < TH; ++t)
            if (HOFF + t < p.keep) {
                double* col = base + (int64_t)cl.c[HOFF + t] * p.ld + r0 + rp;
#pragma unroll
                for (int e = 0; e < ROWS; ++e)
                    if (rp + e * RS < rt) col[e * RS] = acc[e][t];
            }
    }
}

template <int ROWS, int TH>
__global__ void __launch_bounds__(TR_THREADS, 1)
k_transform_ur(const __grid_constant__ TransformParams p, const __grid_constant__ ColList cl,
               const __grid_constant__ UPar U) {
    constexpr int R = 256, C = 8, RS = R / ROWS;
    constexpr int NT = RS * (UR_J / TH);                  // consumer threads that have work
    static_assert(UR_J % TH == 0 && NT <= NCONS && NT % 32 == 0, "consumer layout");
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t ring = smem_u32(smem);
    const uint32_t full = smem_u32(smem + TR_OFF_BAR), empty = full + NS * 8;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, NT / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();
    uint32_t s = 0, ph = 0;
    if (threadIdx.x >= NCONS) {
        const int nch = (p.m + C - 1) / C;
        const int64_t ntiles = (p.n + R - 1) / R;
        const double* base = reinterpret_cast<const double*>(p.base);
        const int lane = threadIdx.x & 31;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t bytes = (uint32_t)((rt * sizeof(double) + 15) & ~(size_t)15);
            for (int c = 0; c < nch; ++c) {
                mbar_wait(empty + 8 * s, ph ^ 1);
                const int ncol = (p.m - c * C) < C ? (p.m - c * C) : C;
                if (lane == 0) mbar_expect_tx(full + 8 * s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol)
                    bulk_g2s(ring + s * SLOT_BYTES + lane * R * 8,
                             base + (int64_t)cl.c[c * C + lane] * p.ld + r0, bytes, full + 8 * s);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    if (threadIdx.x >= NT) return;
    const int tid = threadIdx.x, lane = tid & 31, rp = tid % RS;
    // the output group is warp-uniform; dispatching on it keeps every index into U a uniform constant-bank address
    if (UR_J / TH == 1 || tid < RS) ur_consume<ROWS, TH, 0>(U, p, cl, smem, full, empty, s, ph, rp, lane);
    else ur_consume<ROWS, TH, (UR_J / TH == 1 ? 0 : TH)>(U, p, cl, smem, full, empty, s, ph, rp, lane);
}

// rank1update!: b[cols[i]] = beta*b[cols[i]] + (alpha*conj(x[i])) * y   — orthonormal.jl:219-227
struct CoefList {
    double c[256];
};
template <typename T>
__global__ void __launch_bounds__(256)
k_rank1(T* __restrict__ base, int64_t ld, int64_t n, int k, const T* __restrict__ y, T beta,
        int beta_mode, const __grid_constant__ ColList cl, const __grid_constant__ CoefList cf) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += stride) {
        const T yv = y[r];
        for (int i = 0; i < k; ++i) {
            T* col = base + (int64_t)cl.c[i] * ld;
            const T a = (T)cf.c[i];
            if (beta_mode == 1) col[r] = fma(a, yv, col[r]);
            else if (beta_mode == 0) col[r] = a * yv;
            else col[r] = fma(a, yv, beta * col[r]);
        }
    }
}

// ---------------------------------------------------------------- launch helpers ----

template <typename T, bool U, bool P>
int32_t launch_phase_t(b2k_ctx* ctx, const PhaseParams<T>& p, const ColList& cl, int grid) {
    k_phase<T, U, P><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(p, cl);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

template <typename T>
int32_t launch_phase(b2k_ctx* ctx, const PhaseParams<T>& p, const ColList& cl, int kind, int grid) {
    if (kind == 0) return launch_phase_t<T, false, true>(ctx, p, cl, grid);
    if (kind == 1) return launch_phase_t<T, true, true>(ctx, p, cl, grid);
    return launch_phase_t<T, true, false>(ctx, p, cl, grid);
}

template <typename T>
int grid_for_rows(const b2k_ctx* ctx, int64_t n) {
    int64_t ntiles = (n + Cfg<T>::R - 1) / Cfg<T>::R;
    if (ntiles < 1) ntiles = 1;
    return (int)std::min<int64_t>(ntiles, ctx->num_sms);
}

// Does phase `st` store into a vector that phase `rd` streams (its x or one of its panel columns)?
template <typename T>
bool stores_into_stream(const PhaseParams<T>& st, const PhaseParams<T>& rd, const ColList& cl) {
    if (!st.store_x || !st.xout) return false;
    const T* lo = st.xout;
    const T* hi = st.xout + st.n;
    auto hits = [&](const T* v) { return v && v < hi && lo < v + rd.n; };
    if (hits(rd.x)) return true;
    for (int m = 0; m < rd.k; ++m)
        if (hits(rd.base + (int64_t)cl.c[m] * rd.ld)) return true;
    return false;
}

template <typename T>
int32_t launch_fused(b2k_ctx* ctx, FusedParams<T>& fp, const ColList& cl, int grid) {
    // Producers may run through boundary i into phase i + 1 unless a phase up to i stored into a vector phase
    // i + 1 streams: a bulk copy issued before the boundary's fence.proxy.async could read a row its store has
    // not yet reached.
    for (int i = 0; i + 1 < fp.nph; ++i) {
        bool ra = true;
        for (int j = 0; j <= i; ++j) ra = ra && !stores_into_stream<T>(fp.ph[j], fp.ph[i + 1], cl);
        fp.run_ahead[i] = ra ? 1 : 0;
    }
    // the barrier counter only ever increases; wrap-around is handled by the signed compare
    fp.barrier = ctx->d_sync + 1;
    fp.barrier_base = ctx->barrier_base;
    ctx->barrier_base += (unsigned)(fp.nph - 1) * (unsigned)grid;
    void* args[] = {(void*)&fp, (void*)&cl};
    B2K_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)k_gs_fused<T>, dim3(grid), dim3(NTHREADS),
                                              args, SMEM_BYTES, ctx->stream));
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

int32_t enqueue_finalize(b2k_ctx* ctx, const double* A, const double* B, const double* N, int G,
                         int k, int off, int noff) {
    if (k > NCONS) return b2k_fail(ctx, B2K_ENOTSUP, "finalize: more than %d coefficients per pass", NCONS);
    k_finalize<<<1, NCONS, 0, ctx->stream>>>(A, B, N, G, B2K_KSTRIDE, k, ctx->d_res, off, noff);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

bool g_l2_hints = true;      // B2K_L2_HINTS=0 switches the eviction-priority hints off (A/B measurements)

struct Panel {
    void* base;      // space base pointer
    int64_t ld, n;
    int32_t sharded;
    std::vector<int32_t> idx;
};

int32_t make_panel(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, Panel* pn) {
    int32_t sp = 0;
    B2K_TRY(b2k_resolve_cols(ctx, cols, k, &sp, &pn->idx));
    if (k == 0) {
        pn->base = nullptr;
        return B2K_OK;
    }
    const B2kSpace& s = ctx->spaces[sp];
    pn->base = s.base;
    pn->ld = s.ld;
    pn->n = s.n;
    pn->sharded = s.sharded;
    return B2K_OK;
}

template <typename T>
void fill_cols(ColList& cl, const std::vector<int32_t>& idx, int off, int cnt) {
    for (int i = 0; i < cnt; ++i) cl.c[i] = idx[off + i];
}

// Column list of a Lanczos step's sweeps.  With the three-term prologue (PhaseParams::prologue) it is rotated by
// two, [v_prev, v, q_0, ..., q_{K1-3}], so that the prologue's operands are the first chunk of every tile.
void lanczos_cols(ColList& cl, const Panel& pn, int K1, bool prologue) {
    const int rot = prologue ? 2 : 0;
    for (int i = 0; i < K1; ++i) cl.c[(i + rot) % K1] = pn.idx[i];
}

template <typename T>
PhaseParams<T> base_params(const Panel& pn, int k, const void* x, void* xout) {
    PhaseParams<T> p;
    memset(&p, 0, sizeof(p));
    p.base = (const T*)pn.base;
    p.ld = pn.ld;
    p.n = pn.n;
    p.k = k;
    p.x = (const T*)x;
    p.xout = (T*)xout;
    p.beta_mode = 1;
    p.betax = (T)1;
    p.alphac = (T)1;
    p.l2_hints = g_l2_hints ? 1 : 0;
    return p;
}

// The two sweeps of a CGS2 Lanczos step (lanczos.jl:313-324) over the column list of lanczos_cols, as fp.ph[0..1]:
//   A (project): with `prologue`, w' = (w + c1 v_prev) + c2 v; h = V^T w' -> per-CTA partials (part set 0);
//   C (update):  the same prologue; w'' = w' - V h stored in place; ||w''||^2 -> per-CTA partials (part set 2).
// C sums h from A's per-CTA partials; a caller that reduces h elsewhere points C's coefficients there.  The prologue
// reads c1 / c2 from the device when c1_dev / c2_dev are given (PhaseParams).
template <typename T>
void lanczos_sweeps(b2k_ctx* ctx, FusedParams<T>& fp, const Panel& pn, int K1, const VecRef& w, int grid,
                    bool prologue, double c1, double c2, const double* c1_dev, const double* c2_dev) {
    memset(&fp, 0, sizeof(fp));
    PhaseParams<T>& a = fp.ph[0];
    PhaseParams<T>& c = fp.ph[1];
    a = base_params<T>(pn, K1, w.ptr, nullptr);
    c = base_params<T>(pn, K1, w.ptr, w.ptr);
    if (prologue) {
        for (PhaseParams<T>* q : {&a, &c}) {
            q->prologue = 1; q->c1 = (T)c1; q->c2 = (T)c2;
            q->c1_dev = c1_dev; q->c2_dev = c2_dev;
        }
    }
    a.part_h = b2k_part_set(ctx, 0);
    c.store_x = 1; c.coef = a.part_h; c.coef_sets = grid; c.coef_stride = B2K_KSTRIDE;
    c.alphac = (T)-1; c.part_n = b2k_part_set(ctx, 2);
    fp.kind[0] = 0; fp.kind[1] = 2; fp.nph = 2;
}

// ------------------------------------------------------------------------------------
// project: d_res[0..k) = Q^T x   (all passes), single-GPU or dist (allreduce by caller)
// ------------------------------------------------------------------------------------
template <typename T>
int32_t project_t(b2k_ctx* ctx, const Panel& pn, const VecRef& x, int k, int res_off) {
    const int grid = grid_for_rows<T>(ctx, pn.n);
    const int KC = kcap<T>();
    for (int off = 0; off < k; off += KC) {
        const int kk = std::min(KC, k - off);
        ColList cl;
        fill_cols<T>(cl, pn.idx, off, kk);
        PhaseParams<T> p = base_params<T>(pn, kk, x.ptr, nullptr);
        p.part_h = b2k_part_set(ctx, 0);
        const int pr = b2k_prof_begin(ctx, 3, (kk + 1.0) * sizeof(T) * (double)pn.n);
        B2K_TRY((launch_phase_t<T, false, true>(ctx, p, cl, grid)));
        b2k_prof_end(ctx, pr);
        B2K_TRY(enqueue_finalize(ctx, b2k_part_set(ctx, 0), nullptr, nullptr, grid, kk,
                                 res_off + off, 0));
    }
    return B2K_OK;
}

// unproject: y = beta*y + alpha * sum_j Q[:,j] c[j], coefficients from d_coef (double) or a
// device T vector.  Multi-pass when k > KCAP (beta applies to the first pass only).
template <typename T>
int32_t unproject_t(b2k_ctx* ctx, const Panel& pn, const VecRef& y, int k, const double* dcoef,
                    const T* coef_t, double alpha, double beta, double* part_n) {
    const int grid = grid_for_rows<T>(ctx, pn.n);
    const int KC = kcap<T>();
    int off = 0;
    do {
        const int kk = std::min(KC, k - off);
        ColList cl;
        fill_cols<T>(cl, pn.idx, off, kk);
        PhaseParams<T> p = base_params<T>(pn, kk, y.ptr, y.ptr);
        p.store_x = 1;
        p.coef = dcoef ? dcoef + off : nullptr;
        p.coef_t = coef_t ? coef_t + off : nullptr;
        p.coef_sets = 1;
        p.coef_stride = 0;
        p.alphac = (T)alpha;
        if (off == 0) {
            p.beta_mode = beta == 0.0 ? 0 : (beta == 1.0 ? 1 : 2);
            p.betax = (T)beta;
        }
        p.part_n = (off + kk >= k) ? part_n : nullptr;
        const int pr = b2k_prof_begin(ctx, 4, (kk + 2.0) * sizeof(T) * (double)pn.n);
        B2K_TRY((launch_phase_t<T, true, false>(ctx, p, cl, grid)));
        b2k_prof_end(ctx, pr);
        off += kk;
    } while (off < k);
    return B2K_OK;
}

// ------------------------------------------------------------------------------------
// Gram-Schmidt drivers (device side: everything stays enqueued; results land in d_res)
// d_res layout for orthogonalize: [0..k) h, [k] ||v||^2
// ------------------------------------------------------------------------------------
// One classical Gram-Schmidt pass set.  passes = 1 (CGS) or 2 (CGS2).  Results:
// d_res[0..k) = h (sum over passes), d_res[k] = ||v_out||^2.  Single-GPU fused path.
template <typename T>
int32_t cgs_fused_t(b2k_ctx* ctx, const Panel& pn, const VecRef& v, int k, int passes,
                    bool use_coop) {
    const int grid = grid_for_rows<T>(ctx, pn.n);
    ColList cl;
    fill_cols<T>(cl, pn.idx, 0, k);
    double* PA = b2k_part_set(ctx, 0);
    double* PB = b2k_part_set(ctx, 1);
    double* PN = b2k_part_set(ctx, 2);
    FusedParams<T> fp;
    memset(&fp, 0, sizeof(fp));
    int nph = 0;
    {   // phase A: h1 = Q^T v
        PhaseParams<T> p = base_params<T>(pn, k, v.ptr, nullptr);
        p.part_h = PA;
        fp.ph[nph] = p; fp.kind[nph] = 0; ++nph;
    }
    if (passes == 2) {   // phase B: v1 = v - Q h1 ; h2 = Q^T v1
        PhaseParams<T> p = base_params<T>(pn, k, v.ptr, v.ptr);
        p.store_x = 1;
        p.coef = PA; p.coef_sets = grid; p.coef_stride = B2K_KSTRIDE;
        p.alphac = (T)-1;
        p.part_h = PB;
        fp.ph[nph] = p; fp.kind[nph] = 1; ++nph;
    }
    {   // phase C: v2 = v1 - Q h_last ; ||v2||^2
        PhaseParams<T> p = base_params<T>(pn, k, v.ptr, v.ptr);
        p.store_x = 1;
        p.coef = (passes == 2) ? PB : PA; p.coef_sets = grid; p.coef_stride = B2K_KSTRIDE;
        p.alphac = (T)-1;
        p.part_n = PN;
        fp.ph[nph] = p; fp.kind[nph] = 2; ++nph;
    }
    fp.nph = nph;
    const double W = (double)sizeof(T) * (double)pn.n;
    const int pr = b2k_prof_begin(ctx, 1, (passes == 2 ? (3.0 * k + 5.0) : (2.0 * k + 3.0)) * W);
    if (use_coop) {
        B2K_TRY(launch_fused<T>(ctx, fp, cl, grid));
    } else {
        for (int i = 0; i < nph; ++i) B2K_TRY(launch_phase<T>(ctx, fp.ph[i], cl, fp.kind[i], grid));
    }
    b2k_prof_end(ctx, pr);
    B2K_TRY(enqueue_finalize(ctx, PA, passes == 2 ? PB : nullptr, PN, grid, k, 0, k));
    return B2K_OK;
}

// Distributed / large-k classical Gram-Schmidt: project (all passes) -> allreduce -> update.
// d_res[res_off..+k) receives this pass's h, d_res[nslot] = ||v||^2 (local partial sum, reduced).
template <typename T>
int32_t cgs_pass_unfused_t(b2k_ctx* ctx, const Panel& pn, const VecRef& v, int k, int res_off,
                           int nslot) {
    B2K_TRY(project_t<T>(ctx, pn, v, k, res_off));
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + res_off, k, pn.sharded));
    B2K_TRY(unproject_t<T>(ctx, pn, v, k, ctx->d_res + res_off, nullptr, -1.0, 1.0,
                           b2k_part_set(ctx, 2)));
    const int grid = grid_for_rows<T>(ctx, pn.n);
    // norm partials -> d_res[nslot]
    k_finalize<<<1, NCONS, 0, ctx->stream>>>(b2k_part_set(ctx, 2), nullptr, b2k_part_set(ctx, 2), grid,
                                          B2K_KSTRIDE, 0, ctx->d_res, 0, nslot);
    B2K_LAUNCH_CHECK(ctx);
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + nslot, 1, pn.sharded));
    return B2K_OK;
}

// whether ncols columns fit the panel ring of the cooperative sweep (C columns per chunk)
bool ring_holds(int dtype, int ncols) {
    const int C = dtype == B2K_F64 ? 8 : 16;
    return (ncols + C - 1) / C <= NS && ncols <= MAXCH * C;
}

bool fused_ok(const b2k_ctx* ctx, int k, int sharded, int dtype) {
    return !(ctx->nranks > 1 && sharded) && ring_holds(dtype, k);
}

bool g_use_coop = true;
bool g_use_dmma = true;
int g_transform_ur = 0;      // B2K_TRANSFORM_UR: 0 = DMMA kernel, 1 = <2 rows x 18>, 2 = <2 x 36>, 3 = <4 x 18> (DFMA, U in the constant bank)
int g_transform_hyb = 2;     // B2K_TRANSFORM_HYB: 2 (default) = DFMA 8 x 9 tile for keep <= 36 (k_transform_f89),
                             // 0 = DMMA kernel, 1 = DMMA + DFMA hybrid (k_transform_hyb)
// the restart-GEMM kernel the last b2k_basis_transform launched (b2k_debug_transform_kernel): 0 = none yet,
// 1 / 2 = k_transform<double, U in smem / global>, 3 / 4 = k_transform<float, smem / global>,
// 5 / 6 = k_transform_big<double / float>, 7 / 8 / 9 = k_transform_ur<2,18> / <2,36> / <4,18>,
// 10 = k_transform_f89, 11 = k_transform_f89w, 12 = k_transform_hyb, 13 = k_transform_dmma
int g_transform_kernel = 0;

// modified Gram-Schmidt sweep, pipelined: launch j computes v -= s_{j-1} q_{j-1} and
// s_j = <q_j, v> in one pass (orthonormal.jl:417-421).  d_res[res_off + j] = s_j;
// with accumulate, d_res[acc_off + j] += s_j (reorthogonalize!!, :427-431).
// While a modified Gram-Schmidt sweep runs, the vector being orthogonalised is re-read and
// re-written once per basis vector (4W per column).  If it fits the persisting-L2 carve-out
// (n*8 <= the device's persisting-L2 maximum) it is pinned there for the duration of the sweep, so HBM
// only sees the two basis columns of each pass.
void mgs_pin_vector(b2k_ctx* ctx, const VecRef& v, bool on) {
    if (ctx->l2_persist_bytes == 0) return;
    const size_t bytes = (size_t)v.n * ctx->esize;
    if (bytes > ctx->l2_persist_bytes || bytes > ctx->l2_window_max) return;
    cudaStreamAttrValue attr;
    memset(&attr, 0, sizeof(attr));
    attr.accessPolicyWindow.base_ptr = v.ptr;
    attr.accessPolicyWindow.num_bytes = on ? bytes : 0;
    attr.accessPolicyWindow.hitRatio = 1.0f;
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    // turning the window off is enough: lines left in the persisting carve-out are replaced by the next
    // pinned vector.  (cudaCtxResetPersistingL2Cache() would be a process-wide side effect inside a
    // library call.)
    cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
}

int32_t mgs_sweep(b2k_ctx* ctx, const Panel& pn, const VecRef& v, int k, int res_off, int acc_off) {
    const int es = ctx->esize;
    const bool dist = ctx->nranks > 1 && pn.sharded;
    struct Pin {
        b2k_ctx* c; const VecRef& v; bool on;
        Pin(b2k_ctx* c_, const VecRef& v_, bool on_) : c(c_), v(v_), on(on_) { if (on) mgs_pin_vector(c, v, true); }
        ~Pin() { if (on) mgs_pin_vector(c, v, false); }
    } pin(ctx, v, k >= 4);
    struct Hints {     // without a set-aside the vector is kept L2-resident by eviction-priority hints instead
        b2k_ctx* c;
        explicit Hints(b2k_ctx* c_, bool on) : c(c_) { c->dot_hints = (on && g_l2_hints) ? 1 : 0; }
        ~Hints() { c->dot_hints = 0; }
    } hints(ctx, k >= 4);
    for (int j = 0; j < k; ++j) {
        const char* qj = (const char*)pn.base + (size_t)pn.idx[j] * pn.ld * es;
        const char* qp = j > 0 ? (const char*)pn.base + (size_t)pn.idx[j - 1] * pn.ld * es : nullptr;
        B2K_TRY(b2k_enqueue_dot(ctx, qj, v.ptr, pn.n, qp, j > 0 ? res_off + j - 1 : -1, res_off + j,
                                (!dist && acc_off >= 0) ? acc_off + j : -1));
        if (dist) B2K_TRY(b2k_allreduce(ctx, ctx->d_res + res_off + j, 1, 1));
    }
    if (k > 0) {
        const char* ql = (const char*)pn.base + (size_t)pn.idx[k - 1] * pn.ld * es;
        B2K_TRY(b2k_enqueue_axpy_dev(ctx, v.ptr, ql, res_off + k - 1, pn.n));
    }
    return B2K_OK;
}

// One classical pass of a synchronous CGS2 / CGSIR Lanczos step, K1 <= kcap<T>(): d_res[s_h..+K1) = h,
// d_res[s_n] = ||w||^2.  fused: both sweeps in one cooperative launch (per-phase launches under
// b2k_debug_set_coop(0)).  Otherwise (row-sharded, or more chunks than ring slots) one launch per sweep, and the
// all-reduce of the coefficients sits where the grid barrier was.
template <typename T>
int32_t lanczos_step_gs(b2k_ctx* ctx, const Panel& pn, int K1, const VecRef& rw, bool prologue, double c1,
                        double c2, const double* c2_dev, bool fused, int s_h, int s_n) {
    const int grid = grid_for_rows<T>(ctx, pn.n);
    ColList cl;
    lanczos_cols(cl, pn, K1, prologue);
    FusedParams<T> fp;
    lanczos_sweeps<T>(ctx, fp, pn, K1, rw, grid, prologue, c1, c2, nullptr, c2_dev);
    double* PA = fp.ph[0].part_h;
    double* PN = fp.ph[1].part_n;
    const int pr = b2k_prof_begin(ctx, 1, (2.0 * K1 + 3.0) * sizeof(T) * (double)pn.n);
    if (fused && g_use_coop) {
        B2K_TRY(launch_fused<T>(ctx, fp, cl, grid));
    } else {
        B2K_TRY(launch_phase<T>(ctx, fp.ph[0], cl, 0, grid));
        if (!fused) {
            B2K_TRY(enqueue_finalize(ctx, PA, nullptr, nullptr, grid, K1, s_h, s_n));
            B2K_TRY(b2k_allreduce(ctx, ctx->d_res + s_h, K1, pn.sharded));
            fp.ph[1].coef = ctx->d_res + s_h; fp.ph[1].coef_sets = 1; fp.ph[1].coef_stride = 0;
        }
        B2K_TRY(launch_phase<T>(ctx, fp.ph[1], cl, 2, grid));
    }
    b2k_prof_end(ctx, pr);
    if (fused) return enqueue_finalize(ctx, PA, nullptr, PN, grid, K1, s_h, s_n);
    k_finalize<<<1, NCONS, 0, ctx->stream>>>(PN, nullptr, PN, grid, B2K_KSTRIDE, 0, ctx->d_res, 0, s_n);
    B2K_LAUNCH_CHECK(ctx);
    return b2k_allreduce(ctx, ctx->d_res + s_n, 1, pn.sharded);
}

}  // namespace

int32_t b2k_cross_init(b2k_ctx* ctx);     // b2k_basis_cross_inner, below

// called once per context (ctx.cu): opt in to > 48 KB dynamic shared memory
int32_t b2k_basis_init(b2k_ctx* ctx) {
    if (const char* e = getenv("B2K_L2_HINTS")) g_l2_hints = e[0] != '0';
    if (const char* e = getenv("B2K_TRANSFORM_UR")) g_transform_ur = (e[0] >= '0' && e[0] <= '3') ? e[0] - '0' : 0;
    if (const char* e = getenv("B2K_TRANSFORM_HYB")) g_transform_hyb = (e[0] >= '0' && e[0] <= '3') ? e[0] - '0' : 0;
#define SETATTR(fn, bytes) \
    B2K_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes))
    SETATTR((k_phase<double, false, true>), SMEM_BYTES);
    SETATTR((k_phase<double, true, true>), SMEM_BYTES);
    SETATTR((k_phase<double, true, false>), SMEM_BYTES);
    SETATTR((k_phase<float, false, true>), SMEM_BYTES);
    SETATTR((k_phase<float, true, true>), SMEM_BYTES);
    SETATTR((k_phase<float, true, false>), SMEM_BYTES);
    SETATTR(k_gs_fused<double>, SMEM_BYTES);
    SETATTR(k_gs_fused<float>, SMEM_BYTES);
    SETATTR(k_transform_dmma, TD_SMEM);
    SETATTR(k_transform_hyb, TD_SMEM);
    SETATTR(k_transform_f89, TR_SMEM);
    SETATTR(k_transform_f89w, TR_SMEM);
    SETATTR((k_transform_ur<2, 18>), TR_SMEM);
    SETATTR((k_transform_ur<2, 36>), TR_SMEM);
    SETATTR((k_transform_ur<4, 18>), TR_SMEM);
    SETATTR((k_transform<double, true>), TR_SMEM);
    SETATTR((k_transform<double, false>), TR_SMEM);
    SETATTR((k_transform<float, true>), TR_SMEM);
    SETATTR((k_transform<float, false>), TR_SMEM);
    SETATTR(k_transform_big<double>, TB_SMEM_MAX);
    SETATTR(k_transform_big<float>, TB_SMEM_MAX);
#undef SETATTR
    return b2k_cross_init(ctx);
}

extern "C" int32_t b2k_debug_set_dmma(int32_t on) {
    g_use_dmma = on != 0;
    return B2K_OK;
}

// restart-GEMM kernel for tests / A-B runs: 0 = default, 1..3 = constant-bank DFMA variants (k_transform_ur),
// 4 = DMMA + DFMA hybrid, 5 = DFMA 8 x 9 tile, 6 = DMMA
extern "C" int32_t b2k_debug_set_transform(int32_t mode) {
    g_transform_ur = (mode >= 0 && mode <= 3) ? mode : 0;
    g_transform_hyb = mode == 4 ? 1 : (mode == 5 ? 2 : (mode == 7 ? 3 : (mode == 0 ? 2 : 0)));   // 0 = default, 4 = hybrid, 5 = 8 x 9 (two sets, alternate tiles), 6 = DMMA, 7 = 8 x 9 on 512-row tiles
    return B2K_OK;
}

// which kernel the last b2k_basis_transform launched (ids at g_transform_kernel): tests assert the dispatch with it
extern "C" int32_t b2k_debug_transform_kernel(void) { return g_transform_kernel; }

extern "C" int32_t b2k_debug_set_coop(int32_t on) {
    g_use_coop = on != 0;
    return B2K_OK;
}

// ------------------------------------------------------------------ C ABI ----

extern "C" int32_t b2k_basis_project(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, b2k_vec x,
                                     double alpha, double beta, double* h_host) {
    if (!ctx || (k > 0 && !h_host)) return B2K_EINVAL;
    if (k == 0) return B2K_OK;
    if (k > B2K_RES_DOUBLES - 8) return b2k_fail(ctx, B2K_EINVAL, "basis_project: k too large");
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, k, &pn));
    VecRef rx;
    B2K_TRY(b2k_resolve(ctx, x, &rx));
    if (rx.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "basis_project: x has %lld rows, basis %lld",
                                      (long long)rx.n, (long long)pn.n);
    B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return project_t<decltype(t)>(ctx, pn, rx, k, 0); }));
    B2K_TRY(b2k_fetch_results(ctx, k, pn.sharded));
    for (int j = 0; j < k; ++j)
        h_host[j] = (beta == 0.0) ? alpha * ctx->h_res[j] : beta * h_host[j] + alpha * ctx->h_res[j];
    return B2K_OK;
}

extern "C" int32_t b2k_basis_unproject(b2k_ctx* ctx, b2k_vec y, const b2k_vec* cols, int32_t k,
                                       const double* c_host, double alpha, double beta) {
    if (!ctx || (k > 0 && !c_host)) return B2K_EINVAL;
    VecRef ry;
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    if (k == 0) {   // orthonormal.jl:162-164
        if (beta == 1.0) return B2K_OK;
        if (beta == 0.0) return b2k_vec_zero(ctx, y);
        return b2k_vec_scale(ctx, y, y, beta);
    }
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, k, &pn));
    if (ry.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "basis_unproject: y has %lld rows, basis %lld",
                                      (long long)ry.n, (long long)pn.n);
    for (int j = 0; j < k; ++j)
        if (pn.idx[j] == ry.col && ry.space == B2K_VEC_SPACE(cols[j]))
            return b2k_fail(ctx, B2K_EINVAL, "basis_unproject: y aliases basis vector %d", j);
    B2K_TRY(b2k_put_coef(ctx, c_host, k, 0));
    return b2k_dispatch(ctx, [&](auto t) {
        return unproject_t<decltype(t)>(ctx, pn, ry, k, ctx->d_coef, nullptr, alpha, beta, nullptr);
    });
}

// internal: used by the dense operator (spmv.cu): y = A x / y = A' x through the engine
int32_t b2k_panel_unproject_dev(b2k_ctx* ctx, void* base, int64_t ld, int64_t n, int32_t k,
                                const VecRef& y, const void* coef_t) {
    Panel pn;
    pn.base = base; pn.ld = ld; pn.n = n; pn.sharded = y.sharded;
    pn.idx.resize(k);
    for (int i = 0; i < k; ++i) pn.idx[i] = i;
    return b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        return unproject_t<T>(ctx, pn, y, k, nullptr, (const T*)coef_t, 1.0, 0.0, nullptr);
    });
}

int32_t b2k_panel_project_dev(b2k_ctx* ctx, void* base, int64_t ld, int64_t n, int32_t k,
                              const VecRef& x, void* out_vec, int32_t sharded) {
    Panel pn;
    pn.base = base; pn.ld = ld; pn.n = n; pn.sharded = sharded;
    pn.idx.resize(k);
    for (int i = 0; i < k; ++i) pn.idx[i] = i;
    if (k > B2K_RES_DOUBLES) return b2k_fail(ctx, B2K_ENOTSUP, "dense adjoint: too many columns");
    B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return project_t<decltype(t)>(ctx, pn, x, k, 0); }));
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, k, sharded));
    const int blocks = (k + 127) / 128;
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
        k_res_to_vec<T><<<blocks, 128, 0, ctx->stream>>>(ctx->d_res, (T*)out_vec, k, T(1));
    });
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_basis_orthogonalize(b2k_ctx* ctx, b2k_vec v, const b2k_vec* cols, int32_t k,
                                           double* h_host, int32_t alg, double eta,
                                           double* nrm_out, int32_t* passes_out) {
    if (!ctx || (k > 0 && !h_host)) return B2K_EINVAL;
    if (alg < B2K_CGS || alg > B2K_MGS2B)
        return b2k_fail(ctx, B2K_EINVAL, "basis_orthogonalize: unknown orthogonalizer %d", alg);
    VecRef rv;
    B2K_TRY(b2k_resolve(ctx, v, &rv));
    if (passes_out) *passes_out = 0;
    if (k == 0) {
        if (nrm_out) return b2k_vec_norm(ctx, v, nrm_out);
        return B2K_OK;
    }
    if (k + 8 > 2048) return b2k_fail(ctx, B2K_ENOTSUP, "basis_orthogonalize: k > 2040");
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, k, &pn));
    if (rv.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "basis_orthogonalize: v has %lld rows, basis %lld",
                                      (long long)rv.n, (long long)pn.n);
    for (int j = 0; j < k; ++j)
        if (pn.idx[j] == rv.col && rv.space == B2K_VEC_SPACE(cols[j]))
            return b2k_fail(ctx, B2K_EINVAL, "basis_orthogonalize: v aliases basis vector %d", j);
    const bool fusable = fused_ok(ctx, k, pn.sharded, ctx->dtype);
    const double eps = b2k_eps(ctx);   // of the IR loops (orthonormal.jl, lanczos.jl)
    const int NS_ = 2 * k + 4;   // slot of ||v||^2 results for unfused / MGS paths

    auto cgs_passes = [&](int passes) -> int32_t {   // leaves h in h_res[0..k), norm^2 in h_res[k]
        if (fusable) {
            B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return cgs_fused_t<decltype(t)>(ctx, pn, rv, k, passes, g_use_coop); }));
            return b2k_fetch_results(ctx, k + 1, 0);
        }
        // unfused: pass p writes h_p to d_res[p*k ..], norm to d_res[NS_]
        for (int ps = 0; ps < passes; ++ps) {
            B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return cgs_pass_unfused_t<decltype(t)>(ctx, pn, rv, k, ps * k, NS_); }));
        }
        B2K_TRY(b2k_fetch_results(ctx, NS_ + 1, 0));
        if (passes == 2)
            for (int j = 0; j < k; ++j) ctx->h_res[j] += ctx->h_res[k + j];
        ctx->h_res[k] = ctx->h_res[NS_];
        return B2K_OK;
    };
    auto mgs_passes = [&](int passes) -> int32_t {
        B2K_TRY(mgs_sweep(ctx, pn, rv, k, 0, -1));
        if (passes == 2) B2K_TRY(mgs_sweep(ctx, pn, rv, k, k, -1));
        B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rv.ptr, pn.n, nullptr, -1, NS_, -1));
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res + NS_, 1, pn.sharded));
        B2K_TRY(b2k_fetch_results(ctx, NS_ + 1, 0));
        if (passes == 2)
            for (int j = 0; j < k; ++j) ctx->h_res[j] += ctx->h_res[k + j];
        ctx->h_res[k] = ctx->h_res[NS_];
        return B2K_OK;
    };

    int passes = 0;
    double nrm = 0.0;
    switch (alg) {
        case B2K_CGS:
            B2K_TRY(cgs_passes(1)); passes = 1; break;
        case B2K_CGS2:
        case B2K_MGS2B:      // flagged: both sweeps as classical blocks
            B2K_TRY(cgs_passes(2)); passes = 2; break;
        case B2K_MGS:
            B2K_TRY(mgs_passes(1)); passes = 1; break;
        case B2K_MGS2:
            B2K_TRY(mgs_passes(2)); passes = 2; break;
        case B2K_CGSIR:
        case B2K_MGSIR: {
            // orthonormal.jl:400-412 / 440-452: nold = norm(v); one pass; loop while
            // eps < nnew < eta*nold
            double nold;
            B2K_TRY(b2k_vec_norm(ctx, v, &nold));
            std::vector<double> hsum(k, 0.0);
            double nnew = 0.0;
            for (;;) {
                if (alg == B2K_CGSIR) B2K_TRY(cgs_passes(1));
                else B2K_TRY(mgs_passes(1));
                ++passes;
                for (int j = 0; j < k; ++j) hsum[j] += ctx->h_res[j];
                nnew = sqrt(ctx->h_res[k]);
                if (!(eps < nnew && nnew < eta * nold)) break;
                nold = nnew;
            }
            for (int j = 0; j < k; ++j) h_host[j] = hsum[j];
            if (nrm_out) *nrm_out = nnew;
            if (passes_out) *passes_out = passes;
            return B2K_OK;
        }
    }
    for (int j = 0; j < k; ++j) h_host[j] = ctx->h_res[j];
    nrm = sqrt(ctx->h_res[k]);
    if (nrm_out) *nrm_out = nrm;
    if (passes_out) *passes_out = passes;
    return B2K_OK;
}

// expand! + lanczosrecurrence — src/factorizations/lanczos.jl:250-272, 295-376
extern "C" int32_t b2k_lanczos_expand(b2k_ctx* ctx, const b2k_op* op, const b2k_vec* cols,
                                      int32_t k, b2k_vec r, b2k_vec w, double beta_old,
                                      int32_t alg, double eta, double* alpha_out,
                                      double* beta_out) {
    if (!ctx || !op || !cols || k < 1 || !alpha_out || !beta_out) return B2K_EINVAL;
    if (alg < B2K_CGS || alg > B2K_MGS2B)
        return b2k_fail(ctx, B2K_EINVAL, "lanczos_expand: unknown orthogonalizer %d", alg);
    if (cols[k] != r) return b2k_fail(ctx, B2K_EINVAL, "lanczos_expand: cols[k] must be r");
    if (beta_old == 0.0) return b2k_fail(ctx, B2K_EINVAL, "lanczos_expand: beta_old == 0");
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, k + 1, &pn));   // V after push!: k+1 vectors
    VecRef rv, rw, vprev;
    B2K_TRY(b2k_resolve(ctx, r, &rv));
    B2K_TRY(b2k_resolve(ctx, w, &rw));
    B2K_TRY(b2k_resolve(ctx, cols[k - 1], &vprev));
    if (rv.n != pn.n || rw.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "lanczos_expand: length mismatch");
    for (int j = 0; j <= k; ++j)
        if (cols[j] == w) return b2k_fail(ctx, B2K_EINVAL, "lanczos_expand: w aliases the basis");
    const int K1 = k + 1;
    const double eps = b2k_eps(ctx);   // of the IR loops (orthonormal.jl, lanczos.jl)
    // d_res slots
    const int S_H = 0;             // [0..K1) projection coefficients
    const int S_N = K1;            // ||w||^2
    const int S_A0 = K1 + 1;       // <v, A v>

    // v = r / beta_old  (the residual's storage becomes the new basis vector, lanczos.jl:257)
    B2K_TRY(b2k_vec_scale(ctx, r, r, 1.0 / beta_old));

    if (alg == B2K_CGS || alg == B2K_CGS2 || alg == B2K_CGSIR) {
        // w = A v ; alpha = <v, w>   (one pass)
        B2K_TRY(b2k_enqueue_apply(ctx, op, rv, rw, 0.0, 1.0, false, &rv, S_A0));
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_A0, 1, pn.sharded));
        // CGS2 on the fused path keeps alpha on the device (the prologue reads it from d_res) so
        // that the whole step needs ONE host synchronisation; the other variants fetch it now.
        const bool one_pass = K1 <= b2k_dispatch(ctx, [](auto t) { return kcap<decltype(t)>(); });
        const bool defer_alpha = (alg == B2K_CGS2) && one_pass;
        double alpha = 0.0;
        if (!defer_alpha) {
            B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
            alpha = ctx->h_res[S_A0];
        }
        if (alg == B2K_CGS) {
            // w = (w - beta v_prev) - alpha v ; beta = ||w||
            B2K_TRY(b2k_vec_axpy2(ctx, w, cols[k - 1], -beta_old, r, -alpha));
            B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
            B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
            B2K_TRY(b2k_fetch_results(ctx, S_N + 1, 0));
            *alpha_out = alpha;
            *beta_out = sqrt(ctx->h_res[S_N]);
            return B2K_OK;
        }
        // CGS2 / CGSIR: three-term prologue fused into the projection sweep, then update+norm
        double ab2 = alpha * alpha + beta_old * beta_old;
        double beta = 0.0, nold = 0.0;
        bool first = true;
        for (;;) {
            const bool fusable = fused_ok(ctx, K1, pn.sharded, ctx->dtype);
            const bool prologue = first;
            if (alg == B2K_CGSIR && first) {
                // need beta = ||w'|| before deciding on reorthogonalisation (lanczos.jl:346-349)
                B2K_TRY(b2k_vec_axpy2(ctx, w, cols[k - 1], -beta_old, r, -alpha));
                B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
                B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
                B2K_TRY(b2k_fetch_results(ctx, S_N + 1, 0));
                beta = sqrt(ctx->h_res[S_N]);
                nold = sqrt(beta * beta + ab2);
                first = false;
                if (!(eps < beta && beta < eta * nold)) break;
                nold = beta;
                continue;
            }
            if (one_pass) {
                const double* c2_dev = defer_alpha ? ctx->d_res + S_A0 : nullptr;
                B2K_TRY(b2k_dispatch(ctx, [&](auto t) {
                    return lanczos_step_gs<decltype(t)>(ctx, pn, K1, rw, prologue, -beta_old, -alpha, c2_dev, fusable,
                                                        S_H, S_N);
                }));
                B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
                if (defer_alpha) alpha = ctx->h_res[S_A0];
            } else {
                if (prologue) B2K_TRY(b2k_vec_axpy2(ctx, w, cols[k - 1], -beta_old, r, -alpha));
                B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return cgs_pass_unfused_t<decltype(t)>(ctx, pn, rw, K1, S_H, S_N); }));
                B2K_TRY(b2k_fetch_results(ctx, S_N + 1, 0));
            }
            alpha += ctx->h_res[S_H + k];        // α += s[end]
            beta = sqrt(ctx->h_res[S_N]);
            first = false;
            if (alg == B2K_CGS2) break;
            if (!(eps < beta && beta < eta * nold)) break;
            nold = beta;
        }
        *alpha_out = alpha;
        *beta_out = beta;
        return B2K_OK;
    }

    // MGS family (lanczos.jl:304-312, 325-338, 357-376): w = A v ; w -= beta v_prev ;
    // alpha = <v, w> ; w -= alpha v ; [second sweep over all of V]
    int32_t op_kind = -1;
    B2K_TRY(b2k_op_info(op, nullptr, nullptr, nullptr, &op_kind));
    if (alg == B2K_MGS2B && op_kind != 1) {
        // alpha = <v, A v - beta v_prev> fused into the SpMV epilogue (dot_sub_vec), the order of the chained step
        // (lanczos_chain), so that a chained batch and these steps give the same bits
        SpmvFuse fz;
        memset(&fz, 0, sizeof(fz));
        fz.dot_sub_vec = vprev.ptr;
        fz.dot_sub_scale = ctx->d_coef;
        B2K_TRY(b2k_put_coef(ctx, &beta_old, 1, 0));
        B2K_TRY(b2k_enqueue_apply_fused(ctx, op, rv, rw, 0.0, 1.0, false, &rv, ctx->d_res + S_A0, &fz));
        B2K_TRY(b2k_vec_axpby(ctx, w, cols[k - 1], -beta_old, 1.0));
    } else {
        B2K_TRY(b2k_enqueue_apply(ctx, op, rv, rw, 0.0, 1.0, false, nullptr, -1));
        B2K_TRY(b2k_vec_axpby(ctx, w, cols[k - 1], -beta_old, 1.0));
        B2K_TRY(b2k_enqueue_dot(ctx, rv.ptr, rw.ptr, pn.n, nullptr, -1, S_A0, -1));
    }
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_A0, 1, pn.sharded));
    B2K_TRY(b2k_enqueue_axpy_dev(ctx, rw.ptr, rv.ptr, S_A0, pn.n));
    double alpha = 0.0, beta = 0.0;
    if (alg == B2K_MGS) {
        B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
        B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
        alpha = ctx->h_res[S_A0];
        beta = sqrt(ctx->h_res[S_N]);
    } else if (alg == B2K_MGS2B) {
        // flagged: the second sweep over all of V as ONE classical pass (project, update + norm)
        if (fused_ok(ctx, K1, pn.sharded, ctx->dtype)) {
            B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return cgs_fused_t<decltype(t)>(ctx, pn, rw, K1, 1, g_use_coop); }));
        } else {
            B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return cgs_pass_unfused_t<decltype(t)>(ctx, pn, rw, K1, S_H, S_N); }));
        }
        B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
        alpha = ctx->h_res[S_A0] + ctx->h_res[S_H + k];   // α += s (coefficient vs V[end])
        beta = sqrt(ctx->h_res[S_N]);
    } else if (alg == B2K_MGS2) {
        B2K_TRY(mgs_sweep(ctx, pn, rw, K1, S_H, -1));
        B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
        B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
        alpha = ctx->h_res[S_A0] + ctx->h_res[S_H + k];   // α += s (coefficient vs V[end])
        beta = sqrt(ctx->h_res[S_N]);
    } else {   // MGSIR
        B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
        B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
        B2K_TRY(b2k_fetch_results(ctx, S_A0 + 1, 0));
        alpha = ctx->h_res[S_A0];
        beta = sqrt(ctx->h_res[S_N]);
        double nold = sqrt(beta * beta + alpha * alpha + beta_old * beta_old);
        while (eps < beta && beta < eta * nold) {
            nold = beta;
            B2K_TRY(mgs_sweep(ctx, pn, rw, K1, S_H, -1));
            B2K_TRY(b2k_enqueue_dot(ctx, nullptr, rw.ptr, pn.n, nullptr, -1, S_N, -1));
            B2K_TRY(b2k_allreduce(ctx, ctx->d_res + S_N, 1, pn.sharded));
            B2K_TRY(b2k_fetch_results(ctx, S_N + 1, 0));
            alpha += ctx->h_res[S_H + k];
            beta = sqrt(ctx->h_res[S_N]);
        }
    }
    *alpha_out = alpha;
    *beta_out = beta;
    return B2K_OK;
}

// The inner loop of eigsolve (src/eigsolve/lanczos.jl:33-78 while K < krylovdim and beta > tol):
// consecutive expand! steps without returning to the caller.  One host synchronisation per
// step remains (the reference checks beta after every step), but the per-step host work is
// C++ instead of interpreter time.
// ---------------------------------------------------------------------------------------
// Device-chained Lanczos steps (ClassicalGramSchmidt2, lanczos.jl:250-272 + 313-324), TWO launches per step
// and no host round trip between steps:
//   1. SpMV with the normalisation fused into the gather: reads the residual r (unnormalised), the scalar
//      1/β from the previous step's device record, writes v = r·(1/β) into a column of its own (it becomes the
//      new basis vector; r's column is recycled by a later step), w = A v, and α₀ = <v, w> into this step's record;
//   2. the cooperative Gram-Schmidt kernel: prologue w − β v₋ − α₀ v with β, α₀ read from the records, projection
//      on all of V, grid barrier, update + ||w||², and the last CTA finalises the step's record {α, β, 1/β}.
// The reference looks at β after every step (eigsolve/lanczos.jl:45: `while K < krylovdim && β > tol`), so do
// the kernels: a record with β <= tol raises a device flag and everything enqueued behind it does nothing.  The
// host reads all records with ONE synchronisation at the end of the batch and commits the steps up to the
// first β <= tol — same α, β, V, r as stepping one at a time, bit for bit (same kernels, same operand bits).  The
// flagged ModifiedGramSchmidt2Blocked chains too: its α₀ = <v, A v − β v₋> comes from the SpMV epilogue
// (dot_sub_vec) in the chain and in the synchronous step (b2k_lanczos_expand) alike, on CSR and stencil operators.
bool g_use_chain = true;

bool chain_ok(const b2k_ctx* ctx, const b2k_op* op, const b2k_vec* cols, int32_t k, int32_t nsteps, int32_t alg,
              double beta_old) {
    if (!g_use_chain || !g_use_coop || (alg != B2K_CGS2 && alg != B2K_MGS2B) || nsteps < 1 || nsteps > B2K_MAX_CHAIN)
        return false;
    int64_t op_rows = 0, op_cols = 0;
    int32_t op_kind = -1;
    if (b2k_op_info(op, &op_rows, &op_cols, nullptr, &op_kind) != B2K_OK) return false;
    if ((op_kind != 0 && op_kind != 2) || beta_old == 0.0 || !(beta_old == beta_old)) return false;
    const int32_t sp = B2K_VEC_SPACE(cols[k]);
    if (sp < 0 || sp >= (int32_t)ctx->spaces.size()) return false;
    const B2kSpace& s = ctx->spaces[sp];
    if (ctx->nranks > 1) {
        // row-sharded: every exchange of the step goes through the NVLink peer window (no NCCL, no extra launch)
        if (!s.sharded || !b2k_peer_ok(ctx) || !b2k_op_has_peer_halo(op) || op_rows != s.n) return false;
    } else if (op_rows != s.n || op_cols != s.n) {
        return false;
    }
    const int K1 = k + nsteps;
    return ring_holds(ctx->dtype, K1) && K1 <= PEER_SLOT;
}

// The cooperative CGS sweep of one chained step over the K1 columns of pn, finalised into the device record rec.
// Lanczos: with the three-term prologue (beta from rec_prev, <v, A v> from rec).  GKL (b2k_gkl_expand_many): no
// prologue (the SpMV epilogue has subtracted alpha u already), and a non-finite norm raises the stop flag too.
// skip_on (b2k_lsmr_chain): the device flag that makes the launch do nothing, instead of the batch's stop flag.
template <typename T>
int32_t chain_step_gs(b2k_ctx* ctx, const Panel& pn, int K1, const VecRef& rw, double* rec_prev, double* rec,
                      double tol, const PeerStep* psp, bool prologue = true, int stop_nonfinite = 0,
                      const int* skip_on = nullptr) {
    const int grid = grid_for_rows<T>(ctx, pn.n);
    ColList cl;
    lanczos_cols(cl, pn, K1, prologue);
    double* PA = b2k_part_set(ctx, 0);
    double* PN = b2k_part_set(ctx, 2);
    FusedParams<T> fp;
    // the prologue's beta is the previous step's, <v, A v> this step's (the SpMV wrote it)
    lanczos_sweeps<T>(ctx, fp, pn, K1, rw, grid, prologue, 0.0, 0.0, prologue ? rec_prev + 2 : nullptr,
                      prologue ? rec + 0 : nullptr);
    fp.fin.stop_nonfinite = stop_nonfinite;
    fp.stop = skip_on ? skip_on : reinterpret_cast<const int*>(ctx->d_sync + B2K_SYNC_STOP);
    fp.trace = ctx->d_trace;
    fp.fin.A = PA; fp.fin.B = nullptr; fp.fin.N = PN; fp.fin.G = grid; fp.fin.stride = B2K_KSTRIDE;
    fp.fin.k = K1; fp.fin.res = nullptr; fp.fin.off = 0; fp.fin.noff = 0; fp.fin.rec = rec;
    fp.fin.alpha_col = K1 - 1; fp.fin.tol = tol;
    fp.fin.stop = reinterpret_cast<int*>(ctx->d_sync + B2K_SYNC_STOP);
    fp.fin.ticket = ctx->d_sync + B2K_SYNC_GSFIN; fp.fin.enabled = 1;
    fp.fin.peer = 0; fp.fin.G_local = grid;
    if (psp && psp->on) {
        const PeerStep& ps = *psp;
        fp.ps = ps;
        char* win = b2k_peer_local(ctx);
        auto slot = [&](int ch, unsigned long long seq) {
            return reinterpret_cast<double*>(win + PEER_OFF_SLOTS) + (size_t)((ch * 2 + (int)(seq & 1ull)) * PEER_MAXR) * PEER_SLOT;
        };
        // <v, A v>: the per-rank partials the SpMV published (rank order)
        for (int i = 0; i < 2; ++i) {
            fp.ph[i].c2_dev = slot(PEER_CH_ALPHA, ps.seq_alpha);
            fp.ph[i].c2_sets = ps.pd.nranks;
            fp.ph[i].c2_stride = PEER_SLOT;
        }
        // projection coefficients: the per-rank sums in my window instead of the per-CTA partials
        fp.ph[1].coef = slot(PEER_CH_COEF, ps.seq_coef[0]);
        fp.ph[1].coef_sets = ps.pd.nranks;
        fp.ph[1].coef_stride = PEER_SLOT;
        fp.ph[1].coef_ranks = 1;
        fp.fin.A = fp.ph[1].coef; fp.fin.G = ps.pd.nranks; fp.fin.stride = PEER_SLOT; fp.fin.peer = 1;
        // rows the neighbours need for their next SpMV leave with the final store
        if (ps.seq_halo) {
            PhaseParams<T>& c = fp.ph[1];
            c.send_lo = ps.send_lo;
            c.send_hi = ps.send_hi;
            c.halo_dn = ps.send_lo ? reinterpret_cast<T*>(ps.pd.win[ps.pd.rank - 1] + ps.dn_off) : nullptr;
            c.halo_up = ps.send_hi ? reinterpret_cast<T*>(ps.pd.win[ps.pd.rank + 1] + ps.up_off) : nullptr;
        }
    }
    const int pr = b2k_prof_begin(ctx, 1, (2.0 * K1 + 3.0) * sizeof(T) * (double)pn.n);
    B2K_TRY(launch_fused<T>(ctx, fp, cl, grid));
    b2k_prof_end(ctx, pr);
    return B2K_OK;
}

int32_t lanczos_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec* cols, int32_t k, int32_t nsteps,
                      double beta_old, double tol, int32_t alg, double* alphas_out, double* betas_out,
                      int32_t* steps_done, b2k_vec* r_out) {
    const int32_t space = B2K_VEC_SPACE(cols[k]);
    {   // every handle must be live before anything is enqueued
        VecRef t;
        for (int i = 0; i <= k; ++i) B2K_TRY(b2k_resolve(ctx, cols[i], &t));
    }
    // record i of the batch is rec_{i-1} of the step protocol below; the seed is rec_{-1}
    B2kChain fr(ctx, B2K_REC);
    k_lanczos_seed<<<1, 1, 0, ctx->stream>>>(fr.st, beta_old, fr.stop);
    B2K_LAUNCH_CHECK(ctx);
    B2kChainCols cc(ctx, cols[k]);
    int32_t enq = 0, rc = B2K_OK;
    const bool dist = ctx->nranks > 1;
    unsigned long long halo_seq = 0;
    for (int32_t i = 0; i < nsteps; ++i) {
        const int32_t K = k + i;                 // basis size before this step's push!
        const b2k_vec R = cols[K];
        b2k_vec V = -1, W = -1;
        if ((rc = cc.alloc(space, &V)) != B2K_OK || (rc = cc.alloc(space, &W)) != B2K_OK) break;
        VecRef rR, rV, rW, vprev;
        rc = b2k_resolve(ctx, R, &rR);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, V, &rV);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, W, &rW);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, cols[K - 1], &vprev);
        if (rc != B2K_OK) break;
        double* rec_prev = fr.st + (size_t)B2K_REC * i;
        double* rec = fr.rec0 + (size_t)B2K_REC * i;
        SpmvFuse fz;
        memset(&fz, 0, sizeof(fz));
        fz.xscale = rec_prev + 3;
        fz.vout = rV.ptr;
        fz.stop = fr.stop;
        fz.dot_self = 1;
        fz.l2_hints = g_l2_hints ? 1 : 0;
        fz.trace = ctx->d_trace;
        if (alg == B2K_MGS2B) {                  // alpha = <v, A v - beta v_prev>: the modified order
            fz.dot_sub_vec = vprev.ptr;
            fz.dot_sub_scale = rec_prev + 2;
        }
        PeerStep ps;
        memset(&ps, 0, sizeof(ps));
        if (dist) {
            ps.on = 1;
            ps.pd = *b2k_peer_dev(ctx);
            ps.seq_alpha = b2k_peer_next_seq(ctx, PEER_CH_ALPHA);
            ps.seq_coef[0] = b2k_peer_next_seq(ctx, PEER_CH_COEF);
            ps.seq_norm = b2k_peer_next_seq(ctx, PEER_CH_NORM);
            fz.seq_alpha = ps.seq_alpha;
            fz.seq_halo = halo_seq;                    // 0: the apply pushes its operand's boundary rows itself
            halo_seq = b2k_peer_next_seq(ctx, 4);      // this step's Gram-Schmidt launch pushes the next operand's
            rc = b2k_op_peer_halo(ctx, op, halo_seq, &ps);
            if (rc != B2K_OK) break;
        }
        rc = b2k_enqueue_apply_fused(ctx, op, rR, rW, 0.0, 1.0, false, nullptr, rec + 0, &fz);
        if (rc != B2K_OK) break;
        cols[K] = V;                             // the normalised residual is the new basis vector ...
        Panel pn;
        rc = make_panel(ctx, cols, K + 1, &pn);
        if (rc != B2K_OK) break;
        rc = b2k_dispatch(ctx, [&](auto t) {
            return chain_step_gs<decltype(t)>(ctx, pn, K + 1, rW, rec_prev, rec, tol, &ps);
        });
        if (rc != B2K_OK) break;
        cols[K + 1] = W;                         // ... and w the new residual
        cc.ran(V, -1, W);
        cc.consumed(R);
        ++enq;
    }
    int32_t d = 0;
    if (enq > 0) {
        B2K_TRY(fr.fetch(enq));                  // ... and the peer-window watchdog latch of the batch
        d = fr.count(enq, [&](const double* r) { return r[2] <= tol; });
        for (int32_t i = 0; i < d; ++i) {
            alphas_out[i] = fr.hrec[(size_t)B2K_REC * i + 1];
            betas_out[i] = fr.hrec[(size_t)B2K_REC * i + 2];
        }
    } else {
        fr.fail(rc);
    }
    *steps_done = d;
    *r_out = cc.commit(d, cols, nullptr, k);
    return rc;
}

extern "C" int32_t b2k_debug_set_chain(int32_t on) {
    g_use_chain = on != 0;
    return B2K_OK;
}

extern "C" int32_t b2k_lanczos_expand_many(b2k_ctx* ctx, const b2k_op* op, b2k_vec* cols, int32_t k,
                                           int32_t nsteps, double beta_old, double tol, int32_t alg,
                                           double eta, double* alphas_out, double* betas_out,
                                           int32_t* steps_done, b2k_vec* r_out) {
    if (!ctx || !op || !cols || k < 1 || nsteps < 0 || !alphas_out || !betas_out || !steps_done || !r_out)
        return B2K_EINVAL;
    *steps_done = 0;
    b2k_vec r = cols[k];
    *r_out = r;
    if (chain_ok(ctx, op, cols, k, nsteps, alg, beta_old))
        return lanczos_chain(ctx, op, cols, k, nsteps, beta_old, tol, alg, alphas_out, betas_out, steps_done, r_out);
    double beta = beta_old;
    for (int32_t i = 0; i < nsteps; ++i) {
        b2k_vec w;
        B2K_TRY(b2k_vec_alloc(ctx, B2K_VEC_SPACE(r), &w));
        double a = 0.0, b = 0.0;
        int32_t rc = b2k_lanczos_expand(ctx, op, cols, k, r, w, beta, alg, eta, &a, &b);
        if (rc != B2K_OK) {
            b2k_vec_free(ctx, w);
            return rc;
        }
        alphas_out[i] = a;
        betas_out[i] = b;
        ++k;                 // cols[k-1] == old r is now the newest basis vector
        cols[k] = w;         // the new residual
        r = w;
        beta = b;
        *steps_done = i + 1;
        *r_out = r;
        if (beta <= tol) break;
    }
    return B2K_OK;
}

// ---------------------------------------------------------------------------------------
// Device-chained GKL steps (gkl.jl:246-269 + 308-323, CGS2 / the flagged MGS2B), THREE launches per CGS2 step and no
// host round trip between steps.  The operators are rectangular, so each SpMV finishes the previous vector of its own
// row space in its epilogue (SpmvFuse::pvec) instead of storing its normalised operand:
//   1. A' r (n rows): gathers r * (1/beta) (u_k, xscale); row j: v_{k-1} = rn(v~_{k-1} * (1/alpha_{k-1})) stored in
//      place, v~_k = fma(-beta, v_{k-1}, y_j); sum v~_k^2 -> alpha, 1/alpha in the step record (CGS2);
//      MGS2B: the cooperative sweep over V then removes V' v~_k and its finaliser writes alpha instead;
//   2. A v~_k (m rows): gathers v~_k * (1/alpha) (v_k); row i: u_k = rn(r_i * (1/beta)) stored to its column,
//      r'_i = fma(-alpha, u_k, y_i);
//   3. the cooperative CGS sweep of r' over U (chain_step_gs without the Lanczos prologue); its finaliser writes beta,
//      1/beta and raises the stop flag on beta <= tol or a non-finite beta.
// A flush launch at the end of the call normalises the v~ of the last step that ran (k_gkl_flush).
// Rounding: every vector is rounded like the scale!! / add!! it replaces, given the same scalars; alpha and beta are
// the CTA-ordered sums of the fused dot (b2k_op_apply_dot) and the sweep, which may differ from b2k_vec_norm in the
// last bits.  A batch of N steps gives the bits of N calls of one step.
namespace {

int32_t gkl_refuse(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, const b2k_vec* ucols, const b2k_vec* vcols,
                   int32_t k, int32_t nsteps, int32_t alg) {
    if (alg != B2K_CGS2 && alg != B2K_MGS2B)
        return b2k_fail(ctx, B2K_ENOTSUP, "gkl_expand_many: ClassicalGramSchmidt2 / ModifiedGramSchmidt2Blocked only");
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "gkl_expand_many: row-sharded contexts are not supported");
    int64_t m = 0, n = 0, tm = 0, tn = 0;
    int32_t ka = -1, kt = -1;
    B2K_TRY(b2k_op_info(A, &m, &n, nullptr, &ka));
    B2K_TRY(b2k_op_info(At, &tm, &tn, nullptr, &kt));
    if (ka != 0 || kt != 0)
        return b2k_fail(ctx, B2K_ENOTSUP, "gkl_expand_many: A and A' must be stored CSR matrices");
    if (!g_use_coop || !b2k_spmv_tma_on())
        return b2k_fail(ctx, B2K_ENOTSUP, "gkl_expand_many: needs the cooperative sweep and the TMA SpMV kernels");
    if (tm != n || tn != m)
        return b2k_fail(ctx, B2K_EDIM, "gkl_expand_many: A' is %lld x %lld, A is %lld x %lld", (long long)tm,
                        (long long)tn, (long long)m, (long long)n);
    VecRef t;
    int32_t su = -1, sv = -1;
    for (int i = 0; i <= k; ++i) {
        B2K_TRY(b2k_resolve(ctx, ucols[i], &t));
        if (i == 0) su = t.space;
        if (t.space != su || t.n != m)
            return b2k_fail(ctx, B2K_EDIM, "gkl_expand_many: U and r must be columns of one space of length %lld",
                            (long long)m);
    }
    for (int i = 0; i < k; ++i) {
        B2K_TRY(b2k_resolve(ctx, vcols[i], &t));
        if (i == 0) sv = t.space;
        if (t.space != sv || t.n != n)
            return b2k_fail(ctx, B2K_EDIM, "gkl_expand_many: V must be columns of one space of length %lld",
                            (long long)n);
    }
    const int K1 = k + nsteps;
    if (!ring_holds(ctx->dtype, K1) || K1 > 256)
        return b2k_fail(ctx, B2K_ENOTSUP, "gkl_expand_many: %d columns do not fit the sweep's panel ring", K1);
    return B2K_OK;
}

int32_t gkl_chain(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, b2k_vec* ucols, b2k_vec* vcols, int32_t k,
                  int32_t nsteps, double beta_old, double tol, int32_t alg, double* alphas_out, double* betas_out,
                  int32_t* steps_done, b2k_vec* r_out) {
    const int32_t su = B2K_VEC_SPACE(ucols[k]), sv = B2K_VEC_SPACE(vcols[0]);
    B2kChain fr(ctx, B2K_REC);                   // record i of the batch is rec_{i-1} below; the seed is rec_{-1}
    k_lanczos_seed<<<1, 1, 0, ctx->stream>>>(fr.st, beta_old, fr.stop);
    B2K_LAUNCH_CHECK(ctx);
    B2kChainCols cc(ctx, ucols[k]);
    GklFlush fl;
    memset(&fl, 0, sizeof(fl));
    int32_t enq = 0, rc = B2K_OK;
    auto fuse = [&]() {
        SpmvFuse fz;
        memset(&fz, 0, sizeof(fz));
        fz.stop = fr.stop;
        fz.l2_hints = g_l2_hints ? 1 : 0;
        fz.trace = ctx->d_trace;
        return fz;
    };
    for (int32_t i = 0; i < nsteps; ++i) {
        const int32_t K = k + i;                 // basis size before this step
        const b2k_vec R = ucols[K];
        b2k_vec Vc = -1, Uc = -1, W = -1;
        if ((rc = cc.alloc(sv, &Vc)) != B2K_OK || (rc = cc.alloc(su, &Uc)) != B2K_OK || (rc = cc.alloc(su, &W)) != B2K_OK)
            break;
        VecRef rR, rV, rU, rW, vprev;
        rc = b2k_resolve(ctx, R, &rR);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, Vc, &rV);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, Uc, &rU);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, W, &rW);
        if (rc == B2K_OK) rc = b2k_resolve(ctx, vcols[K - 1], &vprev);
        if (rc != B2K_OK) break;
        double* rec_prev = fr.st + (size_t)B2K_REC * i;
        double* rec = fr.rec0 + (size_t)B2K_REC * i;
        // 1. v~_k = A' (r / beta) - beta v_{k-1}, finishing v_{k-1} on the way (the caller's V[k-1] is final)
        SpmvFuse fa = fuse();
        fa.xscale = rec_prev + 3;
        fa.pvec = vprev.ptr;
        if (i > 0) {
            fa.pscale = rec_prev + 6;
            fa.pout = vprev.ptr;
        }
        fa.acoef = rec_prev + 2;
        if (alg == B2K_CGS2) fa.nrm_out = rec + 5;
        if ((rc = b2k_enqueue_apply_fused(ctx, At, rR, rV, 0.0, 1.0, false, nullptr, nullptr, &fa)) != B2K_OK) break;
        vcols[K] = Vc;
        if (alg == B2K_MGS2B) {                  // the flagged MGS2B: v~_k -= V V' v~_k, alpha from the finaliser
            Panel pv;
            if ((rc = make_panel(ctx, vcols, K, &pv)) != B2K_OK) break;
            rc = b2k_dispatch(ctx, [&](auto t) {
                return chain_step_gs<decltype(t)>(ctx, pv, K, rV, nullptr, rec + 3, -INFINITY, nullptr, false, 1);
            });
            if (rc != B2K_OK) break;
        }
        // 2. r' = A (v~_k / alpha) - alpha u_k, u_k = r / beta stored to its column
        SpmvFuse fb = fuse();
        fb.xscale = rec + 6;
        fb.pvec = rR.ptr;
        fb.pscale = rec_prev + 3;
        fb.pout = rU.ptr;
        fb.acoef = rec + 5;
        if ((rc = b2k_enqueue_apply_fused(ctx, A, rV, rW, 0.0, 1.0, false, nullptr, nullptr, &fb)) != B2K_OK) break;
        ucols[K] = Uc;
        // 3. r' -= U U' r', beta = ||r'||
        Panel pu;
        if ((rc = make_panel(ctx, ucols, K + 1, &pu)) != B2K_OK) break;
        rc = b2k_dispatch(ctx, [&](auto t) {
            return chain_step_gs<decltype(t)>(ctx, pu, K + 1, rW, rec_prev, rec, tol, nullptr, false, 1);
        });
        if (rc != B2K_OK) break;
        ucols[K + 1] = W;
        cc.ran(Uc, Vc, W);
        fl.col[i] = B2K_VEC_COL(Vc);
        cc.consumed(R);
        ++enq;
    }
    int32_t d = 0;
    if (enq > 0) {
        const B2kSpace& s = ctx->spaces[sv];
        fl.rec0 = fr.st; fl.tol = tol; fl.nsteps = enq; fl.ld = s.ld; fl.n = s.n;
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((s.n + 255) / 256, (int64_t)ctx->num_sms * 4));
        B2K_TRY(fr.enqueue([&]() -> int32_t {
            b2k_dispatch(ctx, [&](auto t) {
                using T = decltype(t);
                k_gkl_flush<T><<<grid, 256, 0, ctx->stream>>>((T*)s.base, fl);
            });
            B2K_LAUNCH_CHECK(ctx);
            return B2K_OK;
        }));
        B2K_TRY(fr.fetch(enq));
        d = fr.count(enq, [&](const double* r) { return gkl_step_stops(r, tol); });
        for (int32_t i = 0; i < d; ++i) {
            const double* r = fr.hrec + (size_t)B2K_REC * i;
            alphas_out[i] = r[5];
            betas_out[i] = isfinite(r[5]) ? r[2] : NAN;     // a non-finite alpha stopped the step before its beta
        }
    } else {
        fr.fail(rc);
    }
    *steps_done = d;
    *r_out = cc.commit(d, ucols, vcols, k);
    return rc;
}

}  // namespace

extern "C" int32_t b2k_gkl_expand_many(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, b2k_vec* ucols,
                                       b2k_vec* vcols, int32_t k, int32_t nsteps, double beta_old, double tol,
                                       int32_t alg, double* alphas_out, double* betas_out, int32_t* steps_done,
                                       b2k_vec* r_out) {
    if (!ctx) return B2K_EINVAL;
    if (!A || !At || !ucols || !vcols || !alphas_out || !betas_out || !steps_done || !r_out)
        return b2k_fail(ctx, B2K_EINVAL, "gkl_expand_many: null pointer");
    if (k < 1 || nsteps < 1 || nsteps > B2K_MAX_CHAIN)
        return b2k_fail(ctx, B2K_EINVAL, "gkl_expand_many: need k >= 1 and 1 <= nsteps <= %d", B2K_MAX_CHAIN);
    if (!(beta_old > 0.0) || !isfinite(beta_old))
        return b2k_fail(ctx, B2K_EINVAL, "gkl_expand_many: beta_old must be positive and finite");
    B2K_TRY(gkl_refuse(ctx, A, At, ucols, vcols, k, nsteps, alg));
    return gkl_chain(ctx, A, At, ucols, vcols, k, nsteps, beta_old, tol, alg, alphas_out, betas_out, steps_done,
                     r_out);
}

// ---------------------------------------------------------------------------------------
// Device-chained LSMR iterations (lsmr.jl:61-149), b2k_lsmr_chain.  Per iteration k, with one host synchronisation
// per call:
//   1. A SpMV (m rows): gathers v_k = rn(src * (1/alpha_k)) (xscale) into the work column Av;
//   2. k_lsmr_m: iteration k-1's Ah-bar / r tail, Ah, u~_{k+1} = Av - alpha_k u_k, beta_{k+1} (last CTA);
//   3. A' SpMV (n rows): gathers u_{k+1} = rn(u~ * (1/beta)); does nothing when beta <= tol (skip flag);
//   4. k_lsmr_n: v_k into its ring slot, iteration k-1's h-bar / x / h tail, v~_{k+1} = y - beta v_k in the spare
//      column; without reorthogonalisation it also sums v~^2 and runs the scalar recurrence in its last CTA;
//   5. (krylovdim > 1) the reorthogonalisation of v~_{k+1} against the ring in slot order — the pipelined MGS sweep
//      once or twice, or two passes of the cooperative classical sweep — then k_lsmr_alpha: alpha and the recurrence.
// Two flush launches (one per side) apply the tail of the last iteration that ran and normalise u and v.
namespace {

int32_t lsmr_refuse(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, const VecRef* mv, const VecRef* nv,
                    const VecRef* rr, int nring, int32_t krylovdim, int32_t alg) {
    if (ctx->nranks > 1) return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: row-sharded contexts are not supported");
    int64_t m = 0, n = 0, tm = 0, tn = 0;
    int32_t ka = -1, kt = -1;
    B2K_TRY(b2k_op_info(A, &m, &n, nullptr, &ka));
    B2K_TRY(b2k_op_info(At, &tm, &tn, nullptr, &kt));
    if (ka != 0 || kt != 0) return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: A and A' must be stored CSR matrices");
    const bool gs = alg == B2K_CGS2 || alg == B2K_MGS2B;
    if (krylovdim > 1) {
        if (alg != B2K_MGS && alg != B2K_MGS2 && !gs)
            return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: orthogonalizer %d does not chain with krylovdim > 1", alg);
        if (gs && (!g_use_coop || !ring_holds(ctx->dtype, nring)))
            return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: %d ring columns do not fit the sweep's panel ring", nring);
    }
    if (nring > LS_MAXRING)
        return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: krylovdim %d > %d", krylovdim, LS_MAXRING);
    if (tm != n || tn != m)
        return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: A' is %lld x %lld, A is %lld x %lld", (long long)tm, (long long)tn,
                        (long long)m, (long long)n);
    for (int i = 0; i < 5; ++i)
        if (mv[i].n != m) return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: r, Ah, Ah-bar, u, Av must have length %lld",
                                          (long long)m);
    for (int i = 0; i < 4; ++i)
        if (nv[i].n != n) return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: x, h, h-bar, spare must have length %lld",
                                          (long long)n);
    for (int i = 1; i < 5; ++i)
        if (mv[i].space != mv[0].space)
            return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: r, Ah, Ah-bar, u, Av must be columns of one space");
    for (int i = 0; i < 3; ++i)
        if (nv[i].space != nv[3].space)
            return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: x, h, h-bar and the spare must be columns of one space");
    for (int i = 0; i < nring; ++i)
        if (rr[i].n != n || rr[i].space != nv[3].space)
            return b2k_fail(ctx, B2K_EDIM, "lsmr_chain: the ring and the spare column must be columns of one space of "
                                           "length %lld", (long long)n);
    // every vector is written by some launch while others read: no two handles may share storage
    std::vector<const VecRef*> all;
    for (int i = 0; i < 5; ++i) all.push_back(mv + i);
    for (int i = 0; i < 4; ++i) all.push_back(nv + i);
    for (int i = 0; i < nring; ++i) all.push_back(rr + i);
    for (size_t i = 0; i < all.size(); ++i)
        for (size_t j = 0; j < i; ++j)
            if (all[i]->ptr == all[j]->ptr)
                return b2k_fail(ctx, B2K_EINVAL, "lsmr_chain: vectors %zu and %zu are the same", j, i);
    return B2K_OK;
}

}  // namespace

extern "C" int32_t b2k_lsmr_chain(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, b2k_vec x, b2k_vec h,
                                  b2k_vec hbar, b2k_vec r, b2k_vec Ah, b2k_vec Ahbar, b2k_vec u, b2k_vec av,
                                  const b2k_vec* ring, int32_t krylovdim, b2k_vec spare, int32_t alg, int32_t iter0,
                                  const double* state_in, double tol, int32_t nsteps, double* rec_out,
                                  double* state_out, int32_t* steps_done) {
    if (!ctx) return B2K_EINVAL;
    if (!A || !At || !ring || !state_in || !rec_out || !state_out || !steps_done)
        return b2k_fail(ctx, B2K_EINVAL, "lsmr_chain: null pointer");
    if (nsteps < 1 || nsteps > B2K_MAX_CHAIN - 1 || iter0 < 0)
        return b2k_fail(ctx, B2K_EINVAL, "lsmr_chain: need 1 <= nsteps <= %d and iter0 >= 0", B2K_MAX_CHAIN - 1);
    const int nring = krylovdim > 1 ? krylovdim : 1;
    if (nring > LS_MAXRING) return b2k_fail(ctx, B2K_ENOTSUP, "lsmr_chain: krylovdim %d > %d", krylovdim, LS_MAXRING);
    VecRef mv[5], nv[4];
    std::vector<VecRef> rr(nring);
    const b2k_vec mh[5] = {r, Ah, Ahbar, u, av}, nh[4] = {x, h, hbar, spare};
    for (int i = 0; i < 5; ++i) B2K_TRY(b2k_resolve(ctx, mh[i], &mv[i]));
    for (int i = 0; i < 4; ++i) B2K_TRY(b2k_resolve(ctx, nh[i], &nv[i]));
    for (int i = 0; i < nring; ++i) B2K_TRY(b2k_resolve(ctx, ring[i], &rr[i]));
    B2K_TRY(lsmr_refuse(ctx, A, At, mv, nv, rr.data(), nring, krylovdim, alg));
    *steps_done = 0;
    const int64_t m = mv[0].n, n = nv[0].n;
    B2kChain fr(ctx, LS_NSTATE, LS_REC);
    LsmrDev d;
    memset(&d, 0, sizeof(d));
    d.st = fr.st;
    d.rec0 = fr.rec0;
    d.stop = fr.stop;
    d.skip = fr.skip;
    d.tol = tol;
    d.iter0 = iter0;
    d.nring = nring;
    for (int i = 0; i < nring; ++i) d.ring[i] = rr[i].ptr;
    double seed[LS_NSTATE] = {};
    memcpy(seed, state_in, LS_NIO * sizeof(double));
    seed[LS_INVA] = 1.0;                           // u and v are normalised on entry
    seed[LS_INVB] = 1.0;
    B2K_TRY(fr.seed(seed, LS_NSTATE, nsteps, true));
    SpmvFuse fa, ft;
    memset(&fa, 0, sizeof(fa));
    fa.stop = d.stop;
    fa.xscale = d.st + LS_INVA;
    ft = fa;
    ft.stop = d.skip;
    ft.xscale = d.st + LS_INVB;
    const bool reorth = krylovdim > 1;
    // nothing is reported from a call that could not be enqueued
    B2K_TRY(fr.enqueue([&]() -> int32_t {
        for (int32_t i = 0; i < nsteps; ++i) {
            const int k = iter0 + 1 + i;               // v_k sits (or will sit) in ring slot (k - 1) % nring
            const VecRef& P = rr[(k - 1) % nring];
            const VecRef& src = i == 0 ? P : nv[3];
            const VecRef& yv = i == 0 ? nv[3] : P;
            B2K_TRY(b2k_enqueue_apply_fused(ctx, A, src, mv[4], 0.0, 1.0, false, nullptr, nullptr, &fa));
            B2K_TRY(b2k_lsmr_enqueue_m(ctx, m, mv[0].ptr, mv[1].ptr, mv[2].ptr, mv[3].ptr, mv[4].ptr, i > 0, false, d));
            B2K_TRY(b2k_enqueue_apply_fused(ctx, At, mv[3], yv, 0.0, 1.0, false, nullptr, nullptr, &ft));
            B2K_TRY(b2k_lsmr_enqueue_n(ctx, n, nv[0].ptr, nv[1].ptr, nv[2].ptr, P.ptr, nv[3].ptr, i > 0, i > 0, !reorth,
                                       d));
            if (!reorth) continue;
            const int cnt = std::min(krylovdim, k);    // V holds v_1 .. v_k, at most krylovdim of them, in slot order
            Panel pn;
            B2K_TRY(make_panel(ctx, ring, cnt, &pn));
            if (alg == B2K_MGS || alg == B2K_MGS2) {
                ctx->dot_stop = d.skip;
                int32_t rc = mgs_sweep(ctx, pn, nv[3], cnt, 0, -1);
                if (rc == B2K_OK && alg == B2K_MGS2) rc = mgs_sweep(ctx, pn, nv[3], cnt, cnt, -1);
                ctx->dot_stop = nullptr;
                B2K_TRY(rc);
            } else {                                   // orthogonalize!! with CGS2: two classical passes
                for (int ps = 0; ps < 2; ++ps)
                    B2K_TRY(b2k_dispatch(ctx, [&](auto t) {
                        return chain_step_gs<decltype(t)>(ctx, pn, cnt, nv[3], nullptr, d.st + LS_FIN, -INFINITY,
                                                          nullptr, false, 0, d.skip);
                    }));
            }
            B2K_TRY(b2k_lsmr_enqueue_alpha(ctx, n, nv[3].ptr, d));
        }
        B2K_TRY(b2k_lsmr_enqueue_m(ctx, m, mv[0].ptr, mv[1].ptr, mv[2].ptr, mv[3].ptr, nullptr, true, true, d));
        return b2k_lsmr_enqueue_flush_n(ctx, n, nv[0].ptr, nv[1].ptr, nv[2].ptr, nv[3].ptr, d);
    }));
    static_assert(LS_NIO <= LS_NSTATE, "state block");
    B2K_TRY(fr.fetch(nsteps, LS_NIO));
    const int32_t dn = fr.count(nsteps, [](const double* rec) { return rec[7] != 0.0; });
    memcpy(rec_out, fr.hrec, sizeof(double) * LS_REC * dn);
    memcpy(state_out, fr.hst, sizeof(double) * LS_NIO);
    *steps_done = dn;
    return B2K_OK;
}

extern "C" int32_t b2k_basis_transform(b2k_ctx* ctx, const b2k_vec* cols, int32_t m,
                                       const double* U_host, int32_t ldu, int32_t keep) {
    if (!ctx || !cols || !U_host || m < 1 || keep < 1 || keep > m || ldu < m) return B2K_EINVAL;
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, m, &pn));
    {   // a column listed twice would be two outputs in one storage, written by different threads
        std::vector<uint8_t> seen(ctx->spaces[B2K_VEC_SPACE(cols[0])].ncols, 0);
        for (int i = 0; i < m; ++i) {
            if (seen[pn.idx[i]])
                return b2k_fail(ctx, B2K_EINVAL, "basis_transform: column %d is listed twice", pn.idx[i]);
            seen[pn.idx[i]] = 1;
        }
    }
    const bool f64 = ctx->dtype == B2K_F64;
    const int C = f64 ? 8 : 16;
    if (m > 256)
        return b2k_fail(ctx, B2K_ENOTSUP, "basis_transform: m = %d exceeds the supported basis width (256)", m);
    const bool wide = (m + C - 1) / C > NS;       // does not fit the resident ring: staged-tile kernel
    if ((size_t)m * keep > B2K_COEF_DOUBLES)
        return b2k_fail(ctx, B2K_ENOTSUP, "basis_transform: U too large");
    // pack U densely (ldu -> m)
    std::vector<double> Up((size_t)m * keep);
    for (int j = 0; j < keep; ++j)
        for (int i = 0; i < m; ++i) Up[(size_t)j * m + i] = U_host[(size_t)j * ldu + i];
    B2K_TRY(b2k_put_coef(ctx, Up.data(), m * keep, 0));
    TransformParams p;
    p.base = pn.base; p.ld = pn.ld; p.n = pn.n; p.m = m; p.keep = keep; p.ldu = m;
    p.U = ctx->d_coef;
    {
        const int vec = f64 ? 2 : 4;
        const size_t pitch = (size_t)((keep + vec - 1) / vec) * vec;
        p.u_in_smem = ((size_t)m * pitch * ctx->esize <= (size_t)TR_U_BYTES) ? 1 : 0;
    }
    ColList cl;
    for (int i = 0; i < m; ++i) cl.c[i] = pn.idx[i];
    const int pr = b2k_prof_begin(ctx, 2, (double)(m + keep) * ctx->esize * (double)pn.n);
    const bool dmma_ok = f64 && g_use_dmma && (size_t)m * (((keep + 7) / 8) * 8) * 8 <= (size_t)TD_U_BYTES;
    if (wide) {
        const int64_t ntiles = (pn.n + TB_ROWS - 1) / TB_ROWS;
        const size_t smem = (size_t)TB_ROWS * m * ctx->esize;
        const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(200 * 1024) / smem));
        const int grid = (int)std::min<int64_t>(ntiles, (int64_t)ctx->num_sms * per_sm);
        g_transform_kernel = f64 ? 5 : 6;
        if (f64) k_transform_big<double><<<grid, TB_THREADS, smem, ctx->stream>>>(p, cl);
        else k_transform_big<float><<<grid, TB_THREADS, smem, ctx->stream>>>(p, cl);
    } else if (f64 && g_transform_ur && keep <= UR_J && m <= UR_MAXM) {
        UPar up;                                          // by-value kernel parameter: copied at launch
        memset(&up, 0, sizeof(up));
        for (int j = 0; j < keep; ++j)
            for (int i = 0; i < m; ++i) up.u[i * UR_J + j] = U_host[(size_t)j * ldu + i];
        const int grid = grid_for_rows<double>(ctx, pn.n);
        g_transform_kernel = 6 + g_transform_ur;
        if (g_transform_ur == 1) k_transform_ur<2, 18><<<grid, TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl, up);
        else if (g_transform_ur == 2) k_transform_ur<2, 36><<<grid, TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl, up);
        else k_transform_ur<4, 18><<<grid, TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl, up);
    } else if (f64 && g_transform_hyb == 3 && keep <= F89_G * F89_TH &&
               (size_t)F89_G * m * F89_UP * 8 <= (size_t)TR_U_BYTES - 64) {
        const int64_t nt = (pn.n + F89W_R - 1) / F89W_R;
        g_transform_kernel = 11;
        k_transform_f89w<<<(int)std::max<int64_t>(1, std::min<int64_t>(nt, ctx->num_sms)), F89_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
    } else if (f64 && g_transform_hyb == 2 && keep <= F89_G * F89_TH &&
               (size_t)F89_G * m * F89_UP * 8 <= (size_t)TR_U_BYTES - 64) {
        g_transform_kernel = 10;
        k_transform_f89<<<grid_for_rows<double>(ctx, pn.n), F89_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
    } else if (dmma_ok && g_transform_hyb == 1 && keep <= TH_MAXKEEP && (size_t)m * 40 * 8 <= (size_t)TD_U_BYTES) {
        g_transform_kernel = 12;
        k_transform_hyb<<<grid_for_rows<double>(ctx, pn.n), TR_THREADS, TD_SMEM, ctx->stream>>>(p, cl);
    } else if (dmma_ok) {
        g_transform_kernel = 13;
        k_transform_dmma<<<grid_for_rows<double>(ctx, pn.n), TR_THREADS, TD_SMEM, ctx->stream>>>(p, cl);
    } else if (f64) {
        g_transform_kernel = p.u_in_smem ? 1 : 2;
        if (p.u_in_smem) k_transform<double, true><<<grid_for_rows<double>(ctx, pn.n), TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
        else k_transform<double, false><<<grid_for_rows<double>(ctx, pn.n), TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
    } else {
        g_transform_kernel = p.u_in_smem ? 3 : 4;
        if (p.u_in_smem) k_transform<float, true><<<grid_for_rows<float>(ctx, pn.n), TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
        else k_transform<float, false><<<grid_for_rows<float>(ctx, pn.n), TR_THREADS, TR_SMEM, ctx->stream>>>(p, cl);
    }
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

extern "C" int32_t b2k_basis_rank1update(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, b2k_vec y,
                                         const double* x_host, double alpha, double beta) {
    if (!ctx || (k > 0 && (!cols || !x_host))) return B2K_EINVAL;
    if (k == 0) return B2K_OK;
    Panel pn;
    B2K_TRY(make_panel(ctx, cols, k, &pn));
    VecRef ry;
    B2K_TRY(b2k_resolve(ctx, y, &ry));
    if (ry.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "basis_rank1update: length mismatch");
    const int grid = std::max(1, (int)std::min<int64_t>((pn.n + 255) / 256, (int64_t)ctx->num_sms * 8));
    for (int off = 0; off < k; off += 256) {
        const int kk = std::min(256, k - off);
        ColList cl;
        CoefList cf;
        for (int i = 0; i < kk; ++i) {
            cl.c[i] = pn.idx[off + i];
            cf.c[i] = alpha * x_host[off + i];   // real: conj(x) = x
        }
        const int bm = beta == 1.0 ? 1 : (beta == 0.0 ? 0 : 2);
        b2k_dispatch(ctx, [&](auto t) {
            using T = decltype(t);
            k_rank1<T><<<grid, 256, 0, ctx->stream>>>((T*)pn.base, pn.ld, pn.n, kk, (const T*)ry.ptr, T(beta), bm, cl, cf);
        });
        B2K_LAUNCH_CHECK(ctx);
    }
    return B2K_OK;
}

// rmul!(b, H::Householder) — src/dense/reflector.jl:143-154
extern "C" int32_t b2k_basis_householder(b2k_ctx* ctx, const b2k_vec* cols, int32_t k,
                                         const double* v_host, double beta, b2k_vec work) {
    if (!ctx) return B2K_EINVAL;
    if (beta == 0.0 || k == 0) return B2K_OK;   // iszero(β) && return b
    B2K_TRY(b2k_basis_unproject(ctx, work, cols, k, v_host, 1.0, 0.0));
    return b2k_basis_rank1update(ctx, cols, k, work, v_host, -beta, 1.0);
}

// ------------------------------------------------------------------ block ops ----

// b2k_block_inner / b2k_block_axpy: multi-right-hand-side kernels, block.cu

extern "C" int32_t b2k_block_reorthogonalize(b2k_ctx* ctx, const b2k_vec* Rb, int32_t p,
                                             const b2k_vec* V, int32_t k) {
    if (!ctx || !Rb || p < 1) return B2K_EINVAL;
    if (k == 0) return B2K_OK;
    Panel pn;
    B2K_TRY(make_panel(ctx, V, k, &pn));
    if (k > B2K_RES_DOUBLES - 8) return b2k_fail(ctx, B2K_ENOTSUP, "block_reorthogonalize: k too large");
    for (int i = 0; i < p; ++i) {
        VecRef rv;
        B2K_TRY(b2k_resolve(ctx, Rb[i], &rv));
        if (rv.n != pn.n) return b2k_fail(ctx, B2K_EDIM, "block_reorthogonalize: length mismatch");
        B2K_TRY(mgs_sweep(ctx, pn, rv, k, 0, -1));
    }
    return B2K_OK;
}

// block_qr!(block, tol) — src/factorizations/blocklanczos.jl:312-353
extern "C" int32_t b2k_block_qr(b2k_ctx* ctx, const b2k_vec* X, int32_t p, double tol,
                                double* R_host, int32_t* good, int32_t* drift) {
    if (!ctx || !X || !R_host || !good || !drift || p < 1) return B2K_EINVAL;
    for (int i = 0; i < p * p; ++i) R_host[i] = 0.0;
    *drift = 0;
    double nrm;
    B2K_TRY(b2k_vec_norm(ctx, X[0], &nrm));   // β = sqrt(real(inner(block[1], block[1])))
    if (nrm > tol) {
        R_host[0] = nrm;
        B2K_TRY(b2k_vec_scale(ctx, X[0], X[0], 1.0 / nrm));
        good[0] = 1;
    } else {
        B2K_TRY(b2k_vec_zero(ctx, X[0]));
        good[0] = 0;
    }
    std::vector<double> h(p);
    for (int j = 1; j < p; ++j) {
        double beta;
        int32_t passes;
        B2K_TRY(b2k_basis_orthogonalize(ctx, X[j], X, j, h.data(), B2K_MGS, 0.0, &beta, &passes));
        for (int i = 0; i < j; ++i) R_host[(size_t)j * p + i] = h[i];
        if (tol < beta && beta < 100 * tol) {   // DGKS reorthogonalisation
            *drift = 1;
            B2K_TRY(b2k_basis_orthogonalize(ctx, X[j], X, j, h.data(), B2K_MGS, 0.0, &beta, &passes));
            for (int i = 0; i < j; ++i) R_host[(size_t)j * p + i] += h[i];
        }
        if (beta < tol) {
            B2K_TRY(b2k_vec_zero(ctx, X[j]));
            good[j] = 0;
        } else {
            R_host[(size_t)j * p + j] = beta;
            B2K_TRY(b2k_vec_scale(ctx, X[j], X[j], 1.0 / beta));
            good[j] = 1;
        }
    }
    return B2K_OK;
}

// Event trace of the chained Lanczos step (tools/trace_step.py).  on != 0 allocates / clears the buffer and makes the
// kernels of b2k_lanczos_expand_many record (globaltimer ns, code) pairs: SpMV 1 begin, 2 halo rows present, 3 CTA 0
// done, 4 <v, Av> published by the last CTA; sweep 10 begin, 11 alpha present, 12 + i CTA 0 finished phase i,
// 15 + i CTA 0 left boundary i, 18/19 the last CTA enters / leaves the finaliser.
extern "C" int32_t b2k_debug_trace(b2k_ctx* ctx, int32_t on) {
    if (!ctx) return B2K_EINVAL;
    if (on) {
        if (!ctx->d_trace) B2K_CUDA(ctx, cudaMalloc(&ctx->d_trace, sizeof(unsigned long long) * (2 + 2 * B2K_TRACE_CAP)));
        B2K_CUDA(ctx, cudaMemsetAsync(ctx->d_trace, 0, sizeof(unsigned long long) * 2, ctx->stream));
    } else if (ctx->d_trace) {
        B2K_TRY(b2k_stream_sync(ctx));
        cudaFree(ctx->d_trace);
        ctx->d_trace = nullptr;
    }
    return B2K_OK;
}

extern "C" int32_t b2k_debug_trace_read(b2k_ctx* ctx, unsigned long long* out, int64_t cap_events, int64_t* n_events) {
    if (!ctx || !out || !n_events) return B2K_EINVAL;
    *n_events = 0;
    if (!ctx->d_trace) return B2K_OK;
    B2K_TRY(b2k_stream_sync(ctx));
    unsigned long long cnt = 0;
    B2K_CUDA(ctx, cudaMemcpy(&cnt, ctx->d_trace, sizeof(cnt), cudaMemcpyDeviceToHost));
    if (cnt > B2K_TRACE_CAP) cnt = B2K_TRACE_CAP;
    if ((int64_t)cnt > cap_events) cnt = (unsigned long long)cap_events;
    B2K_CUDA(ctx, cudaMemcpy(out, ctx->d_trace + 2, sizeof(unsigned long long) * 2 * cnt, cudaMemcpyDeviceToHost));
    *n_events = (int64_t)cnt;
    return B2K_OK;
}

// ------------------------------------------------------------------ cross Gram ----
// b2k_basis_cross_inner: G[i, j] = <X[i], Y[j]> for two lists of columns, in ONE sweep over the rows per column block.
//
// A column block is at most CI_B = 64 columns of X times at most CI_B columns of Y (the single-pass limit: 256 threads
// x a 4 x 4 register tile = 64 x 64 accumulators; it does not depend on the dtype).  Larger lists are split into
// ceil(p/64) x ceil(q/64) blocks and each block is one sweep that reads its own X and Y columns, so a split call
// reads  sum over blocks of (pb + qb) n sizeof(T)  bytes = (ceil(q/64) p + ceil(p/64) q) n sizeof(T)  instead of
// (p + q) n sizeof(T).  Blocks that lie wholly inside the skip block are not swept.
//
// Kernel: one CTA per SM (grid = min(ceil(n / 64), #SMs)), CTA g owns row tiles g, g + grid, ... of CI_R = 64 rows.
// A producer warp streams each tile's pb + qb column segments into a ring of shared-memory stages with 1-D TMA bulk
// copies (one per column, completion on the stage's mbarrier, as in tsk.cuh); 8 consumer warps form the tile's
// X_tile' Y_tile contribution in registers.  Consumer thread t = s * NO + o owns the 16 entries of entry tile
// o = (oi, oj) — rows oi + a OI, columns oj + b OJ of the block, a, b < 4, OI = ceil(pb/4), OJ = ceil(qb/4),
// NO = OI OJ — and row slice s < RS, where RS is the largest power of two <= min(32, 256 / NO): it reads the rows
// r of the tile with r % RS == s.  Shared memory: nst (pb + qb) (64 + pad) sizeof(T) for the ring
// (pad = 16 bytes, which spreads the columns of one row over the banks), plus 16 RS NO doubles for the slice sums.
//
// Rounding contract (the PROJECT phase of tsk.cuh): a thread accumulates its rows in the vector type T with an fma
// chain, a = fma(X[r, i], Y[r, j], a) from a = 0, over its tiles in ascending order and its rows of each tile in
// ascending order; the RS slice values of an entry are converted to double and added in slice order (from 0.0), and
// the per-CTA values are added in CTA order (from 0.0) by k_cross_finalize.  No FP atomics: the bits depend only on
// n, p, q, the column block and the number of SMs.  Launches per call: 2 per column block that is swept (the sweep
// and k_cross_finalize); none when n == 0 or everything is skipped.  One host synchronisation per call.
namespace {

constexpr int CI_B = 64;                 // columns of X / of Y per block (the single-pass limit)
constexpr int CI_R = 64;                 // rows per tile
constexpr int CI_THREADS = 256 + 32;     // 8 consumer warps + 1 producer warp
constexpr int CI_PART = CI_B * CI_B;     // doubles per CTA partial block
constexpr int CI_SMEM_MAX = 232448;
constexpr int CI_MAXLIST = 256;

template <typename T> constexpr int ci_pitch() { return CI_R + 16 / (int)sizeof(T); }

template <typename T>
struct CrossParams {
    const T* x[CI_B];
    const T* y[CI_B];
    int64_t n;
    int pb, qb;          // block shape
    int oj, no, rs;      // owner tiles per row of tiles, owner tiles, row slices
    int skip_i, skip_j;  // entries (i < skip_i, j < skip_j) of the block are not wanted
    int nst;             // ring stages
    double* part;        // [grid][CI_PART]
};

template <typename T>
__global__ void __launch_bounds__(CI_THREADS, 1) k_cross_inner(const __grid_constant__ CrossParams<T> p) {
    extern __shared__ __align__(128) uint8_t ci_smem[];
    constexpr int P = ci_pitch<T>();
    const int ncol = p.pb + p.qb;
    const uint32_t stage_bytes = (uint32_t)(ncol * P * sizeof(T));
    double* red = reinterpret_cast<double*>(ci_smem + (size_t)p.nst * stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(red + 16 * p.rs * p.no);
    const uint32_t full = smem_u32(bars), empty = full + 8 * p.nst;
    const uint32_t ring = smem_u32(ci_smem);
    const int tid = threadIdx.x;
    const int64_t ntiles = (p.n + CI_R - 1) / CI_R;
    if (tid == 0) {
        for (int i = 0; i < p.nst; ++i) {
            mbar_init(full + 8 * i, 1);
            mbar_init(empty + 8 * i, 8);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (tid >= 256) {     // producer warp
        const int lane = tid & 31;
        int it = 0;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
            const int s = it % p.nst;
            const uint32_t ph = (uint32_t)((it / p.nst) & 1);
            mbar_wait(empty + 8 * s, ph ^ 1);
            const int64_t r0 = tile * CI_R;
            const int rt = (int)((p.n - r0) < CI_R ? (p.n - r0) : CI_R);
            const uint32_t bytes = (uint32_t)((rt * sizeof(T) + 15) & ~(size_t)15);
            if (lane == 0) mbar_expect_tx(full + 8 * s, bytes * (uint32_t)ncol);
            __syncwarp();
            for (int c = lane; c < ncol; c += 32) {
                const T* src = (c < p.pb ? p.x[c] : p.y[c - p.pb]) + r0;
                bulk_g2s(ring + s * stage_bytes + c * P * (uint32_t)sizeof(T), src, bytes, full + 8 * s);
            }
        }
        return;
    }

    // consumers
    const int lane = tid & 31;
    const int sl = tid / p.no, o = tid % p.no;
    const bool active = sl < p.rs;
    // entry tile o = (oi, oj) holds the entries (oi + a OI, oj + b OJ): the lanes of a warp read neighbouring
    // columns, whose segments the 16-byte pad spreads over the banks
    const int OI = p.no / p.oj;
    const int oi = o / p.oj, oj = o % p.oj;
    // a tile wholly inside the skip block does no arithmetic
    const bool work = active && !(oi + 3 * OI < p.skip_i && oj + 3 * p.oj < p.skip_j);
    int xi[4], yj[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        xi[a] = min(oi + a * OI, p.pb - 1) * P;                // clamped: entries past the block are discarded
        yj[a] = (p.pb + min(oj + a * p.oj, p.qb - 1)) * P;
    }
    T acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = (T)0;
    int it = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int s = it % p.nst;
        const uint32_t ph = (uint32_t)((it / p.nst) & 1);
        mbar_wait(full + 8 * s, ph);
        const int64_t r0 = tile * CI_R;
        const int rt = (int)((p.n - r0) < CI_R ? (p.n - r0) : CI_R);
        const T* st = reinterpret_cast<const T*>(ci_smem + (size_t)s * stage_bytes);
        if (work) {
            for (int r = sl; r < rt; r += p.rs) {
                T xv[4], yv[4];
#pragma unroll
                for (int a = 0; a < 4; ++a) { xv[a] = st[xi[a] + r]; yv[a] = st[yj[a] + r]; }
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = fma(xv[a], yv[b], acc[a][b]);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + 8 * s);
    }

    // slice sums in slice order, in double
    if (active) {
        double* mine = red + (size_t)(sl * p.no + o) * 16;
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) mine[a * 4 + b] = (double)acc[a][b];
    }
    named_bar_sync(1, 256);
    double* part = p.part + (size_t)blockIdx.x * CI_PART;
    for (int e = tid; e < p.pb * p.qb; e += 256) {
        const int i = e % p.pb, j = e / p.pb;
        const int OI = p.no / p.oj;
        const int oo = (i % OI) * p.oj + j % p.oj, ab = (i / OI) * 4 + j / p.oj;
        double v = 0.0;
        for (int s2 = 0; s2 < p.rs; ++s2) v += red[(size_t)(s2 * p.no + oo) * 16 + ab];
        part[e] = v;
    }
}

// G[(j0 + j) * ldg + i0 + i] = sum over CTAs g in order of part[g][i + j pb], outside the skip block
__global__ void __launch_bounds__(256) k_cross_finalize(const double* __restrict__ part, int grid, int pb, int qb,
                                                        int i0, int j0, int p0, int q0, double* __restrict__ G,
                                                        int ldg) {
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= pb * qb) return;
    const int i = e % pb, j = e / pb;
    if (i0 + i < p0 && j0 + j < q0) return;
    double v = 0.0;
    for (int g = 0; g < grid; ++g) v += part[(size_t)g * CI_PART + e];
    G[(size_t)(j0 + j) * ldg + i0 + i] = v;
}

template <typename T>
int32_t cross_block(b2k_ctx* ctx, const std::vector<VecRef>& X, const std::vector<VecRef>& Y, int i0, int pb,
                    int j0, int qb, int p0, int q0, int64_t n, double* d_part, double* d_G, int ldg) {
    CrossParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    for (int i = 0; i < pb; ++i) cp.x[i] = (const T*)X[i0 + i].ptr;
    for (int j = 0; j < qb; ++j) cp.y[j] = (const T*)Y[j0 + j].ptr;
    cp.n = n;
    cp.pb = pb;
    cp.qb = qb;
    cp.oj = (qb + 3) / 4;
    cp.no = ((pb + 3) / 4) * cp.oj;
    cp.rs = 1;
    while (cp.rs * 2 <= 32 && cp.rs * 2 * cp.no <= 256) cp.rs *= 2;
    cp.skip_i = std::max(0, std::min(p0 - i0, pb));
    cp.skip_j = std::max(0, std::min(q0 - j0, qb));
    const size_t stage = (size_t)(pb + qb) * ci_pitch<T>() * sizeof(T);
    const size_t red = (size_t)16 * cp.rs * cp.no * sizeof(double);
    cp.nst = (int)std::max<size_t>(2, std::min<size_t>(6, (200 * 1024 - red) / stage));
    const size_t smem = cp.nst * stage + red + 16 * (size_t)cp.nst;
    if (smem > (size_t)CI_SMEM_MAX) return b2k_fail(ctx, B2K_ENOTSUP, "basis_cross_inner: shared memory");
    const int64_t ntiles = (n + CI_R - 1) / CI_R;
    const int grid = (int)std::min<int64_t>(ntiles, ctx->num_sms);
    cp.part = d_part;
    const int pr = b2k_prof_begin(ctx, 9, (double)(pb + qb) * sizeof(T) * (double)n);
    k_cross_inner<T><<<grid, CI_THREADS, smem, ctx->stream>>>(cp);
    B2K_LAUNCH_CHECK(ctx);
    b2k_prof_end(ctx, pr);
    k_cross_finalize<<<(pb * qb + 255) / 256, 256, 0, ctx->stream>>>(d_part, grid, pb, qb, i0, j0, p0, q0, d_G, ldg);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

}  // namespace

int32_t b2k_cross_init(b2k_ctx* ctx) {
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_cross_inner<double>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       CI_SMEM_MAX));
    B2K_CUDA(ctx, cudaFuncSetAttribute(k_cross_inner<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       CI_SMEM_MAX));
    return B2K_OK;
}

extern "C" int32_t b2k_basis_cross_inner(b2k_ctx* ctx, const b2k_vec* X, int32_t p, const b2k_vec* Y, int32_t q,
                                         int32_t p0, int32_t q0, double* G_host, int32_t ldg) {
    if (!ctx || !X || !Y || !G_host) return B2K_EINVAL;
    if (p < 1 || q < 1 || p > CI_MAXLIST || q > CI_MAXLIST || p0 < 0 || p0 > p || q0 < 0 || q0 > q || ldg < p)
        return b2k_fail(ctx, B2K_EINVAL, "basis_cross_inner: need 1 <= p, q <= %d, 0 <= p0 <= p, 0 <= q0 <= q, "
                                         "ldg >= p (p = %d, q = %d, p0 = %d, q0 = %d, ldg = %d)",
                        CI_MAXLIST, p, q, p0, q0, ldg);
    if (ctx->nranks > 1)
        return b2k_fail(ctx, B2K_ENOTSUP, "basis_cross_inner: row-sharded contexts are not supported");
    std::vector<VecRef> xr(p), yr(q);
    for (int i = 0; i < p; ++i) B2K_TRY(b2k_resolve(ctx, X[i], &xr[i]));
    for (int j = 0; j < q; ++j) B2K_TRY(b2k_resolve(ctx, Y[j], &yr[j]));
    const int64_t n = xr[0].n;
    for (const VecRef& v : xr)
        if (v.n != n) return b2k_fail(ctx, B2K_EDIM, "basis_cross_inner: columns of %lld and %lld rows",
                                      (long long)n, (long long)v.n);
    for (const VecRef& v : yr)
        if (v.n != n) return b2k_fail(ctx, B2K_EDIM, "basis_cross_inner: columns of %lld and %lld rows",
                                      (long long)n, (long long)v.n);
    if (p0 == p && q0 == q) return B2K_OK;
    if (n == 0) {
        for (int j = 0; j < q; ++j)
            for (int i = 0; i < p; ++i)
                if (!(i < p0 && j < q0)) G_host[(size_t)j * ldg + i] = 0.0;
        return B2K_OK;
    }
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    const int grid = (int)std::min<int64_t>((n + CI_R - 1) / CI_R, ctx->num_sms);
    double *d_part = nullptr, *d_G = nullptr, *h_G = nullptr;
    const size_t gbytes = sizeof(double) * CI_MAXLIST * CI_MAXLIST;
    auto release = [&]() {
        if (d_part) B2K_DFREE(d_part);
        if (d_G) B2K_DFREE(d_G);
        if (h_G) b2k_hfree(h_G, gbytes);
    };
    int32_t rc = B2K_OK;
    if (B2K_DMALLOC(&d_part, sizeof(double) * (size_t)grid * CI_PART) != cudaSuccess ||
        B2K_DMALLOC(&d_G, sizeof(double) * (size_t)p * q) != cudaSuccess || b2k_hmalloc((void**)&h_G, gbytes) != cudaSuccess)
        rc = b2k_fail(ctx, B2K_ENOMEM, "basis_cross_inner: staging allocation failed");
    for (int i0 = 0; rc == B2K_OK && i0 < p; i0 += CI_B)
        for (int j0 = 0; rc == B2K_OK && j0 < q; j0 += CI_B) {
            const int pb = std::min(CI_B, p - i0), qb = std::min(CI_B, q - j0);
            if (i0 + pb <= p0 && j0 + qb <= q0) continue;
            rc = b2k_dispatch(ctx, [&](auto t) {
                return cross_block<decltype(t)>(ctx, xr, yr, i0, pb, j0, qb, p0, q0, n, d_part, d_G, p);
            });
        }
    if (rc == B2K_OK) {
        const cudaError_t e = cudaMemcpyAsync(h_G, d_G, sizeof(double) * (size_t)p * q, cudaMemcpyDeviceToHost,
                                              ctx->stream);
        if (e != cudaSuccess) rc = b2k_fail(ctx, B2K_ECUDA, "basis_cross_inner: %s", cudaGetErrorString(e));
    }
    if (rc == B2K_OK) rc = b2k_stream_sync(ctx);
    if (rc == B2K_OK)
        for (int j = 0; j < q; ++j)
            for (int i = 0; i < p; ++i)
                if (!(i < p0 && j < q0)) G_host[(size_t)j * ldg + i] = h_G[(size_t)j * p + i];
    release();
    return rc;
}
