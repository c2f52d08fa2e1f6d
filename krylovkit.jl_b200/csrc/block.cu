// block.cu — the block path (SURVEY §8f-3): multi-right-hand-side tall-skinny products for
// BlockLanczos.  The reference runs its block primitives as loops of single-vector calls
// (src/factorizations/blocklanczos.jl:43-52 block_inner, :232-263 block_lanczosrecurrence, :277-284
// block_reorthogonalize!, :312-353 block_qr!); on a GPU that reads the basis once per vector of the block.
// Here a 256-row tile of the kq basis columns AND the p block columns is resident in shared memory (same TMA
// ring as the single-vector engine, tsk.cuh), so the basis is read ONCE for all p vectors:
//
//   k_block_phase<PROJECT> : H = V' R          (kq + p) W bytes   (the reference loop: kq * p * 2W)
//   k_block_phase<UPDATE>  : R -= V H, and the Gram matrix G = R' R of the result for free
//                                               (kq + 2p) W bytes  (reference: kq * p * 3W)
//
// on top of which sit block_inner / the block residual update (exact same mathematics as the reference, one
// launch per 48 basis columns), a flagged block-classical-Gram-Schmidt-twice orthogonalisation against V, and a
// flagged CholeskyQR2 for block_qr! (Gram -> Cholesky on the host -> triangular basis transform, twice).
// Everything is deterministic: per-CTA partials summed in CTA order.
#include "tsk.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

using namespace tsk;

namespace {

constexpr int BK_QMAX = 48;    // basis columns per pass (6 per consumer warp)
constexpr int BK_PMAX = 8;     // block size
constexpr int BK_JW = BK_QMAX / 8;
constexpr int BK_OFF_H = OFF_WRING;                     // coefficients (UPDATE): kq x p doubles <= 3 KB
constexpr int BK_OFF_G = OFF_WRING + 4096;              // Gram reduction scratch: 8 warps x 36 doubles
constexpr int BK_PART = BK_QMAX * BK_PMAX;              // doubles per CTA partial row (384)
constexpr int BK_GRAM = BK_PMAX * BK_PMAX;              // 64

template <typename T>
struct BlockParams {
    const T* base;        // slab base of the space
    int64_t ld, n;
    int32_t kq, p;        // basis columns in this pass, block size; columns list = [kq basis | p block]
    const double* H;      // UPDATE: device coefficients, column-major kq x p with leading dimension ldh
    int32_t ldh;
    T alpha;              // UPDATE: R -= alpha-signed: r = fma(q, alpha * H[j][i], r)
    double* part;         // PROJECT: [grid][BK_PART] partials (index i * BK_QMAX + j)
    double* gpart;        // UPDATE: [grid][BK_GRAM] Gram partials (may be nullptr)
    int32_t store;        // UPDATE: write the block back (0 when only the Gram matrix is wanted)
};

// the panel part of producer_phase (no streamed vector): chunk g of every tile is issued by producer warp g % NPROD
template <typename T>
__device__ __forceinline__ void producer_cols(const T* base, int64_t ld, int64_t n, int k, const ColList& cl,
                                              const SmemView& sm) {
    using CF = Cfg<T>;
    constexpr int R = CF::R, C = CF::C;
    const int lane = threadIdx.x & 31;
    const uint32_t me = (threadIdx.x - NCONS) >> 5;
    const int nch = (k + C - 1) / C;
    const int64_t ntiles = (n + R - 1) / R;
    uint32_t s = 0, ph = 0, g = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((n - r0) < R ? (n - r0) : R);
        const uint32_t bytes = (uint32_t)((rt * sizeof(T) + 15) & ~(size_t)15);
        for (int c = 0; c < nch; ++c) {
            if ((g % NPROD) == me) {
                mbar_wait(sm.empty + 8 * s, ph ^ 1);
                const int ncol = (k - c * C) < C ? (k - c * C) : C;
                if (lane == 0) mbar_expect_tx(sm.full + 8 * s, bytes * (uint32_t)ncol);
                __syncwarp();
                if (lane < ncol)
                    bulk_g2s(sm.ring + s * SLOT_BYTES + lane * R * (int)sizeof(T),
                             base + (int64_t)cl.c[c * C + lane] * ld + r0, bytes, sm.full + 8 * s);
            }
            ++g;
            if (++s == NS) { s = 0; ph ^= 1; }
        }
    }
}

// column j of the resident tile that starts at ring slot s0
template <typename T>
__device__ __forceinline__ const T* tile_col(uint8_t* smem, uint32_t s0, int j) {
    constexpr int C = Cfg<T>::C, R = Cfg<T>::R;
    uint32_t s = s0 + (uint32_t)(j / C);
    if (s >= NS) s -= NS;
    return reinterpret_cast<const T*>(smem + OFF_RING + s * SLOT_BYTES) + (j % C) * R;
}

// PROJECT work on one resident tile: warp w owns basis columns j = w, w + 8, ...; lane <-> rows (128-bit LDS).
// One row chunk at a time: the p block columns are read once per chunk and feed every basis column of this warp
// (they were re-read per basis column before: 88 % LSU utilisation at k = 20, p = 4).  Rows >= rt of a ragged last
// tile hold stale but FINITE data: masking the block side is enough.
template <typename T, int PP>
__device__ __forceinline__ void block_project_tile(uint8_t* smem, uint32_t s0, int kq, int pb, int rt, int lane, int w,
                                                   T (&acc)[BK_JW][PP]) {
    using CF = Cfg<T>;
    using V16 = typename CF::V16;
    constexpr int R = CF::R, VEC = CF::VEC;
    constexpr int NLD = R / (32 * VEC);
    const T* qc[BK_JW];
    const T* rc[PP];
#pragma unroll
    for (int a = 0; a < BK_JW; ++a) qc[a] = tile_col<T>(smem, s0, (a * 8 + w < kq) ? a * 8 + w : 0);
#pragma unroll
    for (int i = 0; i < PP; ++i) rc[i] = tile_col<T>(smem, s0, kq + (i < pb ? i : 0));
#pragma unroll
    for (int u = 0; u < NLD; ++u) {
        V16 x[PP];
#pragma unroll
        for (int i = 0; i < PP; ++i) {
            if (i < pb) {
                x[i] = *reinterpret_cast<const V16*>(rc[i] + VEC * lane + 32 * VEC * u);
                T* xe = reinterpret_cast<T*>(&x[i]);
#pragma unroll
                for (int e = 0; e < VEC; ++e)
                    if (VEC * lane + 32 * VEC * u + e >= rt) xe[e] = (T)0;
            }
        }
#pragma unroll
        for (int a = 0; a < BK_JW; ++a) {
            if (a * 8 + w < kq) {
                const V16 q = *reinterpret_cast<const V16*>(qc[a] + VEC * lane + 32 * VEC * u);
#pragma unroll
                for (int i = 0; i < PP; ++i)
                    if (i < pb) VecOps<T>::fma_acc(acc[a][i], q, x[i]);
            }
        }
    }
}

// per-CTA partials of the projection: part[cta][i * BK_QMAX + j]
template <typename T, int PP>
__device__ __forceinline__ void block_project_partials(const T (&acc)[BK_JW][PP], double* part, int kq, int pb, int lane,
                                                       int w) {
#pragma unroll
    for (int a = 0; a < BK_JW; ++a) {
        const int j = a * 8 + w;
#pragma unroll
        for (int i = 0; i < PP; ++i) {
            const double v = warp_sum((double)acc[a][i]);
            if (j < kq && i < pb && lane == 0) part[(size_t)blockIdx.x * BK_PART + i * BK_QMAX + j] = v;
        }
    }
}

// MODE 0: PROJECT, 1: UPDATE (+ Gram matrix of the result), 2: UPDATE followed by the PROJECT of the updated block on
// the same resident tile (the middle sweep of BCGS2: three passes over V instead of four).
// PP = 4 or 8: register block of the block dimension (p <= PP); p <= 4 halves the broadcast loads of H and the
// accumulators
template <typename T, int MODE, int PP>
__global__ void __launch_bounds__(NTHREADS, 1)
k_block_phase(const __grid_constant__ BlockParams<T> p, const __grid_constant__ ColList cl) {
    using CF = Cfg<T>;
    constexpr int R = CF::R, C = CF::C;
    extern __shared__ __align__(128) uint8_t smem[];
    SmemView sm(smem);
    pipe_setup(sm, true);     // ragged tiles multiply stale rows by nothing here, but keep the ring finite
    const int kt = p.kq + p.p;
    const int nch = (kt + C - 1) / C;
    const int64_t ntiles = (p.n + R - 1) / R;
    if (threadIdx.x >= NCONS) {
        producer_cols<T>(p.base, p.ld, p.n, kt, cl, sm);
        return;
    }
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    uint32_t s = 0, ph = 0;
    if (MODE == 0) {
        T acc[BK_JW][PP];
#pragma unroll
        for (int a = 0; a < BK_JW; ++a)
#pragma unroll
            for (int i = 0; i < PP; ++i) acc[a][i] = (T)0;
        for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int64_t r0 = tile * R;
            const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
            const uint32_t s0 = s;
            for (int c = 0; c < nch; ++c) {
                mbar_wait(sm.full + 8 * s, ph);
                if (++s == NS) { s = 0; ph ^= 1; }
            }
            block_project_tile<T, PP>(smem, s0, p.kq, p.p, rt, lane, w, acc);
            // release the tile
            __syncwarp();
            uint32_t ss = s0;
            for (int c = 0; c < nch; ++c) {
                if (lane == 0) mbar_arrive(sm.empty + 8 * ss);
                if (++ss == NS) ss = 0;
            }
        }
        block_project_partials<T, PP>(acc, p.part, p.kq, p.p, lane, w);
        return;
    }
    // ---- UPDATE: thread <-> row; r_i -= sum_j q_j H[j][i] (sequential fma over j: the association of the
    // reference's chain of add!! calls), then the Gram matrix of the updated block (MODE 1) or its projection (MODE 2)
    T* Hs = reinterpret_cast<T*>(smem + BK_OFF_H);
    for (int idx = tid; idx < p.kq * PP; idx += NCONS) {
        const int j = idx / PP, i = idx - j * PP;
        Hs[idx] = (i < p.p) ? p.alpha * (T)p.H[(size_t)i * p.ldh + j] : (T)0;
    }
    named_bar_sync(1, NCONS);
    constexpr int NG = (MODE == 1) ? PP * (PP + 1) / 2 : 1;
    T g[NG];
#pragma unroll
    for (int t = 0; t < NG; ++t) g[t] = (T)0;
    constexpr int NA = (MODE == 2) ? BK_JW : 1;
    T acc[NA][PP];
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
        for (int i = 0; i < PP; ++i) acc[a][i] = (T)0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * R;
        const int rt = (int)((p.n - r0) < R ? (p.n - r0) : R);
        const uint32_t s0 = s;
        for (int c = 0; c < nch; ++c) {
            mbar_wait(sm.full + 8 * s, ph);
            if (++s == NS) { s = 0; ph ^= 1; }
        }
        T r[PP];
#pragma unroll
        for (int i = 0; i < PP; ++i) r[i] = (i < p.p && tid < rt) ? tile_col<T>(smem, s0, p.kq + i)[tid] : (T)0;
        for (int j = 0; j < p.kq; ++j) {
            const T q = (tid < rt) ? tile_col<T>(smem, s0, j)[tid] : (T)0;
            const T* h = Hs + j * PP;
#pragma unroll
            for (int i = 0; i < PP; ++i) r[i] = fma(q, h[i], r[i]);
        }
        if (p.store && tid < rt) {
#pragma unroll
            for (int i = 0; i < PP; ++i)
                if (i < p.p) const_cast<T*>(p.base)[(int64_t)cl.c[p.kq + i] * p.ld + r0 + tid] = r[i];
        }
        if (MODE == 1 && p.gpart) {
            int t = 0;
#pragma unroll
            for (int i1 = 0; i1 < PP; ++i1)
#pragma unroll
                for (int i2 = i1; i2 < PP; ++i2) { g[t] = fma(r[i1], r[i2], g[t]); ++t; }
        }
        if constexpr (MODE == 2) {
            // the updated block replaces the staged one in the resident tile, then every warp projects it
#pragma unroll
            for (int i = 0; i < PP; ++i)
                if (i < p.p) const_cast<T*>(tile_col<T>(smem, s0, p.kq + i))[tid] = r[i];
            named_bar_sync(1, NCONS);
            block_project_tile<T, PP>(smem, s0, p.kq, p.p, rt, lane, w, acc);
            fence_proxy_async();      // generic-proxy writes to the slots precede their reuse by the TMA unit
        }
        __syncwarp();
        uint32_t ss = s0;
        for (int c = 0; c < nch; ++c) {
            if (lane == 0) mbar_arrive(sm.empty + 8 * ss);
            if (++ss == NS) ss = 0;
        }
    }
    if constexpr (MODE == 2) block_project_partials<T, PP>(acc, p.part, p.kq, p.p, lane, w);
    if (MODE == 1 && p.gpart) {
        double* red = reinterpret_cast<double*>(smem + BK_OFF_G);      // [8 warps][36]
        constexpr int NT = PP * (PP + 1) / 2;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const double v = warp_sum((double)g[t]);
            if (lane == 0) red[w * NT + t] = v;
        }
        named_bar_sync(1, NCONS);
        if (tid < NT) {
            double a = 0.0;
            for (int ww = 0; ww < NCONS / 32; ++ww) a += red[ww * NT + tid];
            // unpack t -> (i1, i2)
            int i1 = 0, t = tid;
            while (t >= PP - i1) { t -= PP - i1; ++i1; }
            const int i2 = i1 + t;
            p.gpart[(size_t)blockIdx.x * BK_GRAM + i1 * BK_PMAX + i2] = a;
            p.gpart[(size_t)blockIdx.x * BK_GRAM + i2 * BK_PMAX + i1] = a;
        }
    }
}

// out[idx] (+)= sum over CTAs of part[g * stride + map(idx)], fixed order.  PROJECT layout: idx = i * ldo + j
// reads part[i * BK_QMAX + j]; Gram layout: idx = i1 * p + i2 reads part[i1 * BK_PMAX + i2].
__global__ void __launch_bounds__(256)
k_block_finalize(const double* __restrict__ part, int G, int stride, int rows, int cols, int src_ld, double* out,
                 int out_ld, int accumulate) {
    for (int idx = threadIdx.x; idx < rows * cols; idx += blockDim.x) {
        const int i = idx / rows, j = idx - i * rows;     // column i, row j of the (rows x cols) result
        double a = 0.0;
        const double* src = part + i * src_ld + j;
        int g = 0;
        for (; g + 8 <= G; g += 8) {           // eight independent loads in flight, added in CTA order
            double v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = src[(size_t)(g + u) * stride];
#pragma unroll
            for (int u = 0; u < 8; ++u) a += v[u];
        }
        for (; g < G; ++g) a += src[(size_t)g * stride];
        double* o = out + (size_t)i * out_ld + j;
        *o = accumulate ? (*o + a) : a;
    }
}

// X <- X U in place for a block of P <= 8 columns and an UPPER triangular U (the CholeskyQR step X L^-T):
// thread <-> row, out_j = sum_{i <= j} x_i U[i, j] by fma over i in increasing order (k_transform's order), plain
// 128-bit streaming accesses with all loads of a trip ahead of its stores; optionally the Gram matrix of the
// RESULT (per-CTA partials in the k_block_phase<UPDATE> layout), which is the second round's input — CholeskyQR2
// costs two passes over the block instead of three.
template <typename T> __device__ __forceinline__ void ld_vec(const T* p, T (&v)[16 / sizeof(T)]);
template <> __device__ __forceinline__ void ld_vec<double>(const double* p, double (&v)[2]) {
    const double2 t = *reinterpret_cast<const double2*>(p);
    v[0] = t.x; v[1] = t.y;
}
template <> __device__ __forceinline__ void ld_vec<float>(const float* p, float (&v)[4]) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <typename T> __device__ __forceinline__ void st_vec(T* p, const T (&v)[16 / sizeof(T)]);
template <> __device__ __forceinline__ void st_vec<double>(double* p, const double (&v)[2]) {
    *reinterpret_cast<double2*>(p) = make_double2(v[0], v[1]);
}
template <> __device__ __forceinline__ void st_vec<float>(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

struct RmulParams {
    void* base;
    int64_t ld, n;
    int32_t cols[BK_PMAX];
    double u[BK_PMAX * BK_PMAX];      // column-major P x P
    double* gpart;                    // [grid][BK_GRAM] or nullptr
};

template <typename T, int P>
__global__ void __launch_bounds__(256)
k_block_rmul(const __grid_constant__ RmulParams rp) {
    __shared__ double red[8][P * (P + 1) / 2];
    constexpr int NT = P * (P + 1) / 2;
    T* base = reinterpret_cast<T*>(rp.base);
    T* col[P];
#pragma unroll
    for (int i = 0; i < P; ++i) col[i] = base + (int64_t)rp.cols[i] * rp.ld;
    T g[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) g[t] = (T)0;
    // thread <-> VEC consecutive rows (one 128-bit access per column); the products are formed in place, last
    // output column first (out_j needs x_0..x_j only), to keep the kernel at 4 CTAs per SM
    constexpr int VEC = 16 / (int)sizeof(T);
    const int64_t nv = rp.n / VEC;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t v0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v0 < nv; v0 += stride) {
        T x[P][VEC];
#pragma unroll
        for (int i = 0; i < P; ++i) ld_vec<T>(col[i] + v0 * VEC, x[i]);
#pragma unroll
        for (int j = P - 1; j >= 0; --j) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                T a = (T)0;
#pragma unroll
                for (int i = 0; i <= j; ++i) a = fma(x[i][e], (T)rp.u[j * P + i], a);
                x[j][e] = a;
            }
        }
#pragma unroll
        for (int j = 0; j < P; ++j) st_vec<T>(col[j] + v0 * VEC, x[j]);
        if (rp.gpart) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                int t = 0;
#pragma unroll
                for (int a = 0; a < P; ++a)
#pragma unroll
                    for (int b = a; b < P; ++b) { g[t] = fma(x[a][e], x[b][e], g[t]); ++t; }
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < rp.n - nv * VEC) {      // tail rows
        const int64_t r = nv * VEC + threadIdx.x;
        T x[P], o[P];
#pragma unroll
        for (int i = 0; i < P; ++i) x[i] = col[i][r];
#pragma unroll
        for (int j = 0; j < P; ++j) {
            T a = (T)0;
#pragma unroll
            for (int i = 0; i <= j; ++i) a = fma(x[i], (T)rp.u[j * P + i], a);
            o[j] = a;
        }
#pragma unroll
        for (int j = 0; j < P; ++j) col[j][r] = o[j];
        if (rp.gpart) {
            int t = 0;
#pragma unroll
            for (int a = 0; a < P; ++a)
#pragma unroll
                for (int b = a; b < P; ++b) { g[t] = fma(o[a], o[b], g[t]); ++t; }
        }
    }
    if (!rp.gpart) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
        double v = (double)g[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) red[w][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < NT) {
        double a = 0.0;
        for (int ww = 0; ww < 8; ++ww) a += red[ww][threadIdx.x];
        int t = threadIdx.x, i1 = 0;
        while (t >= P - i1) { t -= P - i1; ++i1; }
        const int i2 = i1 + t;
        rp.gpart[(size_t)blockIdx.x * BK_GRAM + i1 * BK_PMAX + i2] = a;
        rp.gpart[(size_t)blockIdx.x * BK_GRAM + i2 * BK_PMAX + i1] = a;
    }
}

int grid_rows(const b2k_ctx* ctx, int64_t n) {
    int64_t ntiles = (n + 255) / 256;
    if (ntiles < 1) ntiles = 1;
    return (int)std::min<int64_t>(ntiles, ctx->num_sms);
}

struct BPanel {
    void* base = nullptr;
    int64_t ld = 0, n = 0;
    int32_t sharded = 1, space = -1;
    std::vector<int32_t> q, r;
};

int32_t make_bpanel(b2k_ctx* ctx, const b2k_vec* V, int32_t k, const b2k_vec* Rb, int32_t p, BPanel* bp) {
    int32_t sv = -1, sr = -1;
    B2K_TRY(b2k_resolve_cols(ctx, Rb, p, &sr, &bp->r));
    if (k > 0) {
        B2K_TRY(b2k_resolve_cols(ctx, V, k, &sv, &bp->q));
        if (sv != sr) return b2k_fail(ctx, B2K_EDIM, "block operation: basis and block live in different spaces");
    }
    const B2kSpace& s = ctx->spaces[sr];
    bp->base = s.base; bp->ld = s.ld; bp->n = s.n; bp->sharded = s.sharded; bp->space = sr;
    return B2K_OK;
}

// d_blk layout (doubles): [0, HCAP) H1, [HCAP, 2 HCAP) H2, then the Gram matrix
constexpr int HCAP = B2K_BLK_HCAP;
static_assert(BK_PART == B2K_BLK_PART, "partial row size");

template <typename T>
int32_t launch_project(b2k_ctx* ctx, const BPanel& bp, int q0, int kq, double* d_H, int ldh, bool accumulate) {
    const int p = (int)bp.r.size();
    ColList cl;
    for (int j = 0; j < kq; ++j) cl.c[j] = bp.q[q0 + j];
    for (int i = 0; i < p; ++i) cl.c[kq + i] = bp.r[i];
    BlockParams<T> bpar;
    memset(&bpar, 0, sizeof(bpar));
    bpar.base = (const T*)bp.base; bpar.ld = bp.ld; bpar.n = bp.n; bpar.kq = kq; bpar.p = p;
    bpar.part = ctx->d_blkpart;
    const int grid = grid_rows(ctx, bp.n);
    const int pr = b2k_prof_begin(ctx, 5, (double)(kq + p) * sizeof(T) * (double)bp.n);
    if (p <= 4) k_block_phase<T, 0, 4><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(bpar, cl);
    else k_block_phase<T, 0, 8><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(bpar, cl);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    k_block_finalize<<<1, 256, 0, ctx->stream>>>(ctx->d_blkpart, grid, BK_PART, kq, p, BK_QMAX, d_H + q0, ldh,
                                                accumulate ? 1 : 0);
    B2K_LAUNCH_CHECK(ctx);
    return B2K_OK;
}

template <typename T>
int32_t launch_update(b2k_ctx* ctx, const BPanel& bp, int q0, int kq, const double* d_H, int ldh, double alpha,
                      double* d_G, bool store) {
    const int p = (int)bp.r.size();
    ColList cl;
    for (int j = 0; j < kq; ++j) cl.c[j] = bp.q[q0 + j];
    for (int i = 0; i < p; ++i) cl.c[kq + i] = bp.r[i];
    BlockParams<T> bpar;
    memset(&bpar, 0, sizeof(bpar));
    bpar.base = (const T*)bp.base; bpar.ld = bp.ld; bpar.n = bp.n; bpar.kq = kq; bpar.p = p;
    bpar.H = d_H ? d_H + q0 : nullptr; bpar.ldh = ldh; bpar.alpha = (T)alpha;
    bpar.gpart = d_G ? ctx->d_blkpart : nullptr;
    bpar.store = store ? 1 : 0;
    const int grid = grid_rows(ctx, bp.n);
    const int pr = b2k_prof_begin(ctx, 6, (double)(kq + (store ? 2 : 1) * p) * sizeof(T) * (double)bp.n);
    if (p <= 4) k_block_phase<T, 1, 4><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(bpar, cl);
    else k_block_phase<T, 1, 8><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(bpar, cl);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    if (d_G) {
        k_block_finalize<<<1, 256, 0, ctx->stream>>>(ctx->d_blkpart, grid, BK_GRAM, p, p, BK_PMAX, d_G, p, 0);
        B2K_LAUNCH_CHECK(ctx);
    }
    return B2K_OK;
}

// R += alpha V H1 and H2 = V' R_new in ONE sweep (k <= BK_QMAX, p <= 4): the middle of BCGS2
template <typename T>
int32_t launch_update_project(b2k_ctx* ctx, const BPanel& bp, const double* d_H1, double alpha, double* d_H2) {
    const int k = (int)bp.q.size(), p = (int)bp.r.size();
    ColList cl;
    for (int j = 0; j < k; ++j) cl.c[j] = bp.q[j];
    for (int i = 0; i < p; ++i) cl.c[k + i] = bp.r[i];
    BlockParams<T> bpar;
    memset(&bpar, 0, sizeof(bpar));
    bpar.base = (const T*)bp.base; bpar.ld = bp.ld; bpar.n = bp.n; bpar.kq = k; bpar.p = p;
    bpar.H = d_H1; bpar.ldh = k; bpar.alpha = (T)alpha;
    bpar.part = ctx->d_blkpart;
    bpar.store = 1;
    const int grid = grid_rows(ctx, bp.n);
    const int pr = b2k_prof_begin(ctx, 6, (double)(k + 2 * p) * sizeof(T) * (double)bp.n);
    k_block_phase<T, 2, 4><<<grid, NTHREADS, SMEM_BYTES, ctx->stream>>>(bpar, cl);
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    k_block_finalize<<<1, 256, 0, ctx->stream>>>(ctx->d_blkpart, grid, BK_PART, k, p, BK_QMAX, d_H2, k, 0);
    B2K_LAUNCH_CHECK(ctx);
    return b2k_allreduce(ctx, d_H2, k * p, bp.sharded);
}

// H (k x p, ld = k) = V' R on the device, all passes; all-reduced when sharded
int32_t block_project_dev(b2k_ctx* ctx, const BPanel& bp, double* d_H, bool accumulate) {
    const int k = (int)bp.q.size(), p = (int)bp.r.size();
    for (int q0 = 0; q0 < k; q0 += BK_QMAX) {
        const int kq = std::min(BK_QMAX, k - q0);
        B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return launch_project<decltype(t)>(ctx, bp, q0, kq, d_H, k, accumulate); }));
    }
    if (!accumulate) B2K_TRY(b2k_allreduce(ctx, d_H, k * p, bp.sharded));
    return B2K_OK;
}

// R += alpha * V H; optionally the Gram matrix of the result (last pass)
int32_t block_update_dev(b2k_ctx* ctx, const BPanel& bp, const double* d_H, double alpha, double* d_G) {
    const int k = (int)bp.q.size(), p = (int)bp.r.size();
    for (int q0 = 0; q0 < k; q0 += BK_QMAX) {
        const int kq = std::min(BK_QMAX, k - q0);
        const bool lastp = q0 + kq >= k;
        B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return launch_update<decltype(t)>(ctx, bp, q0, kq, d_H, k, alpha, lastp ? d_G : nullptr, true); }));
    }
    if (d_G) B2K_TRY(b2k_allreduce(ctx, d_G, p * p, bp.sharded));
    return B2K_OK;
}

// X <- X U (U upper triangular, column-major p x p on the host); d_G != nullptr: Gram matrix of the result
int32_t block_rmul_upper(b2k_ctx* ctx, const BPanel& bp, const double* U, double* d_G) {
    const int p = (int)bp.r.size();
    RmulParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.base = bp.base; rp.ld = bp.ld; rp.n = bp.n;
    for (int i = 0; i < p; ++i) rp.cols[i] = bp.r[i];
    memcpy(rp.u, U, sizeof(double) * p * p);
    rp.gpart = d_G ? ctx->d_blkpart : nullptr;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((bp.n + 511) / 512, 4 * (int64_t)ctx->num_sms));
    const int pr = b2k_prof_begin(ctx, 6, 2.0 * p * ctx->esize * (double)bp.n);
    b2k_dispatch(ctx, [&](auto t) {
        using T = decltype(t);
#define RMUL(P) k_block_rmul<T, P><<<grid, 256, 0, ctx->stream>>>(rp)
        switch (p) {
            case 1: RMUL(1); break; case 2: RMUL(2); break; case 3: RMUL(3); break;
            case 4: RMUL(4); break; case 5: RMUL(5); break; case 6: RMUL(6); break;
            case 7: RMUL(7); break; default: RMUL(8); break;
        }
#undef RMUL
    });
    b2k_prof_end(ctx, pr);
    B2K_LAUNCH_CHECK(ctx);
    if (d_G) {
        k_block_finalize<<<1, 256, 0, ctx->stream>>>(ctx->d_blkpart, grid, BK_GRAM, p, p, BK_PMAX, d_G, p, 0);
        B2K_LAUNCH_CHECK(ctx);
        B2K_TRY(b2k_allreduce(ctx, d_G, p * p, bp.sharded));
    }
    return B2K_OK;
}

int32_t block_gram_dev(b2k_ctx* ctx, const BPanel& bp, double* d_G) {
    const int p = (int)bp.r.size();
    B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return launch_update<decltype(t)>(ctx, bp, 0, 0, nullptr, 1, 0.0, d_G, false); }));
    return b2k_allreduce(ctx, d_G, p * p, bp.sharded);
}

int32_t fetch(b2k_ctx* ctx, const double* d, double* h, int count) {
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, d, sizeof(double) * count, cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    memcpy(h, ctx->h_res, sizeof(double) * count);
    return B2K_OK;
}

}  // namespace

// B2K_BLOCK_KERNELS=0 routes block_inner / block_axpy / apply_block through loops of the single-vector entry points
// (the round-1 behaviour) — an escape hatch and the A/B baseline for the multi-right-hand-side kernels.
static bool g_block_kernels = true;
static bool g_block_fuse = true;      // B2K_BLOCK_FUSE=0: BCGS2 as four separate sweeps (A/B switch)
bool b2k_block_kernels_enabled() { return g_block_kernels; }

int32_t b2k_block_init(b2k_ctx* ctx) {
    if (const char* e = getenv("B2K_BLOCK_KERNELS")) g_block_kernels = e[0] != '0';
    if (const char* e = getenv("B2K_BLOCK_FUSE")) g_block_fuse = e[0] != '0';
#define BK_ATTR(T, U, PP) \
    B2K_CUDA(ctx, cudaFuncSetAttribute((k_block_phase<T, U, PP>), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES))
    BK_ATTR(double, 0, 4); BK_ATTR(double, 0, 8); BK_ATTR(double, 1, 4); BK_ATTR(double, 1, 8); BK_ATTR(double, 2, 4);
    BK_ATTR(float, 0, 4); BK_ATTR(float, 0, 8); BK_ATTR(float, 1, 4); BK_ATTR(float, 1, 8); BK_ATTR(float, 2, 4);
#undef BK_ATTR
    return B2K_OK;
}

// ------------------------------------------------------------------ C ABI ----

// block_inner(X, Y): M[i, j] = <X[i], Y[j]> — blocklanczos.jl:43-52 — one launch per 48 vectors of X
extern "C" int32_t b2k_block_inner(b2k_ctx* ctx, const b2k_vec* X, int32_t p, const b2k_vec* Y,
                                   int32_t q, double* M_host) {
    if (!ctx || !X || !Y || !M_host || p < 1 || q < 1) return B2K_EINVAL;
    if (!g_block_kernels) {
        for (int j = 0; j < q; ++j) B2K_TRY(b2k_basis_project(ctx, X, p, Y[j], 1.0, 0.0, M_host + (size_t)j * p));
        return B2K_OK;
    }
    if (p * BK_PMAX > HCAP || (int64_t)p * q > B2K_RES_DOUBLES) return b2k_fail(ctx, B2K_ENOTSUP, "block_inner: p*q too large");
    for (int j0 = 0; j0 < q; j0 += BK_PMAX) {           // blocks of up to 8 right-hand sides
        const int qq = std::min(BK_PMAX, q - j0);
        BPanel bp;
        B2K_TRY(make_bpanel(ctx, X, p, Y + j0, qq, &bp));
        B2K_TRY(block_project_dev(ctx, bp, ctx->d_blk, false));
        B2K_TRY(fetch(ctx, ctx->d_blk, M_host + (size_t)j0 * p, p * qq));
    }
    return B2K_OK;
}

// Y[j] -= sum_i X[i] M[i, j] — the double loops of blocklanczos.jl:177-181, 245-252 — one launch per 48 vectors of X
extern "C" int32_t b2k_block_axpy(b2k_ctx* ctx, const b2k_vec* Y, int32_t q, const b2k_vec* X,
                                  int32_t p, const double* M_host, int32_t ldm) {
    if (!ctx || !X || !Y || !M_host || p < 1 || q < 1 || ldm < p) return B2K_EINVAL;
    if (!g_block_kernels) {
        for (int j = 0; j < q; ++j)
            B2K_TRY(b2k_basis_unproject(ctx, Y[j], X, p, M_host + (size_t)j * ldm, -1.0, 1.0));
        return B2K_OK;
    }
    if (p * BK_PMAX > HCAP) return b2k_fail(ctx, B2K_ENOTSUP, "block_axpy: p too large");
    for (int i = 0; i < p; ++i)
        for (int j = 0; j < q; ++j)
            if (X[i] == Y[j]) return b2k_fail(ctx, B2K_EINVAL, "block_axpy: Y[%d] aliases X[%d]", j, i);
    for (int j0 = 0; j0 < q; j0 += BK_PMAX) {
        const int qq = std::min(BK_PMAX, q - j0);
        BPanel bp;
        B2K_TRY(make_bpanel(ctx, X, p, Y + j0, qq, &bp));
        std::vector<double> Hc((size_t)p * qq);
        for (int j = 0; j < qq; ++j)
            for (int i = 0; i < p; ++i) Hc[(size_t)j * p + i] = M_host[(size_t)(j0 + j) * ldm + i];
        if (p * qq > B2K_COEF_DOUBLES) return b2k_fail(ctx, B2K_ENOTSUP, "block_axpy: coefficient block too large");
        B2K_TRY(b2k_put_coef(ctx, Hc.data(), p * qq, 0));
        B2K_TRY(block_update_dev(ctx, bp, ctx->d_coef, -1.0, nullptr));
    }
    return B2K_OK;
}

// Flagged replacement of block_reorthogonalize! (blocklanczos.jl:277-284, one MGS sweep per vector):
// block classical Gram-Schmidt against V, `passes` times (2 = BCGS2), the basis read once per pass for the whole
// block.  H_host (k x p, column-major, may be NULL) receives the summed coefficients, G_host (p x p, may be NULL)
// the Gram matrix R' R of the orthogonalised block (what CholeskyQR needs next).  One host synchronisation.
extern "C" int32_t b2k_block_orthogonalize(b2k_ctx* ctx, const b2k_vec* Rb, int32_t p, const b2k_vec* V, int32_t k,
                                           int32_t passes, double* H_host, double* G_host) {
    if (!ctx || !Rb || p < 1 || p > BK_PMAX || k < 0 || (k > 0 && !V) || passes < 1 || passes > 2) return B2K_EINVAL;
    if (k * p > HCAP) return b2k_fail(ctx, B2K_ENOTSUP, "block_orthogonalize: k * p > %d", HCAP);
    BPanel bp;
    B2K_TRY(make_bpanel(ctx, V, k, Rb, p, &bp));
    for (int i = 0; i < p; ++i)
        for (int j = 0; j < k; ++j)
            if (Rb[i] == V[j]) return b2k_fail(ctx, B2K_EINVAL, "block_orthogonalize: R[%d] aliases V[%d]", i, j);
    double* d_H1 = ctx->d_blk;
    double* d_H2 = ctx->d_blk + HCAP;
    double* d_G = ctx->d_blk + 2 * HCAP;
    if (k == 0) {
        if (G_host) {
            B2K_TRY(block_gram_dev(ctx, bp, d_G));
            B2K_TRY(fetch(ctx, d_G, G_host, p * p));
        }
        return B2K_OK;
    }
    B2K_TRY(block_project_dev(ctx, bp, d_H1, false));
    if (passes == 2 && p <= 4 && k <= BK_QMAX && g_block_fuse) {
        // three sweeps over V: project | update + project of the updated block on the resident tile | update (+ Gram)
        B2K_TRY(b2k_dispatch(ctx, [&](auto t) { return launch_update_project<decltype(t)>(ctx, bp, d_H1, -1.0, d_H2); }));
        B2K_TRY(block_update_dev(ctx, bp, d_H2, -1.0, G_host ? d_G : nullptr));
    } else {
        B2K_TRY(block_update_dev(ctx, bp, d_H1, -1.0, (passes == 1 && G_host) ? d_G : nullptr));
        if (passes == 2) {
            B2K_TRY(block_project_dev(ctx, bp, d_H2, false));
            B2K_TRY(block_update_dev(ctx, bp, d_H2, -1.0, G_host ? d_G : nullptr));
        }
    }
    static_assert(2 * HCAP + BK_GRAM <= B2K_RES_DOUBLES, "block results must fit the pinned result buffer");
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, ctx->d_blk, sizeof(double) * (2 * HCAP + BK_GRAM), cudaMemcpyDeviceToHost,
                                  ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    if (H_host)
        for (int t = 0; t < k * p; ++t) H_host[t] = ctx->h_res[t] + (passes == 2 ? ctx->h_res[HCAP + t] : 0.0);
    if (G_host) memcpy(G_host, ctx->h_res + 2 * HCAP, sizeof(double) * p * p);
    return B2K_OK;
}

// Flagged block_qr! (blocklanczos.jl:312-353): CholeskyQR2.  G = X' X (one pass), G = L L' on the host,
// X <- X L^-T (triangular basis transform, in place), twice; R = L2' L1' is upper triangular with a positive
// diagonal, i.e. the SAME factor modified Gram-Schmidt produces (the QR factorization with positive diagonal is
// unique), to rounding.  *ok = 0 when a Cholesky pivot falls below (100 tol)^2 or 9e4 u times its column's norm^2
// (numerically rank-deficient block: the caller falls back to the reference's MGS b2k_block_qr, which knows how
// to drop vectors); X is then unchanged.
extern "C" int32_t b2k_block_cholqr(b2k_ctx* ctx, const b2k_vec* X, int32_t p, double tol, const double* G0_host,
                                    double* R_host, int32_t* ok) {
    if (!ctx || !X || !R_host || !ok || p < 1 || p > BK_PMAX) return B2K_EINVAL;
    *ok = 0;
    BPanel bp;
    B2K_TRY(make_bpanel(ctx, nullptr, 0, X, p, &bp));
    double* d_G = ctx->d_blk + 2 * HCAP;
    std::vector<double> G(p * p), L(p * p), Rtot(p * p, 0.0), Linv(p * p);
    for (int i = 0; i < p; ++i) Rtot[i * p + i] = 1.0;
    // A Cholesky pivot is ||x_j - proj||^2 formed by SUBTRACTION: it carries an absolute error of ~u ||x_j||^2, with
    // u the unit roundoff of the vector type (the Gram matrix is accumulated from products rounded in T), so
    // CholeskyQR can neither resolve a residual below sqrt(u) ||x_j|| nor orthogonalise a block with condition number
    // above ~u^-1/2.  Accept only pivots well above that noise: relative 9e4 u, i.e. 1e-11 in Float64 (kappa < 3e5 —
    // the second round then restores orthogonality to eps) and 5.4e-3 in Float32 (kappa < 14; a Float32 pivot of
    // relative 1e-11 is noise, and the second Cholesky of such a block can fail) — AND above block_qr!'s own absolute
    // scale (100 tol)^2; everything else goes to the reference MGS path.
    const double rel_pivot = 1e-11 * (ctx->dtype == B2K_F64 ? 1.0 : 0x1p-24 / 0x1p-53);
    for (int round = 0; round < 2; ++round) {
        if (round == 0 && G0_host) {
            memcpy(G.data(), G0_host, sizeof(double) * p * p);
        } else {
            if (round == 0) B2K_TRY(block_gram_dev(ctx, bp, d_G));      // round 1: left by the first X <- X U pass
            B2K_TRY(fetch(ctx, d_G, G.data(), p * p));
        }
        // Cholesky G = L L' (column-major, lower)
        std::fill(L.begin(), L.end(), 0.0);
        for (int j = 0; j < p; ++j) {
            double d = G[j * p + j];
            for (int t = 0; t < j; ++t) d -= L[t * p + j] * L[t * p + j];
            const double thr = (round == 0) ? std::max((100.0 * tol) * (100.0 * tol), rel_pivot * G[j * p + j]) : 0.0;
            if (!(d > thr) || !(d > 1e-28 * G[j * p + j])) {
                if (round == 0) return B2K_OK;             // *ok = 0, X untouched
                return b2k_fail(ctx, B2K_ECUDA, "block_cholqr: second Cholesky lost positivity");
            }
            L[j * p + j] = sqrt(d);
            for (int i = j + 1; i < p; ++i) {
                double s = G[j * p + i];
                for (int t = 0; t < j; ++t) s -= L[t * p + i] * L[t * p + j];
                L[j * p + i] = s / L[j * p + j];
            }
        }
        // U = L^-T (upper triangular): X <- X U
        std::fill(Linv.begin(), Linv.end(), 0.0);       // Linv = L^-1 (lower), column-major
        for (int j = 0; j < p; ++j) {
            Linv[j * p + j] = 1.0 / L[j * p + j];
            for (int i = j + 1; i < p; ++i) {
                double s = 0.0;
                for (int t = j; t < i; ++t) s += L[t * p + i] * Linv[j * p + t];
                Linv[j * p + i] = -s / L[i * p + i];
            }
        }
        std::vector<double> U(p * p, 0.0);               // U[i, j] = Linv[j, i]
        for (int j = 0; j < p; ++j)
            for (int i = 0; i <= j; ++i) U[j * p + i] = Linv[i * p + j];
        B2K_TRY(block_rmul_upper(ctx, bp, U.data(), round == 0 ? d_G : nullptr));
        // R_total <- L' * R_total
        std::vector<double> Rn(p * p, 0.0);
        for (int j = 0; j < p; ++j)
            for (int i = 0; i < p; ++i) {
                double s = 0.0;
                for (int t = i; t < p; ++t) s += L[i * p + t] * Rtot[j * p + t];    // L'[i, t] = L[t, i]
                Rn[j * p + i] = s;
            }
        Rtot = Rn;
    }
    memcpy(R_host, Rtot.data(), sizeof(double) * p * p);
    *ok = 1;
    return B2K_OK;
}
