// common.cuh — context, error handling and PTX helpers shared by all translation units
// of libb200krylov.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/b200krylov.h"

// ----------------------------------------------------------------------------------
// limits
// ----------------------------------------------------------------------------------
constexpr int B2K_MAX_SPACES   = 8;
constexpr int B2K_RES_DOUBLES  = 8192;     // device/host scalar result buffer
constexpr int B2K_COEF_DOUBLES = 65536;    // host->device coefficient staging (512 KB)
constexpr int B2K_MAX_GRID     = 1024;     // upper bound on partial-producing CTAs (basis kernels)
constexpr int B2K_KSTRIDE      = 256;      // stride (doubles) between per-CTA partial rows
constexpr int B2K_MAX_CHAIN    = 512;      // Lanczos steps enqueued back to back without a host round trip
constexpr int B2K_REC          = 8;        // doubles per step record (tsk.cuh FinalizeParams)
// d_sync slots: [0] ticket of the BLAS-1 / SpMV reductions, [1] grid-barrier counter, [2] ticket of the
// in-kernel Gram-Schmidt finalisation, [4] breakdown flag of a chained Lanczos batch
constexpr int B2K_SYNC_GSFIN   = 2;
constexpr int B2K_SYNC_STOP    = 4;
constexpr int B2K_SYNC_HALO    = 5;        // ticket of k_halo_push

struct B2kSpace {
    void*   base   = nullptr;   // device pointer, column-major n x ncols, leading dim ld
    int64_t n      = 0;         // local rows
    int64_t ld     = 0;         // elements; multiple of 32 (256 B for f64, 128 B for f32)
    int32_t ncols  = 0;
    int32_t sharded = 1;        // reductions over this space are summed across ranks
    std::vector<uint8_t> used;
};

struct B2kNccl;   // dist.cu

// optional per-kernel-class timing (CUDA events on the context stream), used by bench.py
// for the roofline figure: class 0 = CSR SpMV, 1 = fused Gram-Schmidt, 2 = basis transform,
// 3 = project, 4 = unproject, ..., 9 = cross Gram sweep (b2k_basis_cross_inner)
constexpr int B2K_PROF_CLASSES = 10;
struct B2kProfRec { int cls; double bytes; cudaEvent_t e0, e1; };
struct B2kProf {
    bool on = false;
    std::vector<cudaEvent_t> pool;
    size_t next = 0;
    std::vector<B2kProfRec> recs;
};

struct b2k_ctx {
    int32_t device = 0;
    int32_t dtype  = B2K_F64;
    int32_t esize  = 8;
    int32_t num_sms = 0;
    size_t  l2_persist_bytes = 0;   // persisting-L2 carve-out (0 = unavailable)
    int     dot_hints = 0;          // set by the MGS sweep: its k_dot launches carry L2 eviction-priority hints
    unsigned long long* d_trace = nullptr;   // b2k_debug_trace: [0] event count, then (globaltimer ns, code) pairs
    size_t  l2_window_max = 0;      // max access-policy window
    cudaStream_t stream = nullptr;
    std::vector<B2kSpace> spaces;
    std::vector<b2k_op*> ops;   // operators created on this context (destroyed with it)

    // scratch
    double*   d_part   = nullptr;   // partial sums: 4 sets x B2K_MAX_GRID x B2K_KSTRIDE doubles
    double*   d_part_s = nullptr;   // scalar partial sums for BLAS-1 / SpMV dots (1<<20 doubles)
    double*   d_res    = nullptr;   // reduced results on device
    double*   h_res    = nullptr;   // pinned
    double*   d_coef   = nullptr;   // coefficients uploaded from host
    double*   h_coef   = nullptr;   // pinned staging
    unsigned* d_sync   = nullptr;   // [0] ticket, [1] grid barrier counter, ... (B2K_SYNC_*)
    double*   d_steps  = nullptr;   // (B2K_MAX_CHAIN + 1) step records of B2K_REC doubles
    double*   d_blk    = nullptr;   // block path (block.cu): coefficient blocks H1 | H2 | Gram
    double*   d_blkpart = nullptr;  // block path: per-CTA partials
    cudaEvent_t ev_coef = nullptr;  // guards reuse of the pinned staging buffers
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;   // b2k_timer_start/stop
    bool      coef_busy = false;

    // dist
    int32_t rank = 0, nranks = 1;
    int64_t n_global = 0, row_offset = 0;
    B2kNccl* nccl = nullptr;

    B2kProf prof;
    unsigned barrier_base = 0;      // value of d_sync[1] before the next cooperative launch
    int64_t launches = 0;
    std::string err;
};

extern std::string g_b2k_create_error;

// ----------------------------------------------------------------------------------
// error handling
// ----------------------------------------------------------------------------------
int32_t b2k_fail(b2k_ctx* ctx, int32_t code, const char* fmt, ...);

#define B2K_CUDA(ctx, call)                                                              \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess)                                                          \
            return b2k_fail((ctx), B2K_ECUDA, "%s:%d: %s -> %s", __FILE__, __LINE__,     \
                            #call, cudaGetErrorString(e__));                             \
    } while (0)

#define B2K_TRY(call)                                                                    \
    do {                                                                                 \
        int32_t s__ = (call);                                                            \
        if (s__ != B2K_OK) return s__;                                                   \
    } while (0)

#define B2K_LAUNCH_CHECK(ctx)                                                            \
    do {                                                                                 \
        (ctx)->launches++;                                                               \
        cudaError_t e__ = cudaGetLastError();                                            \
        if (e__ != cudaSuccess)                                                          \
            return b2k_fail((ctx), B2K_ECUDA, "%s:%d: kernel launch -> %s", __FILE__,    \
                            __LINE__, cudaGetErrorString(e__));                          \
    } while (0)

// ----------------------------------------------------------------------------------
// handle decoding
// ----------------------------------------------------------------------------------
struct VecRef {
    void*   ptr;
    int64_t n;
    int64_t ld;
    int32_t space;
    int32_t col;
    int32_t sharded;
};

int32_t b2k_resolve(b2k_ctx* ctx, b2k_vec v, VecRef* out);
// all handles must share one space; fills col indices; returns space id in *space
int32_t b2k_resolve_cols(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, int32_t* space,
                         std::vector<int32_t>* idx);

// scalar plumbing (ctx.cu)
// reduce-across-ranks (if sharded & dist) the first `count` doubles of d_res, copy to h_res, sync.
int32_t b2k_fetch_results(b2k_ctx* ctx, int32_t count, int32_t sharded);
// allreduce `count` doubles in place on device (no-op on single GPU / non-sharded)
int32_t b2k_allreduce(b2k_ctx* ctx, double* dptr, int32_t count, int32_t sharded);
// upload `count` doubles of host coefficients into d_coef + offset (async, pinned staging)
int32_t b2k_put_coef(b2k_ctx* ctx, const double* host, int32_t count, int32_t offset);

// Device memory comes from the CUDA stream-ordered pool with an unbounded release
// threshold: a cudaMalloc/cudaFree of a multi-GB slab per solve would dominate the
// host-buffer path (tools/e2e_breakdown.py times it); the pool makes context/operator
// creation and destruction O(microseconds) after the first use.
cudaError_t b2k_dmalloc(void** p, size_t bytes, cudaStream_t stream);
cudaError_t b2k_dfree(void* p, cudaStream_t stream);
#define B2K_DMALLOC(p, bytes) b2k_dmalloc((void**)(p), (bytes), ctx->stream)
#define B2K_DFREE(p) b2k_dfree((p), ctx->stream)
// small cache of page-locked host scratch buffers (cudaHostAlloc is slow per call)
cudaError_t b2k_hmalloc(void** p, size_t bytes);
void b2k_hfree(void* p, size_t bytes);

// profiling (ctx.cu): returns a record index (or -1 when profiling is off)
int  b2k_prof_begin(b2k_ctx* ctx, int cls, double bytes);
void b2k_prof_end(b2k_ctx* ctx, int idx);

// partial buffers
static inline double* b2k_part_set(b2k_ctx* ctx, int set) {
    return ctx->d_part + (size_t)set * B2K_MAX_GRID * B2K_KSTRIDE;
}

// spmv.cu: free the device arrays of an operator (called by b2k_op_destroy / b2k_ctx_destroy)
void b2k_op_release(b2k_ctx* ctx, b2k_op* op);

// Lightweight in-kernel event trace (b2k_debug_trace): thread 0 of CTA 0 (and the "last CTA" paths) append
// (globaltimer, code) pairs; tools/trace_step.py turns them into the timeline of a chained Lanczos step.
constexpr unsigned long long B2K_TRACE_CAP = 1ull << 16;
#ifdef __CUDACC__
__device__ __forceinline__ void b2k_trace(unsigned long long* tr, unsigned code) {
    if (!tr) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(tr, 1ull);
    if (i < B2K_TRACE_CAP) { tr[2 + 2 * i] = t; tr[3 + 2 * i] = code; }
}
#endif

// Optional fusions of the Lanczos step into the SpMV (basis.cu, b2k_lanczos_expand_many):
//   xscale   : device scalar; the operand is x*(*xscale) — the normalisation v = r/β of lanczos.jl:257 applied
//              while gathering (each gathered entry is rounded exactly like the separate scale!! pass);
//   vout     : the normalised operand is also written out (row r writes x[r]*(*xscale)): it becomes the new
//              basis vector, in a column of its own because other CTAs still gather the unscaled x;
//   dot_self : the fused dot product is <x*(*xscale), y> (no separate read of the normalised vector);
//   stop     : device flag; when set the launch does nothing (a breakdown was detected by an earlier step of
//              a batch that was enqueued without waiting for the host).
struct SpmvFuse {
    const double* xscale;
    void* vout;
    const int* stop;
    int dot_self;
    int l2_hints;          // matrix stream evict_first, y = A x evict_last (it is the next kernel's operand)
    // the fused dot product is taken with y - (*dot_sub_scale) * dot_sub_vec instead of y (y itself is stored
    // unchanged): alpha = <v, A v - beta v_prev>, the ModifiedGramSchmidt order of lanczos.jl:304-306, 326-328
    const void* dot_sub_vec;
    const double* dot_sub_scale;
    // row-sharded contexts with the peer window: sequence number under which <x, y> is published to all ranks
    // (0: not published), and the halo sequence number a previous kernel has already pushed this operand's
    // boundary rows under (0: the apply pushes them itself)
    unsigned long long seq_alpha, seq_halo;
    unsigned long long* trace;     // optional event trace (b2k_debug_trace)
};

int32_t b2k_enqueue_apply(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y,
                          double a0, double a1, bool shifted, const VecRef* dotv, int dot_slot);
int32_t b2k_enqueue_apply_fused(b2k_ctx* ctx, const b2k_op* op, const VecRef& x, const VecRef& y,
                                double a0, double a1, bool shifted, const VecRef* dotv, double* dot_out,
                                const SpmvFuse* fz);

// basis.cu / spmv.cu
int32_t b2k_basis_init(b2k_ctx* ctx);
int32_t b2k_spmv_init(b2k_ctx* ctx);
int32_t b2k_block_init(b2k_ctx* ctx);
bool    b2k_block_kernels_enabled();
constexpr int B2K_BLK_HCAP = 3968;        // doubles per coefficient block (k * p <= HCAP)
constexpr int B2K_BLK_PART = 384;         // doubles per CTA partial row

// ----------------------------------------------------------------------------------
// NVLink peer window (dist.cu).  Every rank owns one cudaMalloc'ed window that all other ranks of the node
// map through CUDA IPC.  It carries the latency-bound exchanges of the Krylov step without NCCL and without
// extra launches: a rank WRITES its contribution into every peer's window (one-way stores over NVLink, then a
// release flag), and READS only its own window (local polling), so a reduction costs one NVLink write latency.
//   channel 0: <v, A v> partial of the SpMV          channel 1: projection coefficients of a Gram-Schmidt sweep
//   channel 2: ||w||^2 partial                        channel 3: generic small-vector all-reduce
// Slots and flags are double-buffered by the parity of the operation's sequence number (a rank can be at most
// one operation ahead of a peer on a channel, because the next operation needs that peer's contribution).
// The rest of the window is a heap for the receive side of halo exchanges (operators allocate from it).
// ----------------------------------------------------------------------------------
constexpr int    PEER_MAXR  = 16;
constexpr int    PEER_SLOT  = 1024;                      // doubles per (channel, parity, source rank)
constexpr int    PEER_NCH   = 4;
constexpr int    PEER_CH_ALPHA = 0, PEER_CH_COEF = 1, PEER_CH_NORM = 2, PEER_CH_GEN = 3;
constexpr size_t PEER_OFF_FLAGS  = 0;                    // u64 [NCH][2][MAXR], then halo flags u64 [2][2]
constexpr size_t PEER_OFF_HFLAGS = 8 * (size_t)(PEER_NCH * 2 * PEER_MAXR);
constexpr size_t PEER_OFF_SLOTS  = 4096;
constexpr size_t PEER_OFF_HEAP   = PEER_OFF_SLOTS + 8 * (size_t)(PEER_NCH * 2 * PEER_MAXR) * PEER_SLOT;

struct PeerDev {
    char* win[PEER_MAXR];      // win[p] = rank p's window as mapped in THIS process (win[rank] = own)
    int rank, nranks;
    // Watchdog of the in-kernel waits (peer_spin): a flag that has not arrived after timeout_ns (0: wait for
    // ever) latches *err — one int in mapped pinned host memory — and the wait gives up, as does every later
    // wait as soon as it sees the latch.  The host looks at the latch after each stream synchronisation
    // (b2k_stream_sync) and fails the call with B2K_ENCCL: a rank of the job died or left the SPMD call order,
    // and the survivors return an error instead of spinning on the GPU until somebody kills them.
    int* err;
    unsigned long long timeout_ns;
};
// what one kernel launch needs to know about the exchanges it takes part in (all seq == 0: single GPU)
struct PeerStep {
    PeerDev pd;
    unsigned long long seq_alpha;   // GS kernel: wait for / SpMV: publish <v, A v>
    unsigned long long seq_coef[2]; // GS kernel: phase boundaries
    unsigned long long seq_norm;    // GS kernel: finaliser
    unsigned long long seq_halo;    // GS kernel: halo rows pushed by the update phase / SpMV: wait before gathering
    // halo push (update phase of the GS kernel, or k_halo_push): my first send_lo rows go to rank-1's window at
    // dn_off, my last send_hi rows to rank+1's window at up_off (byte offsets from the window base)
    long long send_lo, send_hi;
    size_t dn_off, up_off;
    int wait_lo, wait_hi;           // SpMV: my lo / hi halo is filled by rank-1 / rank+1
    int on;
};

int32_t b2k_op_peer_halo(const b2k_ctx* ctx, const b2k_op* op, unsigned long long seq, PeerStep* ps);
bool    b2k_op_has_peer_halo(const b2k_op* op);

int32_t b2k_nccl_init(b2k_ctx* ctx, const void* uid);
void    b2k_nccl_destroy(b2k_ctx* ctx);
int32_t b2k_nccl_allreduce_f64(b2k_ctx* ctx, double* dptr, int32_t count);
// NVLink peer-memory all-reduce of a small vector (dist.cu); b2k_peer_ok says whether it is usable
bool    b2k_peer_ok(const b2k_ctx* ctx);
// cudaStreamSynchronize(ctx->stream) + the peer-window watchdog latch (see PeerDev): B2K_ENCCL if an in-kernel
// wait for another rank timed out in the work just completed.  Every synchronising entry point goes through it.
int32_t b2k_stream_sync(b2k_ctx* ctx);
bool    b2k_has_nccl(const b2k_ctx* ctx);
int32_t b2k_peer_allreduce(b2k_ctx* ctx, double* dptr, int32_t count);
// device view of the windows + host-side sequence counters (identical on every rank: SPMD call order)
const PeerDev* b2k_peer_dev(const b2k_ctx* ctx);
unsigned long long b2k_peer_next_seq(b2k_ctx* ctx, int channel);      // channel 4 = halo
// symmetric allocation from the window heap (same offset on every rank); returns SIZE_MAX if it does not fit
size_t  b2k_peer_heap_alloc(b2k_ctx* ctx, size_t bytes);
char*   b2k_peer_local(const b2k_ctx* ctx);
// host-side all-gather of small blobs over the node-local rendezvous (no NCCL needed)
int32_t b2k_host_allgather(b2k_ctx* ctx, const void* mine, size_t bytes, void* all);
// grouped neighbour exchange; up/dn = peer ranks or -1
int32_t b2k_nccl_halo_exchange(b2k_ctx* ctx, int up, int dn, const void* send_up, size_t send_up_bytes,
                               void* recv_dn, size_t recv_dn_bytes, const void* send_dn,
                               size_t send_dn_bytes, void* recv_up, size_t recv_up_bytes);
int32_t b2k_nccl_allgather(b2k_ctx* ctx, const void* sendbuf, void* recvbuf, size_t bytes);

// ----------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Flag store AFTER an explicit __threadfence_system(): fence + relaxed store is a release pattern too, and unlike a
// sequence of st.release.sys to several peers it does not wait for the previous flag's NVLink round trip before the
// next one is issued (a chain of release stores to 8 ranks serialises 8 round trips).
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ double ld_volatile_f64(const double* p) {
    double v;
    asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double* peer_slot(const PeerDev& pd, int dst, int ch, unsigned long long seq, int src) {
    return reinterpret_cast<double*>(pd.win[dst] + PEER_OFF_SLOTS) +
           (size_t)((ch * 2 + (int)(seq & 1ull)) * PEER_MAXR + src) * PEER_SLOT;
}
__device__ __forceinline__ unsigned long long* peer_flag(const PeerDev& pd, int dst, int ch, unsigned long long seq,
                                                         int src) {
    return reinterpret_cast<unsigned long long*>(pd.win[dst] + PEER_OFF_FLAGS) +
           ((ch * 2 + (int)(seq & 1ull)) * PEER_MAXR + src);
}
// halo flags of a window: [parity][0 = written by rank-1 (my lo halo), 1 = written by rank+1 (my hi halo)]
__device__ __forceinline__ unsigned long long* peer_hflag(const PeerDev& pd, int dst, unsigned long long seq, int side) {
    return reinterpret_cast<unsigned long long*>(pd.win[dst] + PEER_OFF_HFLAGS) + ((int)(seq & 1ull) * 2 + side);
}
// one thread per rank waits until that rank's contribution `seq` has landed in MY window (local polling);
// the caller synchronises its threads afterwards
// Spin on a flag of MY window until it reaches seq.  The fast path is the bare acquire-load loop; every 1024
// polls (about a millisecond: only a wait that is already hopelessly late gets there) the watchdog described at
// PeerDev looks at the latch and at the clock.
__device__ __forceinline__ void peer_spin(const PeerDev& pd, const unsigned long long* f, unsigned long long seq) {
    unsigned polls = 0;
    unsigned long long t0 = 0;
    while (ld_acquire_sys_u64(f) < seq) {
        if ((++polls & 1023u) != 0 || pd.err == nullptr) continue;
        if (*(volatile int*)pd.err != 0) return;                  // an earlier wait has given up: so do we
        if (pd.timeout_ns == 0) continue;
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (t0 == 0) t0 = t;
        else if (t - t0 > pd.timeout_ns) {
            *(volatile int*)pd.err = 1;
            __threadfence_system();
            return;
        }
    }
}
__device__ __forceinline__ void peer_wait(const PeerDev& pd, int ch, unsigned long long seq, int tid) {
    if (tid < pd.nranks) peer_spin(pd, peer_flag(pd, pd.rank, ch, seq, tid), seq);
}
// single-thread publication of ONE double to every rank (SpMV dot epilogue, norm partial)
__device__ __forceinline__ void peer_publish1(const PeerDev& pd, int ch, unsigned long long seq, double v) {
    for (int p = 0; p < pd.nranks; ++p) peer_slot(pd, p, ch, seq, pd.rank)[0] = v;
    __threadfence_system();
    for (int p = 0; p < pd.nranks; ++p) st_relaxed_sys_u64(peer_flag(pd, p, ch, seq, pd.rank), seq);
}
// rank-ordered sum of the `nranks` contributions to element j (identical bits on every rank)
__device__ __forceinline__ double peer_sum1(const PeerDev& pd, int ch, unsigned long long seq, int j) {
    double a = 0.0;
    for (int p = 0; p < pd.nranks; ++p) a += ld_volatile_f64(peer_slot(pd, pd.rank, ch, seq, p) + j);
    return a;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes,
                                         uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}
// L2 eviction-priority hints.  The step alternates between streams that are read once (basis panels, the CSR
// arrays: evict_first) and ONE vector that the next kernel gathers from or re-reads (w = A v, the updated w:
// evict_last) — 80 MB at n = 1e7 against 50 MB of L2, so only part of it stays; without hints the multi-GB
// streams flush all of it.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar,
                                              uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void st_hint(double* p, double v, uint64_t policy) {
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(policy) : "memory");
}
__device__ __forceinline__ void st_hint(float* p, float v, uint64_t policy) {
    asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(policy) : "memory");
}

__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Deterministic block sum (fixed tree); valid result in thread 0.  `red` >= 32 doubles of smem.
__device__ __forceinline__ double block_sum(double v, double* red) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    if (w == 0) {
        s = (lane < nw) ? red[lane] : 0.0;
        s = warp_sum(s);
    }
    return s;
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ double splitmix_unit(uint64_t seed, uint64_t i) {
    return (double)(splitmix64(seed + i) >> 11) * (1.0 / 9007199254740992.0);
}

#endif  // __CUDACC__
