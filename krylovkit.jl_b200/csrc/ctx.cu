// ctx.cu — context, vector spaces (slabs), handle bookkeeping, scalar plumbing.
#include "common.cuh"
#include <cstdarg>
#include <algorithm>

std::string g_b2k_create_error;

// ------------------------------------------------------------------ memory ----
#include <mutex>
static std::mutex g_mem_mutex;
static bool g_pool_configured[64] = {false};
struct HostBlock { void* p; size_t bytes; };
static std::vector<HostBlock> g_host_cache;

// Large blocks (slabs, CSR arrays) are kept in an exact-size free list: repeated solves of the
// same shape — the host-buffer eigsolve path — then never touch the driver allocator.  (The
// stream-ordered pool alone splits a freed 6 GB slab to serve 400 MB requests and has to map
// fresh memory for the next slab: sporadic stalls, tools/e2e_breakdown.py times them.)
// Reuse across streams is made safe by an event recorded at free time.
#include <unordered_map>
#include <cstdlib>
constexpr size_t B2K_BIG_BYTES = (size_t)32 << 20;
struct BigBlock { void* p; size_t bytes; int dev; cudaEvent_t ev; };
static std::vector<BigBlock> g_big_free;
static std::unordered_map<void*, size_t> g_big_live;
static size_t g_big_cached = 0;

static size_t big_cap_bytes() {
    static size_t cap = 0;
    if (!cap) {
        const char* e = getenv("B2K_CACHE_GB");
        cap = (size_t)((e ? atof(e) : 16.0) * (double)((size_t)1 << 30));
    }
    return cap;
}

static void big_evict_locked(size_t keep_bytes) {
    while (!g_big_free.empty() && g_big_cached > keep_bytes) {
        BigBlock blk = g_big_free.front();
        g_big_free.erase(g_big_free.begin());
        cudaEventSynchronize(blk.ev);
        cudaEventDestroy(blk.ev);
        cudaFree(blk.p);
        g_big_cached -= blk.bytes;
    }
}

cudaError_t b2k_dmalloc(void** p, size_t bytes, cudaStream_t stream) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (bytes >= B2K_BIG_BYTES) {
        std::lock_guard<std::mutex> lk(g_mem_mutex);
        for (size_t i = 0; i < g_big_free.size(); ++i)
            if (g_big_free[i].bytes == bytes && g_big_free[i].dev == dev) {
                BigBlock blk = g_big_free[i];
                g_big_free.erase(g_big_free.begin() + i);
                g_big_cached -= bytes;
                cudaStreamWaitEvent(stream, blk.ev, 0);
                cudaEventDestroy(blk.ev);
                g_big_live[blk.p] = bytes;
                *p = blk.p;
                return cudaSuccess;
            }
        cudaError_t e = cudaMalloc(p, bytes);
        if (e != cudaSuccess) {       // give cached blocks back to the driver and retry
            cudaGetLastError();
            big_evict_locked(0);
            e = cudaMalloc(p, bytes);
        }
        if (e == cudaSuccess) g_big_live[*p] = bytes;
        return e;
    }
    {
        std::lock_guard<std::mutex> lk(g_mem_mutex);
        if (dev < 64 && !g_pool_configured[dev]) {
            cudaMemPool_t pool;
            if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
                uint64_t thr = UINT64_MAX;
                cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
            }
            g_pool_configured[dev] = true;
        }
    }
    return cudaMallocAsync(p, bytes ? bytes : 1, stream);
}

cudaError_t b2k_dfree(void* p, cudaStream_t stream) {
    if (!p) return cudaSuccess;
    {
        std::lock_guard<std::mutex> lk(g_mem_mutex);
        auto it = g_big_live.find(p);
        if (it != g_big_live.end()) {
            BigBlock blk;
            blk.p = p;
            blk.bytes = it->second;
            cudaGetDevice(&blk.dev);
            g_big_live.erase(it);
            cudaEventCreateWithFlags(&blk.ev, cudaEventDisableTiming);
            cudaEventRecord(blk.ev, stream);
            g_big_free.push_back(blk);
            g_big_cached += blk.bytes;
            big_evict_locked(big_cap_bytes());
            return cudaSuccess;
        }
    }
    return cudaFreeAsync(p, stream);
}

cudaError_t b2k_hmalloc(void** p, size_t bytes) {
    {
        std::lock_guard<std::mutex> lk(g_mem_mutex);
        for (size_t i = 0; i < g_host_cache.size(); ++i)
            if (g_host_cache[i].bytes == bytes) {
                *p = g_host_cache[i].p;
                g_host_cache.erase(g_host_cache.begin() + i);
                return cudaSuccess;
            }
    }
    return cudaHostAlloc(p, bytes, cudaHostAllocDefault);
}

void b2k_hfree(void* p, size_t bytes) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_mem_mutex);
    if (g_host_cache.size() < 64) g_host_cache.push_back({p, bytes});
    else cudaFreeHost(p);
}

extern "C" int32_t b2k_cache_release(void) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaMemPool_t pool;
    cudaDeviceSynchronize();
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
    std::lock_guard<std::mutex> lk(g_mem_mutex);
    big_evict_locked(0);
    for (auto& b : g_host_cache) cudaFreeHost(b.p);
    g_host_cache.clear();
    return B2K_OK;
}

int32_t b2k_fail(b2k_ctx* ctx, int32_t code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    else g_b2k_create_error = buf;
    return code;
}

extern "C" int32_t b2k_abi_version(void) { return B2K_ABI_VERSION; }

extern "C" const char* b2k_last_error(const b2k_ctx* ctx) {
    return ctx ? ctx->err.c_str() : g_b2k_create_error.c_str();
}

static int32_t make_space(b2k_ctx* ctx, int64_t n_local, int32_t ncols, int32_t sharded,
                          int32_t* space_out) {
    if (n_local < 0 || ncols <= 0 || ncols >= (1 << 20))
        return b2k_fail(ctx, B2K_EINVAL, "space: invalid n_local=%lld ncols=%d",
                        (long long)n_local, ncols);
    if ((int)ctx->spaces.size() >= B2K_MAX_SPACES)
        return b2k_fail(ctx, B2K_ENOMEM, "too many spaces");
    B2kSpace s;
    s.n = n_local;
    s.ld = ((n_local + 31) / 32) * 32;
    if (s.ld == 0) s.ld = 32;
    s.ncols = ncols;
    s.sharded = sharded;
    s.used.assign(ncols, 0);
    size_t bytes = (size_t)s.ld * ncols * ctx->esize;
    cudaError_t e = B2K_DMALLOC(&s.base, bytes);
    if (e != cudaSuccess)
        return b2k_fail(ctx, B2K_ENOMEM, "B2K_DMALLOC(%zu bytes) for slab failed: %s", bytes,
                        cudaGetErrorString(e));
    // zero the slab once: the ld-padding rows are read (never written) by the bulk copies
    B2K_CUDA(ctx, cudaMemsetAsync(s.base, 0, bytes, ctx->stream));
    ctx->spaces.push_back(std::move(s));
    *space_out = (int32_t)ctx->spaces.size() - 1;
    return B2K_OK;
}

static int32_t ctx_create_common(b2k_ctx** out, int32_t device, int64_t n_local,
                                 int32_t ncols, int32_t dtype) {
    if (!out) return b2k_fail(nullptr, B2K_EINVAL, "ctx_create: out is NULL");
    *out = nullptr;
    if (dtype != B2K_F64 && dtype != B2K_F32)
        return b2k_fail(nullptr, B2K_EINVAL, "ctx_create: unknown dtype %d", dtype);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return b2k_fail(nullptr, B2K_ECUDA,
                        "ctx_create: no CUDA device available (%s) — this engine has no CPU "
                        "fallback", cudaGetErrorString(e));
    if (device < 0 || device >= ndev)
        return b2k_fail(nullptr, B2K_EINVAL, "ctx_create: device %d out of range [0,%d)",
                        device, ndev);
    b2k_ctx* ctx = new b2k_ctx();
    ctx->device = device;
    ctx->dtype = dtype;
    ctx->esize = (dtype == B2K_F64) ? 8 : 4;
#define CK(call)                                                                          \
    do {                                                                                  \
        cudaError_t e2 = (call);                                                          \
        if (e2 != cudaSuccess) {                                                          \
            int32_t rc = b2k_fail(nullptr, B2K_ECUDA, "ctx_create: %s -> %s", #call,      \
                                  cudaGetErrorString(e2));                                \
            delete ctx;                                                                   \
            return rc;                                                                    \
        }                                                                                 \
    } while (0)
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        fprintf(stderr, "[b200krylov] warning: device %s is sm_%d%d; this library is built for "
                        "sm_90a only\n", prop.name, prop.major, prop.minor);
    ctx->num_sms = prop.multiProcessorCount;
    // No persisting-L2 set-aside by default: a set-aside shrinks the L2 that every other streaming kernel of the
    // process uses.  Residency is requested per access with L2 eviction-priority hints instead, which need no
    // set-aside.  B2K_L2_CARVE=<bytes> reserves one (and the access-policy window that pins the MGS sweep's vector).
    size_t carve = 0;
    if (const char* e = getenv("B2K_L2_CARVE"))
        carve = std::min((size_t)(prop.persistingL2CacheMaxSize > 0 ? prop.persistingL2CacheMaxSize : 0),
                         (size_t)strtoull(e, nullptr, 10));
    if (carve == 0) {
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0);      // another library in the process may have set one
        cudaGetLastError();
    } else if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve) == cudaSuccess) {
        ctx->l2_persist_bytes = carve;
        ctx->l2_window_max = (size_t)prop.accessPolicyMaxWindowSize;
    } else {
        cudaGetLastError();
    }
    CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    CK(B2K_DMALLOC(&ctx->d_part, sizeof(double) * 4 * (size_t)B2K_MAX_GRID * B2K_KSTRIDE));
    CK(B2K_DMALLOC(&ctx->d_part_s, sizeof(double) * (1 << 20)));
    CK(B2K_DMALLOC(&ctx->d_res, sizeof(double) * B2K_RES_DOUBLES));
    CK(b2k_hmalloc((void**)&ctx->h_res, sizeof(double) * B2K_RES_DOUBLES));
    CK(B2K_DMALLOC(&ctx->d_coef, sizeof(double) * B2K_COEF_DOUBLES));
    CK(b2k_hmalloc((void**)&ctx->h_coef, sizeof(double) * B2K_COEF_DOUBLES));
    CK(B2K_DMALLOC(&ctx->d_steps, sizeof(double) * 2 * B2K_REC * (B2K_MAX_CHAIN + 1)));
    CK(cudaMemsetAsync(ctx->d_steps, 0, sizeof(double) * 2 * B2K_REC * (B2K_MAX_CHAIN + 1), ctx->stream));
    CK(B2K_DMALLOC(&ctx->d_blk, sizeof(double) * (2 * B2K_BLK_HCAP + 64)));
    CK(B2K_DMALLOC(&ctx->d_blkpart, sizeof(double) * (size_t)B2K_MAX_GRID * B2K_BLK_PART));
    CK(B2K_DMALLOC(&ctx->d_sync, sizeof(unsigned) * 64));
    CK(cudaMemsetAsync(ctx->d_sync, 0, sizeof(unsigned) * 64, ctx->stream));
    CK(cudaMemsetAsync(ctx->d_part, 0, sizeof(double) * 4 * (size_t)B2K_MAX_GRID * B2K_KSTRIDE,
                       ctx->stream));
    CK(cudaEventCreateWithFlags(&ctx->ev_coef, cudaEventDisableTiming));
#undef CK
    int32_t sp = 0;
    int32_t rc = b2k_basis_init(ctx);
    if (rc == B2K_OK) rc = b2k_spmv_init(ctx);
    if (rc == B2K_OK) rc = b2k_block_init(ctx);
    if (rc == B2K_OK) rc = make_space(ctx, n_local, ncols, 1, &sp);
    if (rc != B2K_OK) {
        g_b2k_create_error = ctx->err;
        b2k_ctx_destroy(ctx);
        return rc;
    }
    ctx->n_global = n_local;
    ctx->row_offset = 0;
    *out = ctx;
    return B2K_OK;
}

extern "C" int32_t b2k_ctx_create(b2k_ctx** out, int32_t device, int64_t n_local,
                                  int32_t ncols, int32_t dtype) {
    return ctx_create_common(out, device, n_local, ncols, dtype);
}

extern "C" int32_t b2k_ctx_create_dist(b2k_ctx** out, int32_t device, int64_t n_local,
                                       int32_t ncols, int32_t dtype, int32_t rank,
                                       int32_t nranks, const void* nccl_uid, int64_t n_global,
                                       int64_t row_offset) {
    if (nranks < 1 || rank < 0 || rank >= nranks)
        return b2k_fail(nullptr, B2K_EINVAL, "ctx_create_dist: bad rank %d / %d", rank, nranks);
    B2K_TRY(ctx_create_common(out, device, n_local, ncols, dtype));
    b2k_ctx* ctx = *out;
    ctx->rank = rank;
    ctx->nranks = nranks;
    ctx->n_global = n_global;
    ctx->row_offset = row_offset;
    if (nranks > 1) {
        int32_t rc = b2k_nccl_init(ctx, nccl_uid);
        if (rc != B2K_OK) {
            g_b2k_create_error = ctx->err;
            b2k_ctx_destroy(ctx);
            *out = nullptr;
            return rc;
        }
    }
    return B2K_OK;
}

extern "C" int32_t b2k_ctx_destroy(b2k_ctx* ctx) {
    if (!ctx) return B2K_OK;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (b2k_op* op : ctx->ops) b2k_op_release(ctx, op);
    ctx->ops.clear();
    b2k_nccl_destroy(ctx);
    for (auto& s : ctx->spaces)
        if (s.base) B2K_DFREE(s.base);
    if (ctx->d_part) B2K_DFREE(ctx->d_part);
    if (ctx->d_part_s) B2K_DFREE(ctx->d_part_s);
    if (ctx->d_res) B2K_DFREE(ctx->d_res);
    b2k_hfree(ctx->h_res, sizeof(double) * B2K_RES_DOUBLES);
    if (ctx->d_coef) B2K_DFREE(ctx->d_coef);
    b2k_hfree(ctx->h_coef, sizeof(double) * B2K_COEF_DOUBLES);
    if (ctx->d_sync) B2K_DFREE(ctx->d_sync);
    if (ctx->d_steps) B2K_DFREE(ctx->d_steps);
    if (ctx->d_blk) B2K_DFREE(ctx->d_blk);
    if (ctx->d_blkpart) B2K_DFREE(ctx->d_blkpart);
    if (ctx->d_trace) cudaFree(ctx->d_trace);           // b2k_debug_trace left on
    if (ctx->ev_coef) cudaEventDestroy(ctx->ev_coef);
    if (ctx->ev_t0) cudaEventDestroy(ctx->ev_t0);
    if (ctx->ev_t1) cudaEventDestroy(ctx->ev_t1);
    for (cudaEvent_t e : ctx->prof.pool) cudaEventDestroy(e);
    if (ctx->stream) {
        cudaStreamSynchronize(ctx->stream);
        cudaStreamDestroy(ctx->stream);
    }
    delete ctx;
    return B2K_OK;
}

extern "C" int32_t b2k_space_create(b2k_ctx* ctx, int64_t n_local, int32_t ncols,
                                    int32_t sharded, int32_t* space_out) {
    if (!ctx || !space_out) return B2K_EINVAL;
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    return make_space(ctx, n_local, ncols, sharded, space_out);
}

extern "C" int32_t b2k_ctx_sync(b2k_ctx* ctx) {
    if (!ctx) return B2K_EINVAL;
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

extern "C" int64_t b2k_ctx_launch_count(const b2k_ctx* ctx) { return ctx ? ctx->launches : 0; }
// debugging aid (not in the public header): number of slab columns of a space currently handed out
extern "C" int32_t b2k_debug_used_columns(const b2k_ctx* ctx, int32_t space) {
    if (!ctx || space < 0 || space >= (int32_t)ctx->spaces.size()) return -1;
    int32_t c = 0;
    for (uint8_t u : ctx->spaces[space].used) c += u ? 1 : 0;
    return c;
}
extern "C" void* b2k_ctx_stream(b2k_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// ------------------------------------------------------------------ handles ----

int32_t b2k_resolve(b2k_ctx* ctx, b2k_vec v, VecRef* out) {
    int32_t sp = B2K_VEC_SPACE(v), col = B2K_VEC_COL(v);
    if (v < 0 || sp >= (int32_t)ctx->spaces.size())
        return b2k_fail(ctx, B2K_EINVAL, "invalid vector handle 0x%x (space %d)", v, sp);
    B2kSpace& s = ctx->spaces[sp];
    if (col >= s.ncols || !s.used[col])
        return b2k_fail(ctx, B2K_EINVAL, "vector handle 0x%x: column %d not allocated", v, col);
    out->ptr = (char*)s.base + (size_t)col * s.ld * ctx->esize;
    out->n = s.n;
    out->ld = s.ld;
    out->space = sp;
    out->col = col;
    out->sharded = s.sharded;
    return B2K_OK;
}

int32_t b2k_resolve_cols(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, int32_t* space,
                         std::vector<int32_t>* idx) {
    if (k < 0 || (k > 0 && !cols)) return b2k_fail(ctx, B2K_EINVAL, "bad column list");
    idx->resize(k);
    int32_t sp = -1;
    for (int32_t j = 0; j < k; ++j) {
        VecRef r;
        B2K_TRY(b2k_resolve(ctx, cols[j], &r));
        if (sp < 0) sp = r.space;
        else if (sp != r.space)
            return b2k_fail(ctx, B2K_EDIM, "basis vectors live in different spaces");
        (*idx)[j] = r.col;
    }
    *space = sp;
    return B2K_OK;
}

int32_t b2k_resolve_vecs(b2k_ctx* ctx, const char* entry, std::initializer_list<b2k_vec> hs, VecRef* out,
                         bool distinct) {
    const int n = (int)hs.size();
    int i = 0;
    for (b2k_vec h : hs) B2K_TRY(b2k_resolve(ctx, h, &out[i++]));
    for (i = 1; i < n; ++i)
        if (out[i].n != out[0].n) return b2k_fail(ctx, B2K_EDIM, "%s: length mismatch", entry);
    if (distinct)
        for (i = 0; i < n; ++i)
            for (int j = 0; j < i; ++j)
                if (out[i].ptr == out[j].ptr)
                    return b2k_fail(ctx, B2K_EINVAL, "%s: vectors %d and %d are the same", entry, j, i);
    return B2K_OK;
}

extern "C" int32_t b2k_vec_alloc(b2k_ctx* ctx, int32_t space, b2k_vec* out) {
    if (!ctx || !out) return B2K_EINVAL;
    if (space < 0 || space >= (int32_t)ctx->spaces.size())
        return b2k_fail(ctx, B2K_EINVAL, "vec_alloc: bad space %d", space);
    B2kSpace& s = ctx->spaces[space];
    for (int32_t c = 0; c < s.ncols; ++c)
        if (!s.used[c]) {
            s.used[c] = 1;
            *out = B2K_VEC(space, c);
            return B2K_OK;
        }
    return b2k_fail(ctx, B2K_ENOMEM, "vec_alloc: slab %d has no free column (%d in use)", space,
                    s.ncols);
}

extern "C" int32_t b2k_vec_alloc_range(b2k_ctx* ctx, int32_t space, int32_t count,
                                       b2k_vec* first) {
    if (!ctx || !first || count <= 0) return B2K_EINVAL;
    if (space < 0 || space >= (int32_t)ctx->spaces.size())
        return b2k_fail(ctx, B2K_EINVAL, "vec_alloc_range: bad space %d", space);
    B2kSpace& s = ctx->spaces[space];
    int32_t run = 0;
    for (int32_t c = 0; c < s.ncols; ++c) {
        run = s.used[c] ? 0 : run + 1;
        if (run == count) {
            int32_t c0 = c - count + 1;
            for (int32_t i = c0; i <= c; ++i) s.used[i] = 1;
            *first = B2K_VEC(space, c0);
            return B2K_OK;
        }
    }
    return b2k_fail(ctx, B2K_ENOMEM, "vec_alloc_range: no %d consecutive free columns", count);
}

extern "C" int32_t b2k_vec_free(b2k_ctx* ctx, b2k_vec v) {
    if (!ctx) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    ctx->spaces[r.space].used[r.col] = 0;
    return B2K_OK;
}

extern "C" int32_t b2k_vec_upload(b2k_ctx* ctx, b2k_vec v, const void* host) {
    if (!ctx || !host) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    B2K_CUDA(ctx, cudaMemcpyAsync(r.ptr, host, (size_t)r.n * ctx->esize, cudaMemcpyHostToDevice,
                                  ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

extern "C" int32_t b2k_vec_download(b2k_ctx* ctx, b2k_vec v, void* host) {
    if (!ctx || !host) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    B2K_CUDA(ctx, cudaSetDevice(ctx->device));
    B2K_CUDA(ctx, cudaMemcpyAsync(host, r.ptr, (size_t)r.n * ctx->esize, cudaMemcpyDeviceToHost,
                                  ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

extern "C" int32_t b2k_vec_copy(b2k_ctx* ctx, b2k_vec dst, b2k_vec src) {
    if (!ctx) return B2K_EINVAL;
    VecRef d, s;
    B2K_TRY(b2k_resolve(ctx, dst, &d));
    B2K_TRY(b2k_resolve(ctx, src, &s));
    if (d.n != s.n) return b2k_fail(ctx, B2K_EDIM, "vec_copy: length %lld vs %lld",
                                    (long long)d.n, (long long)s.n);
    if (d.ptr == s.ptr) return B2K_OK;
    B2K_CUDA(ctx, cudaMemcpyAsync(d.ptr, s.ptr, (size_t)d.n * ctx->esize,
                                  cudaMemcpyDeviceToDevice, ctx->stream));
    return B2K_OK;
}

extern "C" int32_t b2k_vec_zero(b2k_ctx* ctx, b2k_vec v) {
    if (!ctx) return B2K_EINVAL;
    VecRef r;
    B2K_TRY(b2k_resolve(ctx, v, &r));
    B2K_CUDA(ctx, cudaMemsetAsync(r.ptr, 0, (size_t)r.n * ctx->esize, ctx->stream));
    return B2K_OK;
}

// ------------------------------------------------------------ scalar plumbing ----

int32_t b2k_allreduce(b2k_ctx* ctx, double* dptr, int32_t count, int32_t sharded) {
    if (ctx->nranks > 1 && sharded) {
        // over the peer window every count is the rank-order fold, in slot-sized pieces, whether or not the
        // context also has an NCCL communicator
        if (b2k_peer_ok(ctx)) {
            for (int32_t off = 0; off < count; off += PEER_SLOT)
                B2K_TRY(b2k_peer_allreduce(ctx, dptr + off, std::min<int32_t>(PEER_SLOT, count - off)));
            return B2K_OK;
        }
        return b2k_nccl_allreduce_f64(ctx, dptr, count);
    }
    return B2K_OK;
}

int32_t b2k_fetch_results(b2k_ctx* ctx, int32_t count, int32_t sharded) {
    if (count > B2K_RES_DOUBLES) return b2k_fail(ctx, B2K_EINVAL, "fetch_results: too many");
    B2K_TRY(b2k_allreduce(ctx, ctx->d_res, count, sharded));
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, ctx->d_res, sizeof(double) * count,
                                  cudaMemcpyDeviceToHost, ctx->stream));
    B2K_TRY(b2k_stream_sync(ctx));
    return B2K_OK;
}

static int32_t wait_staging(b2k_ctx* ctx) {
    if (ctx->coef_busy) {
        B2K_CUDA(ctx, cudaEventSynchronize(ctx->ev_coef));
        ctx->coef_busy = false;
    }
    return B2K_OK;
}

int32_t b2k_put_coef(b2k_ctx* ctx, const double* host, int32_t count, int32_t offset) {
    if (count < 0 || offset < 0 || offset + count > B2K_COEF_DOUBLES)
        return b2k_fail(ctx, B2K_EINVAL, "put_coef: %d doubles at %d exceeds staging", count,
                        offset);
    if (count == 0) return B2K_OK;
    B2K_TRY(wait_staging(ctx));
    memcpy(ctx->h_coef + offset, host, sizeof(double) * count);
    B2K_CUDA(ctx, cudaMemcpyAsync(ctx->d_coef + offset, ctx->h_coef + offset,
                                  sizeof(double) * count, cudaMemcpyHostToDevice, ctx->stream));
    B2K_CUDA(ctx, cudaEventRecord(ctx->ev_coef, ctx->stream));
    ctx->coef_busy = true;
    return B2K_OK;
}

// ------------------------------------------------------------ chained calls ----

B2kChain::B2kChain(b2k_ctx* c, int ns, int rl)
    : ctx(c), st(c->d_steps), rec0(c->d_steps + ns), stop(reinterpret_cast<int*>(c->d_sync + B2K_SYNC_STOP)),
      skip(reinterpret_cast<int*>(c->d_sync + B2K_SYNC_SKIP)), nstate(ns), rec_len(rl) {}

int32_t B2kChain::seed(const double* s, int ns, int nclear, bool with_skip) {
    return enqueue([&]() -> int32_t {
        B2K_TRY(b2k_put_coef(ctx, s, ns, 0));
        B2K_CUDA(ctx, cudaMemcpyAsync(st, ctx->d_coef, ns * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        if (nclear > 0)
            B2K_CUDA(ctx, cudaMemsetAsync(rec0, 0, sizeof(double) * rec_len * nclear, ctx->stream));
        B2K_CUDA(ctx, cudaMemsetAsync(stop, 0, sizeof(int), ctx->stream));
        if (with_skip) B2K_CUDA(ctx, cudaMemsetAsync(skip, 0, sizeof(int), ctx->stream));
        return B2K_OK;
    });
}

int32_t B2kChain::fail(int32_t rc) {
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

int32_t B2kChain::fetch(int nrec, int nst) {
    const size_t rbytes = sizeof(double) * rec_len * nrec;
    B2K_TRY(enqueue([&]() -> int32_t {
        if (nst > 0 && nstate + (size_t)rec_len * nrec <= (size_t)B2K_RES_DOUBLES) {
            // state and records are one block of d_steps
            hst = ctx->h_res;
            hrec = ctx->h_res + nstate;
            B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, st, sizeof(double) * nstate + rbytes, cudaMemcpyDeviceToHost,
                                          ctx->stream));
            return B2K_OK;
        }
        hrec = ctx->h_res;
        hst = ctx->h_res + B2K_RES_DOUBLES - nst;
        B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, rec0, rbytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (nst > 0)
            B2K_CUDA(ctx, cudaMemcpyAsync(ctx->h_res + B2K_RES_DOUBLES - nst, st, sizeof(double) * nst,
                                          cudaMemcpyDeviceToHost, ctx->stream));
        return B2K_OK;
    }));
    return b2k_stream_sync(ctx);
}

int32_t B2kChainCols::alloc(int32_t space, b2k_vec* h) {
    B2K_TRY(b2k_vec_alloc(ctx, space, h));
    touched.push_back(*h);
    return B2K_OK;
}

void B2kChainCols::consumed(b2k_vec h) { ctx->spaces[B2K_VEC_SPACE(h)].used[B2K_VEC_COL(h)] = 0; }

void B2kChainCols::ran(b2k_vec ui, b2k_vec vi, b2k_vec wi) {
    u.push_back(ui);
    v.push_back(vi);
    w.push_back(wi);
}

b2k_vec B2kChainCols::commit(int32_t d, b2k_vec* ucols, b2k_vec* vcols, int32_t k) {
    auto keep = [&](b2k_vec* cols, int32_t i, b2k_vec h) {
        cols[i] = h;
        ctx->spaces[B2K_VEC_SPACE(h)].used[B2K_VEC_COL(h)] = 1;
    };
    for (b2k_vec h : touched) consumed(h);
    for (int32_t i = 0; i < d; ++i) {          // (skipped steps overwrote the columns behind ucols[k + d])
        keep(ucols, k + i, u[i]);
        if (vcols) keep(vcols, k + i, v[i]);
    }
    keep(ucols, k + d, d > 0 ? w[d - 1] : touched[0]);
    return ucols[k + d];
}

// ------------------------------------------------------------------ profiling ----

int b2k_prof_begin(b2k_ctx* ctx, int cls, double bytes) {
    B2kProf& pf = ctx->prof;
    if (!pf.on) return -1;
    if (pf.next + 2 > pf.pool.size()) {
        if (pf.pool.size() >= 65536) return -1;
        for (int i = 0; i < 512; ++i) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return -1;
            pf.pool.push_back(e);
        }
    }
    B2kProfRec r;
    r.cls = cls;
    r.bytes = bytes;
    r.e0 = pf.pool[pf.next++];
    r.e1 = pf.pool[pf.next++];
    cudaEventRecord(r.e0, ctx->stream);
    pf.recs.push_back(r);
    return (int)pf.recs.size() - 1;
}

void b2k_prof_end(b2k_ctx* ctx, int idx) {
    if (idx < 0) return;
    cudaEventRecord(ctx->prof.recs[idx].e1, ctx->stream);
}

extern "C" int32_t b2k_prof_enable(b2k_ctx* ctx, int32_t on) {
    if (!ctx) return B2K_EINVAL;
    ctx->prof.on = on != 0;
    return B2K_OK;
}

extern "C" int32_t b2k_prof_reset(b2k_ctx* ctx) {
    if (!ctx) return B2K_EINVAL;
    B2K_TRY(b2k_stream_sync(ctx));
    ctx->prof.recs.clear();
    ctx->prof.next = 0;
    return B2K_OK;
}

extern "C" int32_t b2k_prof_read(b2k_ctx* ctx, int32_t cls, int64_t* count, double* ms,
                                 double* bytes) {
    if (!ctx || cls < 0 || cls >= B2K_PROF_CLASSES) return B2K_EINVAL;
    B2K_TRY(b2k_stream_sync(ctx));
    int64_t c = 0;
    double t = 0.0, b = 0.0;
    for (const B2kProfRec& r : ctx->prof.recs) {
        if (r.cls != cls) continue;
        float m = 0.f;
        if (cudaEventElapsedTime(&m, r.e0, r.e1) != cudaSuccess) continue;
        ++c;
        t += m;
        b += r.bytes;
    }
    if (count) *count = c;
    if (ms) *ms = t;
    if (bytes) *bytes = b;
    return B2K_OK;
}

// ------------------------------------------------------------------ host helpers ----

extern "C" int32_t b2k_pinned_alloc(size_t bytes, void** out) {
    if (!out) return B2K_EINVAL;
    cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) return b2k_fail(nullptr, B2K_ENOMEM, "cudaHostAlloc(%zu) -> %s", bytes,
                                          cudaGetErrorString(e));
    return B2K_OK;
}

extern "C" int32_t b2k_pinned_free(void* p) {
    if (p) cudaFreeHost(p);
    return B2K_OK;
}

extern "C" int32_t b2k_device_sync(void) {
    return cudaDeviceSynchronize() == cudaSuccess ? B2K_OK : B2K_ECUDA;
}

extern "C" int32_t b2k_timer_start(b2k_ctx* ctx) {
    if (!ctx) return B2K_EINVAL;
    if (!ctx->ev_t0) {
        B2K_CUDA(ctx, cudaEventCreate(&ctx->ev_t0));
        B2K_CUDA(ctx, cudaEventCreate(&ctx->ev_t1));
    }
    B2K_TRY(b2k_stream_sync(ctx));
    B2K_CUDA(ctx, cudaEventRecord(ctx->ev_t0, ctx->stream));
    return B2K_OK;
}

extern "C" int32_t b2k_timer_stop(b2k_ctx* ctx, double* ms) {
    if (!ctx || !ms || !ctx->ev_t0) return B2K_EINVAL;
    B2K_CUDA(ctx, cudaEventRecord(ctx->ev_t1, ctx->stream));
    B2K_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1));
    float f = 0.f;
    B2K_CUDA(ctx, cudaEventElapsedTime(&f, ctx->ev_t0, ctx->ev_t1));
    *ms = f;
    return B2K_OK;
}
