// dab_core.cu -- lifecycle, buffers, events, fill!, rand!  (C ABI: include/dab200.h)
#include <cstdarg>
#include <cstdlib>
#include <map>
#include <mutex>
#include <new>
#include <thread>
#include <unordered_map>

#include "dab_common.cuh"

thread_local char dab_tls_err[512] = "";

// Small device blocks (results of dimensional reductions, halo temporaries, ...) are recycled instead of going back to
// cudaFree: once peer access is enabled (CUDA IPC mailboxes / halo mappings) every cudaMalloc / cudaFree has to update the peers'
// page tables and costs milliseconds -- measured 14 ms for a sum(A, dims=1) call that allocates three small arrays.  Blocks stay
// plain cudaMalloc memory, so they remain exportable with cudaIpcGetMemHandle.
struct dab_alloc_cache {
    std::unordered_map<void*, size_t> live;   // block -> rounded size (cacheable blocks only)
    std::multimap<size_t, void*> free_blocks;
    size_t cached_bytes = 0;
    // localpart-sized blocks are recycled too (an `x = A * x` loop allocates and frees the same sizes over and over, and a cudaMalloc /
    // cudaFree pair of a 256 MiB block costs ~5 ms and synchronises the device); when the device runs out of memory the cache is flushed
    static constexpr size_t kMaxBlock = 16ull << 30;
    static constexpr size_t kMaxCached = 32ull << 30;
};

int dab_resident_ctas(const void* kernel, int threads) {
    static std::mutex mu;
    static std::unordered_map<const void*, int> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(kernel);
    if (it != cache.end()) return it->second;
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, 0) != cudaSuccess || n < 1) {
        cudaGetLastError();
        n = 1;
    }
    cache[kernel] = n;
    return n;
}

int32_t dab_fail(dab_ctx* ctx, int32_t status, const char* fmt, ...) {
    char* dst = ctx ? ctx->err : dab_tls_err;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(dst, 512, fmt, ap);
    va_end(ap);
    if (ctx) memcpy(dab_tls_err, dst, 512);
    return status;
}

int32_t dab_fail_cuda(dab_ctx* ctx, cudaError_t e, const char* what, const char* file, int line) {
    // clear the (non-sticky) error state so it does not leak into the next call
    cudaGetLastError();
    return dab_fail(ctx, e == cudaErrorMemoryAllocation ? DAB_ERR_NOMEM : DAB_ERR_CUDA, "CUDA error %d (%s) in %s at %s:%d",
                    (int)e, cudaGetErrorString(e), what, file, line);
}

int32_t dab_scratch_grow(dab_ctx* ctx, void** buf, size_t* have, size_t bytes, bool zero) {
    if (*have >= bytes) return DAB_OK;
    if (*buf) {
        DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        DAB_CUDA(ctx, cudaFree(*buf));
        *buf = nullptr;
        *have = 0;
    }
    DAB_CUDA(ctx, cudaMalloc(buf, bytes));
    if (zero) DAB_CUDA(ctx, cudaMemsetAsync(*buf, 0, bytes, ctx->stream));
    *have = bytes;
    return DAB_OK;
}

extern "C" {

int32_t dab_abi_version(void) { return DAB_ABI_VERSION; }

const char* dab_status_string(int32_t s) {
    switch (s) {
        case DAB_OK: return "ok";
        case DAB_ERR_CUDA: return "CUDA error";
        case DAB_ERR_ARG: return "ArgumentError";
        case DAB_ERR_EMPTY: return "ArgumentError: reducing over an empty collection is not allowed";
        case DAB_ERR_DIM_MISMATCH: return "DimensionMismatch";
        case DAB_ERR_NCCL: return "NCCL error";
        case DAB_ERR_UNSUPPORTED: return "unsupported op/dtype (no host fallback)";
        case DAB_ERR_NVRTC: return "NVRTC error";
        case DAB_ERR_NOMEM: return "out of device memory";
        default: return "unknown status";
    }
}

const char* dab_last_error(const dab_ctx* ctx) { return ctx ? ctx->err : dab_tls_err; }

int32_t dab_device_count(int32_t* count) {
    if (!count) return dab_fail(nullptr, DAB_ERR_ARG, "null count");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        *count = 0;
        return dab_fail_cuda(nullptr, e, "cudaGetDeviceCount", __FILE__, __LINE__);
    }
    *count = n;
    return DAB_OK;
}

int32_t dab_init(int32_t device, dab_ctx** out) {
    if (!out) return dab_fail(nullptr, DAB_ERR_ARG, "null ctx out-pointer");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return dab_fail_cuda(nullptr, e, "cudaGetDeviceCount", __FILE__, __LINE__);
    if (device < 0 || device >= n) return dab_fail(nullptr, DAB_ERR_ARG, "device %d out of range (have %d)", device, n);
    dab_ctx* ctx = new (std::nothrow) dab_ctx();
    if (!ctx) return dab_fail(nullptr, DAB_ERR_NOMEM, "host allocation failed");
    memset(ctx, 0, sizeof(*ctx));
    ctx->device = device;
    ctx->rank = 0;
    ctx->nranks = 1;
    ctx->fuse_op = -1;
    ctx->opt_combine_timeout_ms = 120000;
    ctx->cache = new (std::nothrow) dab_alloc_cache();
#define INIT_CUDA(call)                                                     \
    do {                                                                    \
        cudaError_t e__ = (call);                                           \
        if (e__ != cudaSuccess) {                                           \
            int32_t st = dab_fail_cuda(nullptr, e__, #call, __FILE__, __LINE__); \
            delete ctx;                                                     \
            return st;                                                      \
        }                                                                   \
    } while (0)
    INIT_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    INIT_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code (wgmma, TMA) runs on compute capability 9.0 only
        delete ctx;
        return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "device %d is sm_%d%d; libdab200 is built for sm_90a only", device,
                        prop.major, prop.minor);
    }
    ctx->sm_count = prop.multiProcessorCount;
    INIT_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    {
        cudaMemPool_t pool;
        INIT_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        unsigned long long keep = ~0ull;
        INIT_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    INIT_CUDA(cudaMalloc(&ctx->block_partials, ((size_t)DAB_MAX_REDUCE_BLOCKS + DAB_MAX_REDUCE_BLOCKS / 256 + 16) * 16));
    INIT_CUDA(cudaMalloc((void**)&ctx->counter, (DAB_MAX_REDUCE_BLOCKS / 256 + 16) * 4));
    INIT_CUDA(cudaMemsetAsync(ctx->counter, 0, (DAB_MAX_REDUCE_BLOCKS / 256 + 16) * 4, ctx->stream));
    INIT_CUDA(cudaMalloc(&ctx->result_slot, DAB_SLOT_BYTES));
    INIT_CUDA(cudaMalloc(&ctx->gather_slots, (size_t)DAB_MAX_RANKS * 16));
    INIT_CUDA(cudaHostAlloc(&ctx->host_slot, (size_t)(DAB_MAX_RANKS + 2) * 16, cudaHostAllocDefault));
    INIT_CUDA(cudaStreamSynchronize(ctx->stream));
    memset(ctx->host_slot, 0, (size_t)(DAB_MAX_RANKS + 2) * 16);
#undef INIT_CUDA
    *out = ctx;
    return DAB_OK;
}

int32_t dab_comm_destroy(dab_ctx* ctx);
int32_t dab_mailbox_detach(dab_ctx* ctx);

int32_t dab_shutdown(dab_ctx* ctx) {
    if (!ctx) return DAB_OK;
    cudaSetDevice(ctx->device);
    const int32_t st = dab_flush_pending(ctx);  // no DAB_ENTER here: a deferred dab_affine still runs before the teardown
    cudaStreamSynchronize(ctx->stream);
    if (ctx->comm) dab_comm_destroy(ctx);
    cudaFree(ctx->block_partials);
    cudaFree(ctx->counter);
    cudaFree(ctx->result_slot);
    cudaFree(ctx->gather_slots);
    if (ctx->dim_scratch) cudaFree(ctx->dim_scratch);
    if (ctx->sort_dev) cudaFree(ctx->sort_dev);
    if (ctx->scan_dev) cudaFree(ctx->scan_dev);
    if (ctx->scan_scratch) cudaFree(ctx->scan_scratch);
    if (ctx->sort_host) cudaFreeHost(ctx->sort_host);
    for (int b = 0; b < 2; ++b)
        if (ctx->stage[b]) {
            cudaFreeHost(ctx->stage[b]);
            cudaEventDestroy(ctx->stage_ev[b]);
        }
    if (ctx->cache) {
        for (auto& kv : ctx->cache->free_blocks) cudaFree(kv.second);
        delete ctx->cache;
        ctx->cache = nullptr;
    }
    dab_mailbox_detach(ctx);
    cudaFreeHost(ctx->host_slot);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return st;
}

int32_t dab_sync(dab_ctx* ctx) {
    DAB_ENTER(ctx);
    DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    volatile unsigned long long* status = (volatile unsigned long long*)((char*)ctx->host_slot + (DAB_MAX_RANKS + 1) * 16);
    if (*status != 0) {   // set by peer_barrier_kernel (dab_comm.cu) when a peer never arrived
        *status = 0;
        return dab_fail(ctx, DAB_ERR_NCCL, "device-side peer barrier timed out waiting for another rank (did every rank make the same collective call?)");
    }
    return DAB_OK;
}

int32_t dab_device_info(dab_ctx* ctx, int32_t* device, int32_t* sm_count, size_t* free_bytes, size_t* total_bytes) {
    DAB_ENTER(ctx);
    size_t f = 0, t = 0;
    DAB_CUDA(ctx, cudaMemGetInfo(&f, &t));
    if (device) *device = ctx->device;
    if (sm_count) *sm_count = ctx->sm_count;
    if (free_bytes) *free_bytes = f + (ctx->cache ? ctx->cache->cached_bytes : 0);   // recycled blocks are given back on demand
    if (total_bytes) *total_bytes = t;
    return DAB_OK;
}

// Whoever holds the raw stream may queue work on it directly, and that work expects every earlier call of this ctx to be
// queued already: DAB_ENTER flushes, and dab_affine stops deferring for the rest of the ctx's life.
int32_t dab_stream(dab_ctx* ctx, void** stream) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, stream, DAB_ERR_ARG, "null stream out-pointer");
    ctx->defer_off = 1;
    *stream = (void*)ctx->stream;
    return DAB_OK;
}

// Two switches.  "ew_tma" = 1: unary elementwise kernels (dab_affine, dab_unary, dab_binary_scalar) use the TMA-staged
// shared-memory ring instead of the default flat LDG/STG kernel (same results; measured slower, see dab_elementwise.cu).
// "combine_timeout_ms": how long the fused combine waits for a peer before it reports a dead rank.
int32_t dab_set_option(dab_ctx* ctx, const char* key, int64_t value) {
    if (!ctx || !key) return dab_fail(ctx, DAB_ERR_ARG, "null argument");
    if (ctx->pending.active) {  // no DAB_ENTER here: a deferred dab_affine launches as it was called, before the switch changes
        DAB_CUDA(ctx, cudaSetDevice(ctx->device));
        DAB_FLUSH(ctx);
    }
    if (strcmp(key, "ew_tma") == 0) {
        ctx->opt_ew_tma = value != 0;
        return DAB_OK;
    }
    if (strcmp(key, "combine_timeout_ms") == 0) {
        if (value < 1) return dab_fail(ctx, DAB_ERR_ARG, "combine_timeout_ms must be >= 1");
        ctx->opt_combine_timeout_ms = value;
        return DAB_OK;
    }
    return dab_fail(ctx, DAB_ERR_ARG, "dab_set_option: unknown key %s", key);
}

int32_t dab_launch_count(dab_ctx* ctx, uint64_t* launches) {
    if (!ctx || !launches) return dab_fail(ctx, DAB_ERR_ARG, "null argument");
    if (ctx->pending.active) {  // no DAB_ENTER here: count a deferred dab_affine as launched -- it is, from here on
        DAB_CUDA(ctx, cudaSetDevice(ctx->device));
        DAB_FLUSH(ctx);
    }
    *launches = ctx->launches;
    return DAB_OK;
}

// ---- events -----------------------------------------------------------------------------
int32_t dab_event_create(dab_ctx* ctx, void** event) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, event, DAB_ERR_ARG, "null event out-pointer");
    cudaEvent_t ev;
    DAB_CUDA(ctx, cudaEventCreate(&ev));
    *event = (void*)ev;
    return DAB_OK;
}
int32_t dab_event_record(dab_ctx* ctx, void* event) {
    DAB_ENTER(ctx);
    DAB_CUDA(ctx, cudaEventRecord((cudaEvent_t)event, ctx->stream));
    return DAB_OK;
}
int32_t dab_event_elapsed_ms(dab_ctx* ctx, void* start, void* stop, float* ms) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, ms, DAB_ERR_ARG, "null ms");
    DAB_CUDA(ctx, cudaEventSynchronize((cudaEvent_t)stop));
    DAB_CUDA(ctx, cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
    return DAB_OK;
}
int32_t dab_event_destroy(dab_ctx* ctx, void* event) {
    DAB_ENTER(ctx);
    DAB_CUDA(ctx, cudaEventDestroy((cudaEvent_t)event));
    return DAB_OK;
}

// ---- buffers ----------------------------------------------------------------------------
int32_t dab_alloc(dab_ctx* ctx, size_t nbytes, void** dptr) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dptr, DAB_ERR_ARG, "null dptr out-pointer");
    *dptr = nullptr;
    if (nbytes == 0) nbytes = 16;  // empty localparts still get a valid, distinct address
    dab_alloc_cache* c = ctx->cache;
    if (c && nbytes <= dab_alloc_cache::kMaxBlock) {
        const size_t rounded = (nbytes + 511) & ~(size_t)511;
        auto it = c->free_blocks.find(rounded);
        if (it != c->free_blocks.end()) {
            *dptr = it->second;
            c->free_blocks.erase(it);
            c->cached_bytes -= rounded;
        } else {
            cudaError_t e = cudaMalloc(dptr, rounded);
            if (e == cudaErrorMemoryAllocation) {   // give the cached blocks back and try again
                cudaGetLastError();
                DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                for (auto& kv : c->free_blocks) cudaFree(kv.second);
                c->free_blocks.clear();
                c->cached_bytes = 0;
                e = cudaMalloc(dptr, rounded);
            }
            DAB_CUDA(ctx, e);
        }
        c->live[*dptr] = rounded;
        return DAB_OK;
    }
    {
        cudaError_t e = cudaMalloc(dptr, nbytes);
        if (e == cudaErrorMemoryAllocation && c) {
            cudaGetLastError();
            DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (auto& kv : c->free_blocks) cudaFree(kv.second);
            c->free_blocks.clear();
            c->cached_bytes = 0;
            e = cudaMalloc(dptr, nbytes);
        }
        DAB_CUDA(ctx, e);
    }
    return DAB_OK;
}
int32_t dab_free(dab_ctx* ctx, void* dptr) {
    DAB_ENTER(ctx);
    if (!dptr) return DAB_OK;
    dab_alloc_cache* c = ctx->cache;
    if (c) {
        auto it = c->live.find(dptr);
        if (it != c->live.end()) {
            const size_t rounded = it->second;
            c->live.erase(it);
            if (c->cached_bytes + rounded <= dab_alloc_cache::kMaxCached) {
                // stream order: work already queued on the ctx stream that still touches the block finishes before any later
                // launch (on the same stream) can be handed the block again
                c->free_blocks.emplace(rounded, dptr);
                c->cached_bytes += rounded;
                return DAB_OK;
            }
        }
    }
    DAB_CUDA(ctx, cudaFree(dptr));
    return DAB_OK;
}
// Stream-ordered temporaries (partial slabs, gather stacks, result slots): cudaMallocAsync from the device's default pool with
// an unlimited release threshold, so steady-state calls cost ~1 us and never synchronise.  NOT exportable over CUDA IPC: chunks
// that peers read must come from dab_alloc.
int32_t dab_alloc_async(dab_ctx* ctx, size_t nbytes, void** dptr) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dptr, DAB_ERR_ARG, "null dptr out-pointer");
    *dptr = nullptr;
    if (nbytes == 0) nbytes = 16;
    DAB_CUDA(ctx, cudaMallocAsync(dptr, nbytes, ctx->stream));
    return DAB_OK;
}
int32_t dab_free_async(dab_ctx* ctx, void* dptr) {
    DAB_ENTER(ctx);
    if (dptr) DAB_CUDA(ctx, cudaFreeAsync(dptr, ctx->stream));
    return DAB_OK;
}
int32_t dab_host_alloc(dab_ctx* ctx, size_t nbytes, void** hptr) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, hptr, DAB_ERR_ARG, "null hptr out-pointer");
    DAB_CUDA(ctx, cudaHostAlloc(hptr, nbytes ? nbytes : 16, cudaHostAllocDefault));
    return DAB_OK;
}
int32_t dab_host_free(dab_ctx* ctx, void* hptr) {
    DAB_ENTER(ctx);
    if (hptr) DAB_CUDA(ctx, cudaFreeHost(hptr));
    return DAB_OK;
}
// distribute(A) / copyto!(d, A) from ORDINARY (pageable) host memory: cudaMemcpyAsync would fall back to the driver's small internal
// bounce buffer and block the calling thread at a fraction of the PCIe rate.  Large pageable sources are therefore pipelined through two
// pinned staging buffers: a few host threads copy block k+1 into one buffer while the copy engine sends block k from the other.  The call
// returns when the last block has been STAGED -- the caller's array may be reused at once, the device side stays asynchronous on the ctx
// stream.  Pinned sources (dab_host_alloc / cudaHostRegister) go straight to cudaMemcpyAsync.
static int32_t h2d_staged(dab_ctx* ctx, char* dptr, const char* hptr, size_t nbytes) {
    constexpr size_t BLOCK = 32ull << 20;
    constexpr int NT = 8;
    if (!ctx->stage[0]) {
        for (int b = 0; b < 2; ++b) {
            DAB_CUDA(ctx, cudaHostAlloc(&ctx->stage[b], BLOCK, cudaHostAllocDefault));
            DAB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_ev[b], cudaEventDisableTiming));
        }
    }
    int b = 0;
    for (size_t off = 0; off < nbytes; off += BLOCK, b ^= 1) {
        const size_t n = nbytes - off < BLOCK ? nbytes - off : BLOCK;
        DAB_CUDA(ctx, cudaEventSynchronize(ctx->stage_ev[b]));          // the copy engine has drained this buffer (no-op the first time)
        char* st = (char*)ctx->stage[b];
        const char* src = hptr + off;
        const size_t per = ((n + NT - 1) / NT + 63) & ~(size_t)63;
        std::thread th[NT];
        int nth = 0;
        for (int t = 1; t < NT && (size_t)t * per < n; ++t, ++nth) {
            const size_t lo = (size_t)t * per, len = lo + per <= n ? per : n - lo;
            th[nth] = std::thread([=] { memcpy(st + lo, src + lo, len); });
        }
        memcpy(st, src, per < n ? per : n);
        for (int t = 0; t < nth; ++t) th[t].join();
        DAB_CUDA(ctx, cudaMemcpyAsync(dptr + off, st, n, cudaMemcpyHostToDevice, ctx->stream));
        DAB_CUDA(ctx, cudaEventRecord(ctx->stage_ev[b], ctx->stream));
    }
    return DAB_OK;
}

int32_t dab_h2d(dab_ctx* ctx, void* dptr, const void* hptr, size_t nbytes) {
    DAB_ENTER(ctx);
    if (!nbytes) return DAB_OK;
    if (nbytes >= (16ull << 20)) {
        cudaPointerAttributes at;
        const cudaError_t e = cudaPointerGetAttributes(&at, hptr);
        if (e != cudaSuccess) cudaGetLastError();
        if (e != cudaSuccess || at.type == cudaMemoryTypeUnregistered) return h2d_staged(ctx, (char*)dptr, (const char*)hptr, nbytes);
    }
    DAB_CUDA(ctx, cudaMemcpyAsync(dptr, hptr, nbytes, cudaMemcpyHostToDevice, ctx->stream));
    return DAB_OK;
}
int32_t dab_d2h(dab_ctx* ctx, void* hptr, const void* dptr, size_t nbytes) {
    DAB_ENTER(ctx);
    if (nbytes) DAB_CUDA(ctx, cudaMemcpyAsync(hptr, dptr, nbytes, cudaMemcpyDeviceToHost, ctx->stream));
    return DAB_OK;
}
int32_t dab_d2d(dab_ctx* ctx, void* dst, const void* src, size_t nbytes) {
    DAB_ENTER(ctx);
    if (nbytes) DAB_CUDA(ctx, cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return DAB_OK;
}
int32_t dab_h2d_2d(dab_ctx* ctx, void* dptr, size_t dpitch, const void* hptr, size_t hpitch, size_t row_bytes, size_t cols) {
    DAB_ENTER(ctx);
    if (row_bytes && cols)
        DAB_CUDA(ctx, cudaMemcpy2DAsync(dptr, dpitch, hptr, hpitch, row_bytes, cols, cudaMemcpyHostToDevice, ctx->stream));
    return DAB_OK;
}
int32_t dab_d2h_2d(dab_ctx* ctx, void* hptr, size_t hpitch, const void* dptr, size_t dpitch, size_t row_bytes, size_t cols) {
    DAB_ENTER(ctx);
    if (row_bytes && cols)
        DAB_CUDA(ctx, cudaMemcpy2DAsync(hptr, hpitch, dptr, dpitch, row_bytes, cols, cudaMemcpyDeviceToHost, ctx->stream));
    return DAB_OK;
}

}  // extern "C"

// ---- fill! / rand! kernels ----------------------------------------------------------------
// Write-only streams: 16-byte stores, grid = 8 CTAs/SM, grid-stride.  Alignment: the head (up to
// 16/sizeof(T)-1 elements) and the tail are written as scalars by the last CTA.
template <typename T, typename Gen>
__global__ void __launch_bounds__(256) dab_generate_kernel(T* __restrict__ x, size_t n, Gen gen) {
    constexpr int VPT = 16 / sizeof(T);
    constexpr int UNROLL = 4;
    size_t head = ((16 - ((uintptr_t)x & 15)) & 15) / sizeof(T);
    if (head > n) head = n;
    const size_t nvec = (n - head) / VPT;
    int4* xv = reinterpret_cast<int4*>(x + head);
    constexpr size_t TILE = 256 * UNROLL;
    const size_t ntiles = nvec / TILE;
    if (blockIdx.x < ntiles) {  // flat grid: one CTA per 16 KiB tile (see ew1_kernel)
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const size_t i = (size_t)blockIdx.x * TILE + (size_t)u * 256 + threadIdx.x;
            Pack<T> p;
#pragma unroll
            for (int k = 0; k < VPT; ++k) p.v[k] = gen(head + i * VPT + k);
            st_stream(xv + i, as_int4(p));
        }
        return;
    }
    for (size_t i = ntiles * TILE + threadIdx.x; i < nvec; i += 256) {
        Pack<T> p;
#pragma unroll
        for (int k = 0; k < VPT; ++k) p.v[k] = gen(head + i * VPT + k);
        st_stream(xv + i, as_int4(p));
    }
    for (size_t i = threadIdx.x; i < head; i += blockDim.x) x[i] = gen(i);
    for (size_t i = head + nvec * VPT + threadIdx.x; i < n; i += blockDim.x) x[i] = gen(i);
}

template <typename T>
struct FillGen {
    T v;
    __device__ __forceinline__ T operator()(size_t) const { return v; }
};
template <typename T>
struct RandGen {
    uint64_t seed, off;
    __device__ __forceinline__ T operator()(size_t i) const {
        return (T)(dab_hash_u32(seed, off + i) >> 8) * (T)5.9604644775390625e-08;  // 2^-24
    }
};

// Julia's rand(Float16): 10 random bits k, the value k * 2^-10 (exact in Float16)
struct RandGenF16 {
    uint64_t seed, off;
    __device__ __forceinline__ Half operator()(size_t i) const {
        return Half((float)(dab_hash_u32(seed, off + i) >> 22) * 0.0009765625f);  // 2^-10
    }
};

template <typename T, typename Gen>
static int32_t launch_generate(dab_ctx* ctx, T* x, size_t n, Gen gen) {
    if (n == 0) return DAB_OK;
    size_t head = ((16 - ((uintptr_t)x & 15)) & 15) / sizeof(T);
    if (head > n) head = n;
    size_t grid = ((n - head) / (16 / sizeof(T))) / 1024 + 1;
    if (grid > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_ARG, "array too large for one launch");
    dab_generate_kernel<T, Gen><<<(unsigned)grid, 256, 0, ctx->stream>>>(x, n, gen);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

extern "C" {

int32_t dab_fill(dab_ctx* ctx, int32_t dtype, void* x, size_t n, const void* value) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, (x || n == 0) && value, DAB_ERR_ARG, "dab_fill: null pointer");
    switch (dtype) {
        case DAB_F32: return launch_generate(ctx, (float*)x, n, FillGen<float>{*(const float*)value});
        case DAB_F64: return launch_generate(ctx, (double*)x, n, FillGen<double>{*(const double*)value});
        case DAB_I32: return launch_generate(ctx, (int32_t*)x, n, FillGen<int32_t>{*(const int32_t*)value});
        case DAB_I64: return launch_generate(ctx, (long long*)x, n, FillGen<long long>{*(const long long*)value});
        case DAB_U8: return launch_generate(ctx, (uint8_t*)x, n, FillGen<uint8_t>{*(const uint8_t*)value});
        case DAB_F16: {
            DAB_REQUIRE(ctx, (uintptr_t)x % 2 == 0, DAB_ERR_ARG, "dab_fill: Float16 data needs 2-byte alignment");
            FillGen<Half> g;
            memcpy(&g.v, value, 2);
            return launch_generate(ctx, (Half*)x, n, g);
        }
        case DAB_C64:
        case DAB_C128: {  // interleaved (re, im): one element is 8 / 16 bytes, stored with the same 16-byte vectors
            const size_t es = dab_dtype_size(dtype);
            DAB_REQUIRE(ctx, (uintptr_t)x % es == 0, DAB_ERR_ARG, "dab_fill: complex dtype %d needs %d-byte aligned data", dtype, (int)es);
            if (dtype == DAB_C64) {
                FillGen<Cplx<float>> g;
                memcpy(&g.v, value, 8);
                return launch_generate(ctx, (Cplx<float>*)x, n, g);
            }
            FillGen<Cplx<double>> g;
            memcpy(&g.v, value, 16);
            return launch_generate(ctx, (Cplx<double>*)x, n, g);
        }
        default: return dab_fail(ctx, DAB_ERR_ARG, "dab_fill: bad dtype %d", dtype);
    }
}

int32_t dab_rand_u01(dab_ctx* ctx, int32_t dtype, void* x, size_t n, uint64_t seed, uint64_t global_offset) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, x || n == 0, DAB_ERR_ARG, "dab_rand_u01: null pointer");
    switch (dtype) {
        case DAB_F32: return launch_generate(ctx, (float*)x, n, RandGen<float>{seed, global_offset});
        case DAB_F64: return launch_generate(ctx, (double*)x, n, RandGen<double>{seed, global_offset});
        case DAB_F16:
            DAB_REQUIRE(ctx, (uintptr_t)x % 2 == 0, DAB_ERR_ARG, "dab_rand_u01: Float16 data needs 2-byte alignment");
            return launch_generate(ctx, (Half*)x, n, RandGenF16{seed, global_offset});
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_rand_u01: dtype %d (F32/F64/F16 only)", dtype);
    }
}

}  // extern "C"
