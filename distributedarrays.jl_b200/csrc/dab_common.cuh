// dab_common.cuh -- shared internals of libdab200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../include/dab200.h"

#define DAB_MAX_REDUCE_BLOCKS 262144
#define DAB_SLOT_BYTES 64
#define DAB_MAX_RANKS 64

// A dab_affine call whose kernel has not been launched yet (dab_elementwise.cu).  y .= a.*x .+ b is usually followed by a
// reduction of y (sum(y), map!(f, d, d); sum(d)); the reduce kernel can then compute y itself while it streams x and skip
// re-reading 4 GiB of y from HBM.  The record holds copies of a and b, not the caller's pointers.
struct dab_pending_affine {
    int active;
    int32_t dtype;
    void* y;
    const void* x;
    size_t n;
    unsigned char a[8], b[8];
};

struct dab_ctx {
    int device;
    int sm_count;
    cudaStream_t stream;
    // reduction scratch (device)
    void* block_partials;   // DAB_MAX_REDUCE_BLOCKS * 16 bytes
    unsigned int* counter;  // single ticket counter, self-resetting
    void* result_slot;      // DAB_SLOT_BYTES: result of dab_reduce_host / dab_mapreduce_all
    void* gather_slots;     // DAB_MAX_RANKS * 8 bytes
    void* host_slot;        // pinned, DAB_MAX_RANKS * 8 bytes
    void* dim_scratch;      // scratch for split reducedim partials
    size_t dim_scratch_bytes;
    uint64_t launches;
    // NCCL
    void* comm;
    int rank, nranks;
    // fused reduce + all-gather + ordered fold over peer memory (dab_mailbox_*; dab_reduce.cu)
    void* mailbox;          // this rank's mailbox (device, cudaMalloc'ed, IPC-exported)
    void** peer_mbox_dev;   // device array [nranks] of mailbox addresses as mapped in THIS process
    void* peer_mbox_host[DAB_MAX_RANKS];
    int mbox_ranks;         // 0 = not attached
    unsigned long long mbox_seq;
    unsigned long long barrier_seq;   // dab_peer_barrier: how many device-side barriers this rank has entered
    int fuse_op;            // >= 0: the next launch_reduce appends the cross-rank combine for this DAB_* op
    struct dab_alloc_cache* cache;  // size-bucketed reuse of small cudaMalloc blocks (dab_core.cu)
    void* sort_dev;         // radix-sort scratch: digit histograms + per-tile counts (dab_sort.cu)
    size_t sort_dev_bytes;
    void* stage[2];         // pinned staging buffers of the pipelined pageable H2D path (dab_h2d)
    cudaEvent_t stage_ev[2];
    void* sort_host;        // pinned: split-point staging of dab_sorted_split
    unsigned long long sort_epoch;  // one per digit pass ever launched: tags the look-back words so the scratch is never re-cleared
    void* scan_dev;         // scan: tile ticket counter + look-back words (dab_scan.cu), zeroed once per allocation
    size_t scan_dev_bytes;
    unsigned long long scan_epoch;    // one per flat scan launch: tags its look-back words
    unsigned long long scan_tickets;  // tickets drawn so far from the counter in scan_dev
    void* scan_scratch;     // scan: segment totals of the split strided path
    size_t scan_scratch_bytes;
    long long opt_combine_timeout_ms;  // dab_set_option("combine_timeout_ms"): how long the fused combine waits for a peer (default 120 s)
    int opt_ew_tma;         // dab_set_option("ew_tma"): route aligned unary elementwise launches through the TMA-staged kernel
    dab_pending_affine pending;  // at most one deferred dab_affine; launched by the next entry or consumed by dab_reduce
    int defer_off;          // set by dab_stream: foreign work on the raw stream expects every call to be queued already
    char err[512];
};

extern thread_local char dab_tls_err[512];

int32_t dab_fail(dab_ctx* ctx, int32_t status, const char* fmt, ...);
int32_t dab_fail_cuda(dab_ctx* ctx, cudaError_t e, const char* what, const char* file, int line);

#define DAB_CUDA(ctx, call)                                                             \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess) return dab_fail_cuda((ctx), e__, #call, __FILE__, __LINE__); \
    } while (0)

#define DAB_REQUIRE(ctx, cond, status, ...)                          \
    do {                                                             \
        if (!(cond)) return dab_fail((ctx), (status), __VA_ARGS__);  \
    } while (0)

// Launches the deferred dab_affine kernel, if any (dab_elementwise.cu).  The slot is cleared first; a launch error is
// returned with text naming dab_affine.
int32_t dab_flush_pending(dab_ctx* ctx);

#define DAB_FLUSH(ctx)                                    \
    do {                                                  \
        if ((ctx)->pending.active) {                      \
            int32_t st__ = dab_flush_pending(ctx);        \
            if (st__ != DAB_OK) return st__;              \
        }                                                 \
    } while (0)

// Every entry point starts with DAB_ENTER, which first queues a deferred dab_affine: work is issued in call order.
#define DAB_ENTER(ctx)                                                      \
    do {                                                                    \
        if ((ctx) == nullptr) return dab_fail(nullptr, DAB_ERR_ARG, "null ctx"); \
        DAB_CUDA((ctx), cudaSetDevice((ctx)->device));                      \
        DAB_FLUSH(ctx);                                                     \
    } while (0)

// dab_reduce, dab_reduce_host and dab_mapreduce_all only: dab_reduce either consumes the deferred dab_affine or flushes it.
#define DAB_ENTER_NOFLUSH(ctx)                                              \
    do {                                                                    \
        if ((ctx) == nullptr) return dab_fail(nullptr, DAB_ERR_ARG, "null ctx"); \
        DAB_CUDA((ctx), cudaSetDevice((ctx)->device));                      \
    } while (0)

// after a kernel launch
#define DAB_LAUNCHED(ctx)                          \
    do {                                           \
        (ctx)->launches++;                         \
        DAB_CUDA((ctx), cudaGetLastError());       \
    } while (0)

// Grow-on-demand device scratch owned by the ctx (*buf of *have bytes): returns at once when it holds `bytes`; otherwise waits for
// the stream (earlier launches may still use the old buffer), frees it, allocates `bytes` and, with `zero`, clears the new buffer
// in stream order.  ctx->dim_scratch is shared by the split partials of dab_reducedim, dab_findminmax_dim and dab_gemv: one
// stream, so never two launches' partials at once.
int32_t dab_scratch_grow(dab_ctx* ctx, void** buf, size_t* have, size_t bytes, bool zero);

static inline size_t dab_dtype_size(int32_t dt) {
    switch (dt) {
        case DAB_F32: return 4;
        case DAB_F64: return 8;
        case DAB_I32: return 4;
        case DAB_I64: return 8;
        case DAB_U8: return 1;
        case DAB_C64: return 8;
        case DAB_C128: return 16;
        case DAB_F16: return 2;
        default: return 0;
    }
}

// Cross-rank combine fused into the reduce kernel's last CTA (see reduce_kernel): nranks == 0 disables it.
#define DAB_MBOX_SLOT 32                                   /* [0,8) result  [8,16) wide carrier  [16,24) sequence flag */
#define DAB_MBOX_BARRIER_OFFSET (2 * DAB_MAX_RANKS * DAB_MBOX_SLOT) /* after the two parity banks: one 8-byte arrival counter per rank (dab_peer_barrier) */
#define DAB_MBOX_BYTES (DAB_MBOX_BARRIER_OFFSET + DAB_MAX_RANKS * 8)
struct FusedComm {
    void* const* peers;        // device array of the nranks mailboxes
    void* host_out;            // pinned host slot: [0,8) folded result, [8,16) status (0 ok, 1 timed out)
    unsigned long long seq;
    unsigned long long timeout_ns;   // wall-clock bound of the mailbox poll (%globaltimer), dab_set_option("combine_timeout_ms")
    int rank, nranks, op;
};

// ---- device helpers --------------------------------------------------------------------
__device__ __forceinline__ unsigned long long dab_globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// 16-byte streaming load/store (evict-first: every element of the hot path is touched once).
__device__ __forceinline__ int4 ld_stream(const int4* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(int4* p, int4 v) { __stcs(p, v); }

template <typename T>
struct alignas(16) Pack {
    static constexpr int N = 16 / sizeof(T);
    T v[N];
};

// Complex{T} element: interleaved (re, im), aligned to its size so that one 16-byte vector carries whole elements.
template <typename T>
struct alignas(2 * sizeof(T)) Cplx {
    T re, im;
};

// Float16 element: the IEEE binary16 bits.  Conversions are single PTX cvt instructions: widening is exact, narrowing rounds once to
// nearest even (from Float64 directly, never through Float32) and overflows to +-Inf.
struct alignas(2) Half {
    unsigned short bits;
    Half() = default;
    __device__ __forceinline__ explicit Half(float v) { asm("cvt.rn.f16.f32 %0, %1;" : "=h"(bits) : "f"(v)); }
    __device__ __forceinline__ explicit Half(double v) { asm("cvt.rn.f16.f64 %0, %1;" : "=h"(bits) : "d"(v)); }
    __device__ __forceinline__ explicit Half(int v) : Half((float)v) {}  // 0 / 1 of the ALL / ANY finalisation
    __device__ __forceinline__ explicit operator float() const {
        float f;
        asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(bits));
        return f;
    }
    __device__ __forceinline__ explicit operator double() const {
        double d;
        asm("cvt.f64.f16 %0, %1;" : "=d"(d) : "h"(bits));
        return d;
    }
};
// Host-side Float16 <-> Float32 on the same bit representation (dab_combine_ordered's fold): widening is exact (a NaN keeps its payload);
// narrowing rounds to nearest even, overflows to +-Inf at 65520 and keeps the top payload bits of a NaN (quieted).
static inline float dab_half_to_float(unsigned short h) {
    const uint32_t sign = (uint32_t)(h & 0x8000) << 16, e = (h >> 10) & 0x1f, m = h & 0x3ff;
    uint32_t x;
    if (e == 0x1f) x = sign | 0x7f800000u | (m << 13);
    else if (e) x = sign | ((e + 112) << 23) | (m << 13);
    else {
        const float v = (float)m * 5.9604644775390625e-08f;  // m * 2^-24, exact
        memcpy(&x, &v, 4);
        x |= sign;
    }
    float f;
    memcpy(&f, &x, 4);
    return f;
}
static inline unsigned short dab_float_to_half(float f) {
    uint32_t x;
    memcpy(&x, &f, 4);
    const uint32_t sign = (x >> 16) & 0x8000, ax = x & 0x7fffffffu;
    if (ax > 0x7f800000u) return (unsigned short)(sign | 0x7e00 | ((ax >> 13) & 0x3ff));
    if (ax >= 0x477ff000u) return (unsigned short)(sign | 0x7c00);  // |f| >= 65520 (and Inf)
    uint32_t q, rem, half;
    if (ax < 0x38800000u) {                                          // below 2^-14: a subnormal Float16 (or zero)
        const uint32_t e = ax >> 23;
        if (e < 102) return (unsigned short)sign;                    // below 2^-25
        const uint32_t m = (ax & 0x7fffffu) | 0x800000u, shift = 126 - e;
        q = m >> shift;
        rem = m & ((1u << shift) - 1);
        half = 1u << (shift - 1);
    } else {
        const uint32_t r = ax - 0x38000000u;                         // rebias the exponent from 127 to 15
        q = r >> 13;
        rem = r & 0x1fff;
        half = 0x1000;
    }
    if (rem > half || (rem == half && (q & 1))) ++q;
    return (unsigned short)(sign | q);
}
// evict-first scalar load of a Float16 element (the strided dims kernels read single elements)
__device__ __forceinline__ Half __ldcs(const Half* p) {
    Half h;
    h.bits = __ldcs(reinterpret_cast<const unsigned short*>(p));
    return h;
}

template <typename T>
__device__ __forceinline__ Pack<T> as_pack(int4 r) {
    Pack<T> p;
    memcpy(&p, &r, 16);
    return p;
}
template <typename T>
__device__ __forceinline__ int4 as_int4(const Pack<T>& p) {
    int4 r;
    memcpy(&r, &p, 16);
    return r;
}

// counter-based RNG shared bit-for-bit with oracle/oracle_core.c (hash_u32)
__host__ __device__ __forceinline__ uint32_t dab_hash_u32(uint64_t seed, uint64_t idx) {
    uint64_t z = idx + (seed + 1ull) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (uint32_t)(z >> 32);
}

static inline int dab_grid_for(const dab_ctx* ctx, size_t work_items, int per_sm) {
    size_t cap = (size_t)ctx->sm_count * (size_t)per_sm;
    size_t g = work_items < cap ? work_items : cap;
    return (int)(g < 1 ? 1 : g);
}

// resident CTAs per SM of `kernel` at `threads` threads (cached per kernel): persistent grids are sized to exactly one
// wave (sm_count x resident CTAs) so that the grid-stride loops have no partial second wave.
int dab_resident_ctas(const void* kernel, int threads);

template <typename K>
static inline int dab_persistent_grid(const dab_ctx* ctx, K kernel, int threads, size_t work_items) {
    return dab_grid_for(ctx, work_items, dab_resident_ctas((const void*)kernel, threads));
}
