// dab_scatter.cu -- K24: d[I[k]] = v[k], the scatter behind  d[I::DArray{<:Integer}] = v  (row f14), the inverse of K22.
//
// Replaces Base's generic setindex!(A, v, I::AbstractArray) on a DArray, which writes one element per remote call.  Julia's setindex!
// is sequential: it checks every index before the first store, and a position repeated in I keeps the value of its LAST occurrence in
// column-major order of I.  One call of each entry point serves one block of I (one chunk); the destination d is described by K22's
// table (dims, per-dimension cuts, one pointer per chunk, local or a CUDA-IPC peer mapping) in a __grid_constant__ parameter block,
// which each CTA copies to shared memory.  The host runs, over all blocks of I:
//
//   dab_scatter_check    bounds and duplicates: atomicMin of the first bad position; one bit per destination element in a per-chunk
//                        bitmap (atomicOr, a peer atomic for another GPU's chunk), a bit already set raises the duplicates flag
//   (host)               combines the flags of every rank; a bad index raises BoundsError here, before d is touched
//   dab_scatter_winners  only with duplicates: atomicMax of the 1-based global position in I into a per-element winner table
//   dab_scatter          the stores: d[I[k]] = v[k] (or the scalar); with a winner table only the position that won stores
//
// With unique indices (permutations, findall results) the cost over a plain scatter is one more read of I and the bitmap atomics, whose
// bitmap is 1/32 of a Float32 d and stays in L2.  Values move as bytes (1, 4, 8, 16), so NaN payloads and -0.0 are kept.  64-bit
// indexing throughout.
#include "dab_take_core.cuh"

namespace {

constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 8;                       // indices per thread, all loads issued before the first atomic or store
constexpr int SC_TILE = SC_THREADS * SC_ITEMS;

struct ScatterAux {
    char* ptrs[TK_MAX_CHUNKS];                    // the winner table of each destination chunk (column-major grid order)
};

// Table cuts and the chunk pointers into shared memory; returns the pointer table.
__device__ __forceinline__ char** sc_stage(const TakeSrc& t, unsigned long long* smem) {
    char** ptrs = reinterpret_cast<char**>(smem + t.ncuts);
    for (int i = threadIdx.x; i < t.ncuts; i += SC_THREADS) smem[i] = t.cuts[i];
    for (int i = threadIdx.x; i < t.nchunks; i += SC_THREADS) ptrs[i] = const_cast<char*>(t.chunks[i]);
    return ptrs;
}

// The 0-based global column-major position in I of block element k: the block is a chunk of I, a stack of runs of run_len elements
// that are each contiguous in I's global order and start at run_lin[r].
__device__ __forceinline__ unsigned long long sc_position(unsigned long long k, unsigned long long run_len, unsigned long long run_inv,
                                                          const long long* __restrict__ run_lin) {
    unsigned long long x = k;
    const unsigned long long r = tk_divmod(x, run_len, run_inv);
    return (unsigned long long)run_lin[r] + x;
}

template <typename IDX>
__device__ __forceinline__ void sc_load_indices(const IDX* __restrict__ idx, unsigned long long n, unsigned long long tile,
                                                unsigned long long (&g)[SC_ITEMS]) {
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u) {
        const unsigned long long k = tile + (unsigned long long)u * SC_THREADS + threadIdx.x;
        g[u] = k < n ? (unsigned long long)(long long)idx[k] - 1ull : ~0ull;   // Int32 widened before the subtraction
    }
}

template <typename IDX, bool ND>
__global__ void __launch_bounds__(SC_THREADS) scatter_check_kernel(const IDX* __restrict__ idx, unsigned long long n,
                                                                   const __grid_constant__ TakeSrc bm, unsigned long long* __restrict__ status) {
    extern __shared__ unsigned long long sc_smem[];
    char** bits = sc_stage(bm, sc_smem);
    __syncthreads();
    const unsigned long long tile = (unsigned long long)blockIdx.x * SC_TILE;
    unsigned long long g[SC_ITEMS];
    sc_load_indices(idx, n, tile, g);
    unsigned long long bad = ~0ull;
    unsigned* word[SC_ITEMS];
    unsigned bit[SC_ITEMS];
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u) {
        const unsigned long long k = tile + (unsigned long long)u * SC_THREADS + threadIdx.x;
        word[u] = nullptr;
        bit[u] = 0;
        if (k >= n) continue;
        if (g[u] >= bm.len) {
            bad = min(bad, k);
            continue;
        }
        unsigned long long off;
        const int c = tk_locate<ND>(bm, sc_smem, g[u], off);
        word[u] = reinterpret_cast<unsigned*>(bits[c]) + (off >> 5);
        bit[u] = 1u << (off & 31);
    }
    // one atomicOr per distinct bitmap word in the warp when neighbouring lanes share words (consecutive indices would otherwise serialise
    // 32 atomics on one word); two lanes with the same bit are a duplicate too.  The warp collectives all come first, so that the atomics
    // are issued back to back.
    unsigned dup = 0;
    const int lane = threadIdx.x & 31;
    unsigned lead = 0;
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u) {
        const unsigned* left = reinterpret_cast<const unsigned*>(
            __shfl_up_sync(0xffffffffu, reinterpret_cast<unsigned long long>(word[u]), 1));
        if (!__any_sync(0xffffffffu, lane > 0 && word[u] && word[u] == left)) {   // no shared words (random indices): no aggregation
            lead |= word[u] ? 1u << u : 0u;
            continue;
        }
        const unsigned peers = __match_any_sync(0xffffffffu, (unsigned long long)word[u]);
        const unsigned bits_or = __reduce_or_sync(peers, bit[u]);
        if (word[u] && lane == __ffs(peers) - 1) {
            lead |= 1u << u;
            dup |= __popc(bits_or) != __popc(peers);
        }
        bit[u] = bits_or;
    }
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u)
        if (lead & (1u << u)) dup |= atomicOr(word[u], bit[u]) & bit[u];
    if (bad != ~0ull) atomicMin(status, bad);
    if (dup) atomicOr(status + 1, 1ull);
}

template <typename IDX, bool ND, typename W>
__global__ void __launch_bounds__(SC_THREADS) scatter_winners_kernel(const IDX* __restrict__ idx, unsigned long long n, unsigned long long run_len,
                                                                     unsigned long long run_inv, const long long* __restrict__ run_lin,
                                                                     const __grid_constant__ TakeSrc win) {
    extern __shared__ unsigned long long sc_smem[];
    char** tab = sc_stage(win, sc_smem);
    __syncthreads();
    const unsigned long long tile = (unsigned long long)blockIdx.x * SC_TILE;
    unsigned long long g[SC_ITEMS];
    sc_load_indices(idx, n, tile, g);
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u) {
        const unsigned long long k = tile + (unsigned long long)u * SC_THREADS + threadIdx.x;
        if (k >= n || g[u] >= win.len) continue;
        unsigned long long off;
        const int c = tk_locate<ND>(win, sc_smem, g[u], off);
        atomicMax(reinterpret_cast<W*>(tab[c]) + off, (W)(sc_position(k, run_len, run_inv, run_lin) + 1));
    }
}

// win_bytes 0: every index stores (they are unique); 4 / 8: only the position whose 1-based global position is in the winner table.
// src == NULL: the scalar.
template <typename U, typename IDX, bool ND>
__global__ void __launch_bounds__(SC_THREADS) scatter_kernel(const IDX* __restrict__ idx, unsigned long long n, const U* __restrict__ src, U scalar,
                                                             unsigned long long run_len, unsigned long long run_inv,
                                                             const long long* __restrict__ run_lin, int win_bytes,
                                                             const __grid_constant__ TakeSrc dst, const __grid_constant__ ScatterAux win) {
    extern __shared__ unsigned long long sc_smem[];
    char** out = sc_stage(dst, sc_smem);
    char** wtab = out + dst.nchunks;
    if (win_bytes)
        for (int i = threadIdx.x; i < dst.nchunks; i += SC_THREADS) wtab[i] = win.ptrs[i];
    __syncthreads();
    const unsigned long long tile = (unsigned long long)blockIdx.x * SC_TILE;
    unsigned long long g[SC_ITEMS];
    sc_load_indices(idx, n, tile, g);
#pragma unroll
    for (int u = 0; u < SC_ITEMS; ++u) {
        const unsigned long long k = tile + (unsigned long long)u * SC_THREADS + threadIdx.x;
        if (k >= n || g[u] >= dst.len) continue;
        unsigned long long off;
        const int c = tk_locate<ND>(dst, sc_smem, g[u], off);
        if (win_bytes) {
            const unsigned long long p = sc_position(k, run_len, run_inv, run_lin) + 1;
            const unsigned long long w = win_bytes == 4 ? (unsigned long long)reinterpret_cast<const unsigned*>(wtab[c])[off]
                                                        : reinterpret_cast<const unsigned long long*>(wtab[c])[off];
            if (w != p) continue;
        }
        reinterpret_cast<U*>(out[c])[off] = src ? src[k] : scalar;
    }
}

int32_t sc_blocks(dab_ctx* ctx, const char* name, size_t n, unsigned* blocks) {
    const unsigned long long b = (n + SC_TILE - 1) / SC_TILE;
    if (b > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "%s: %zu indices exceed one launch", name, n);
    *blocks = (unsigned)b;
    return DAB_OK;
}

int32_t sc_check_idx(dab_ctx* ctx, const char* name, const void* idx, int32_t idx_dtype) {
    DAB_REQUIRE(ctx, idx_dtype == DAB_I32 || idx_dtype == DAB_I64, DAB_ERR_ARG, "%s: index dtype %d (served: I32, I64)", name, idx_dtype);
    DAB_REQUIRE(ctx, idx && (uintptr_t)idx % (idx_dtype == DAB_I32 ? 4 : 8) == 0, DAB_ERR_ARG, "%s: null or misaligned index block", name);
    return DAB_OK;
}

int32_t sc_check_runs(dab_ctx* ctx, const char* name, size_t run_len, const int64_t* run_lin) {
    DAB_REQUIRE(ctx, run_len >= 1 && run_lin && (uintptr_t)run_lin % 8 == 0, DAB_ERR_ARG, "%s: null or misaligned run table", name);
    return DAB_OK;
}

template <typename IDX, bool ND>
int32_t launch_check(dab_ctx* ctx, const void* idx, size_t n, unsigned blocks, const TakeSrc& s, unsigned long long* status) {
    const size_t smem = (size_t)s.ncuts * 8 + (size_t)s.nchunks * sizeof(void*);
    scatter_check_kernel<IDX, ND><<<blocks, SC_THREADS, smem, ctx->stream>>>((const IDX*)idx, n, s, status);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename IDX, bool ND, typename W>
int32_t launch_winners(dab_ctx* ctx, const void* idx, size_t n, unsigned blocks, size_t run_len, const int64_t* run_lin, const TakeSrc& s) {
    const size_t smem = (size_t)s.ncuts * 8 + (size_t)s.nchunks * sizeof(void*);
    scatter_winners_kernel<IDX, ND, W><<<blocks, SC_THREADS, smem, ctx->stream>>>((const IDX*)idx, n, run_len, ~0ull / run_len,
                                                                                  (const long long*)run_lin, s);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename U, typename IDX, bool ND>
int32_t launch_scatter(dab_ctx* ctx, const void* idx, size_t n, unsigned blocks, const void* src, const void* scalar, size_t run_len,
                       const int64_t* run_lin, int32_t win_bytes, const TakeSrc& s, const ScatterAux& w) {
    U sv;
    memset(&sv, 0, sizeof(sv));
    if (!src) memcpy(&sv, scalar, sizeof(U));
    const size_t smem = (size_t)s.ncuts * 8 + (size_t)s.nchunks * sizeof(void*) * (win_bytes ? 2 : 1);
    scatter_kernel<U, IDX, ND><<<blocks, SC_THREADS, smem, ctx->stream>>>((const IDX*)idx, n, (const U*)src, sv, run_len,
                                                                          win_bytes ? ~0ull / run_len : 0, (const long long*)run_lin, win_bytes, s, w);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename U, typename IDX>
int32_t scatter_nd(dab_ctx* ctx, const void* idx, size_t n, unsigned blocks, const void* src, const void* scalar, size_t run_len,
                   const int64_t* run_lin, int32_t win_bytes, const TakeSrc& s, const ScatterAux& w) {
    if (s.ndim == 1) return launch_scatter<U, IDX, false>(ctx, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
    return launch_scatter<U, IDX, true>(ctx, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
}

template <typename U>
int32_t scatter_idx(dab_ctx* ctx, int32_t idx_dtype, const void* idx, size_t n, unsigned blocks, const void* src, const void* scalar,
                    size_t run_len, const int64_t* run_lin, int32_t win_bytes, const TakeSrc& s, const ScatterAux& w) {
    if (idx_dtype == DAB_I32) return scatter_nd<U, int32_t>(ctx, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
    return scatter_nd<U, long long>(ctx, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
}

}  // namespace

extern "C" {

int32_t dab_scatter_check(dab_ctx* ctx, const void* idx, int32_t idx_dtype, size_t n, int32_t ndim, const size_t* dims, const int32_t* grid,
                          const size_t* cuts, void* const* bitmap_ptrs, unsigned long long* status) {
    DAB_ENTER(ctx);
    const char* name = "dab_scatter_check";
    TakeSrc s;
    int32_t st = tk_fill_src(ctx, name, ndim, dims, grid, cuts, bitmap_ptrs, 4, &s);
    if (st != DAB_OK || n == 0) return st;
    if ((st = sc_check_idx(ctx, name, idx, idx_dtype)) != DAB_OK) return st;
    DAB_REQUIRE(ctx, status && (uintptr_t)status % 8 == 0, DAB_ERR_ARG, "%s: null or misaligned status", name);
    unsigned blocks = 0;
    if ((st = sc_blocks(ctx, name, n, &blocks)) != DAB_OK) return st;
    if (idx_dtype == DAB_I32)
        return ndim == 1 ? launch_check<int32_t, false>(ctx, idx, n, blocks, s, status) : launch_check<int32_t, true>(ctx, idx, n, blocks, s, status);
    return ndim == 1 ? launch_check<long long, false>(ctx, idx, n, blocks, s, status) : launch_check<long long, true>(ctx, idx, n, blocks, s, status);
}

int32_t dab_scatter_winners(dab_ctx* ctx, const void* idx, int32_t idx_dtype, size_t n, size_t run_len, const int64_t* run_lin, int32_t win_bytes,
                            int32_t ndim, const size_t* dims, const int32_t* grid, const size_t* cuts, void* const* win_ptrs) {
    DAB_ENTER(ctx);
    const char* name = "dab_scatter_winners";
    DAB_REQUIRE(ctx, win_bytes == 4 || win_bytes == 8, DAB_ERR_ARG, "%s: win_bytes %d (served: 4, 8)", name, win_bytes);
    TakeSrc s;
    int32_t st = tk_fill_src(ctx, name, ndim, dims, grid, cuts, win_ptrs, (size_t)win_bytes, &s);
    if (st != DAB_OK || n == 0) return st;
    if ((st = sc_check_idx(ctx, name, idx, idx_dtype)) != DAB_OK) return st;
    if ((st = sc_check_runs(ctx, name, run_len, run_lin)) != DAB_OK) return st;
    unsigned blocks = 0;
    if ((st = sc_blocks(ctx, name, n, &blocks)) != DAB_OK) return st;
    const bool nd = ndim > 1, i32 = idx_dtype == DAB_I32;
    if (win_bytes == 4) {
        using W = unsigned;
        if (i32) return nd ? launch_winners<int32_t, true, W>(ctx, idx, n, blocks, run_len, run_lin, s) : launch_winners<int32_t, false, W>(ctx, idx, n, blocks, run_len, run_lin, s);
        return nd ? launch_winners<long long, true, W>(ctx, idx, n, blocks, run_len, run_lin, s) : launch_winners<long long, false, W>(ctx, idx, n, blocks, run_len, run_lin, s);
    }
    using W = unsigned long long;
    if (i32) return nd ? launch_winners<int32_t, true, W>(ctx, idx, n, blocks, run_len, run_lin, s) : launch_winners<int32_t, false, W>(ctx, idx, n, blocks, run_len, run_lin, s);
    return nd ? launch_winners<long long, true, W>(ctx, idx, n, blocks, run_len, run_lin, s) : launch_winners<long long, false, W>(ctx, idx, n, blocks, run_len, run_lin, s);
}

int32_t dab_scatter(dab_ctx* ctx, int32_t elem_bytes, const void* idx, int32_t idx_dtype, size_t n, const void* src, const void* scalar,
                    size_t run_len, const int64_t* run_lin, int32_t win_bytes, int32_t ndim, const size_t* dims, const int32_t* grid,
                    const size_t* cuts, void* const* chunk_ptrs, void* const* win_ptrs) {
    DAB_ENTER(ctx);
    const char* name = "dab_scatter";
    DAB_REQUIRE(ctx, elem_bytes == 1 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "%s: elem_bytes %d (served: 1, 4, 8, 16)", name, elem_bytes);
    DAB_REQUIRE(ctx, win_bytes == 0 || win_bytes == 4 || win_bytes == 8, DAB_ERR_ARG, "%s: win_bytes %d (served: 0, 4, 8)", name, win_bytes);
    TakeSrc s;
    int32_t st = tk_fill_src(ctx, name, ndim, dims, grid, cuts, chunk_ptrs, (size_t)elem_bytes, &s);
    if (st != DAB_OK) return st;
    ScatterAux w;
    memset(&w, 0, sizeof(w));
    if (win_bytes) {
        TakeSrc ws;                                   // the winner tables have the destination's cuts: the same checks, win_bytes alignment
        if ((st = tk_fill_src(ctx, name, ndim, dims, grid, cuts, win_ptrs, (size_t)win_bytes, &ws)) != DAB_OK) return st;
        for (int c = 0; c < ws.nchunks; ++c) w.ptrs[c] = const_cast<char*>(ws.chunks[c]);
    }
    if (n == 0) return DAB_OK;
    if ((st = sc_check_idx(ctx, name, idx, idx_dtype)) != DAB_OK) return st;
    DAB_REQUIRE(ctx, src ? (uintptr_t)src % elem_bytes == 0 : scalar != nullptr, DAB_ERR_ARG, "%s: misaligned values or no scalar", name);
    if (win_bytes && (st = sc_check_runs(ctx, name, run_len, run_lin)) != DAB_OK) return st;
    unsigned blocks = 0;
    if ((st = sc_blocks(ctx, name, n, &blocks)) != DAB_OK) return st;
    switch (elem_bytes) {
        case 1: return scatter_idx<uint8_t>(ctx, idx_dtype, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
        case 4: return scatter_idx<uint32_t>(ctx, idx_dtype, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
        case 8: return scatter_idx<unsigned long long>(ctx, idx_dtype, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
        default: return scatter_idx<int4>(ctx, idx_dtype, idx, n, blocks, src, scalar, run_len, run_lin, win_bytes, s, w);
    }
}

}  // extern "C"
