// dab_expand.cu -- K25: d[mask::DArray{Bool}] = v  (row f14), the inverse of K23's compaction (dab_compact.cu).
//
// Replaces Base's generic setindex!(A, v, I::AbstractArray{Bool}) on a DArray, which writes one element per remote call.  The chunk is
// K23's (tiles_per_run x runs) table of CP_TILE-element tiles, planned exactly as for d[mask] (dab_compact_count, the K17 scans of the
// tile table, the host's run offsets): the element at run position i of run r that is the p-th true of its run takes
// v[run_info[2r] + p].  Each CTA ranks its tile's flags with a CTA-local scan, lists the positions of its selected elements in rank
// order, and reads their values from the contiguous segment [run offset + tile offset, + tile count) of v -- consecutive threads on
// consecutive positions, through v's cuts-plus-pointers table (local or CUDA-IPC peer mappings) -- storing each into the chunk.  The
// scalar mode (d[mask] = x) needs no plan.  Values move as bytes (1, 4, 8 or 16), so NaN payloads and -0.0 are kept; 64-bit indexing.
#include "dab_compact_core.cuh"

namespace {

// K25 scalar mode: every selected element of the chunk takes `scalar` (no plan, no table).  Thread t visits tile elements t, t + 256, ...
// so that the mask loads and the stores of a warp are contiguous.
template <typename U>
__global__ void __launch_bounds__(CP_THREADS) expand_fill_kernel(const uint8_t* __restrict__ mask, U* __restrict__ dst, unsigned long long run_len,
                                                                 unsigned tpr, U scalar) {
    unsigned r, t;
    unsigned long long base;
    int len;
    cp_tile(run_len, tpr, r, t, base, len);
#pragma unroll
    for (int j = 0; j < CP_ITEMS; ++j) {
        const int i = j * CP_THREADS + threadIdx.x;
        if (i < len && mask[base + i]) dst[base + i] = scalar;
    }
}

// K25, the inverse of compact_kernel: the element at run position i of run r that is the p-th true of its run takes
// src[run_info[2r] + p], read through the source table (local or a CUDA-IPC peer mapping), and is stored into the chunk dst.
template <typename U>
__global__ void __launch_bounds__(CP_THREADS) expand_kernel(const uint8_t* __restrict__ mask, U* dst, unsigned long long run_len,
                                                            unsigned tpr, const long long* __restrict__ tile_incl,
                                                            const long long* __restrict__ run_info, const __grid_constant__ CompactDst src) {
    __shared__ unsigned short pos[CP_TILE];
    __shared__ int warp_tot[CP_WARPS];
    unsigned r, t;
    unsigned long long base;
    int len;
    cp_tile(run_len, tpr, r, t, base, len);
    const unsigned bits = cp_flags(mask, base, len);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c = __popc(bits);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < CP_WARPS; ++w) {
        const int v = warp_tot[w];
        before += w < warp ? v : 0;
        total += v;
    }
    if (total == 0) return;                     // CTA-uniform
    int k = before + incl - c;
    unsigned b = bits;
    while (b) {
        const int j = __ffs(b) - 1;
        b &= b - 1;
        pos[k++] = (unsigned short)(threadIdx.x * CP_ITEMS + j);
    }
    __syncthreads();
    const unsigned long long q0 = (unsigned long long)(run_info[2 * (size_t)r] + tile_incl[blockIdx.x] - total);
    const unsigned long long src_len = src.cuts[src.nchunks];
    const int c0 = cp_search(src.cuts, src.nchunks, q0);
    const unsigned long long lo0 = src.cuts[c0], hi0 = src.cuts[c0 + 1];
    const char* const chunk0 = src.chunks[c0];
    U* const out = dst + base;
    for (int i = threadIdx.x; i < total; i += CP_THREADS) {
        const unsigned long long q = q0 + i;
        if (q >= src_len) break;                 // a plan inconsistent with the mask: never read past the values
        const char* at;
        if (q < hi0) {
            at = chunk0 + (size_t)(q - lo0) * sizeof(U);
        } else {                                 // the segment crosses into later chunks of the values
            const int cq = cp_search(src.cuts, src.nchunks, q);
            at = (const char*)src.chunks[cq] + (size_t)(q - src.cuts[cq]) * sizeof(U);
        }
        out[pos[i]] = *reinterpret_cast<const U*>(at);
    }
}

template <typename U>
int32_t launch_expand(dab_ctx* ctx, const void* mask, void* dst, size_t run_len, unsigned tpr, unsigned tiles, const long long* tile_incl,
                      const long long* run_info, const CompactDst& s, const void* scalar) {
    U sv;
    memset(&sv, 0, sizeof(sv));
    if (scalar) {
        memcpy(&sv, scalar, sizeof(U));
        expand_fill_kernel<U><<<tiles, CP_THREADS, 0, ctx->stream>>>((const uint8_t*)mask, (U*)dst, run_len, tpr, sv);
    } else {
        expand_kernel<U><<<tiles, CP_THREADS, 0, ctx->stream>>>((const uint8_t*)mask, (U*)dst, run_len, tpr, tile_incl, run_info, s);
    }
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_expand(dab_ctx* ctx, int32_t elem_bytes, const void* mask, void* dst, size_t run_len, size_t runs, const int64_t* tile_incl,
                   const int64_t* run_info, int32_t nchunks, const size_t* cuts, const void* const* chunk_ptrs, const void* scalar) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, elem_bytes == 1 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "dab_expand: elem_bytes %d (served: 1, 4, 8, 16)", elem_bytes);
    const size_t es = (size_t)elem_bytes;
    CompactDst s;
    memset(&s, 0, sizeof(s));
    if (!scalar) {
        DAB_REQUIRE(ctx, nchunks >= 1 && nchunks <= CP_MAX_CHUNKS, DAB_ERR_UNSUPPORTED, "dab_expand: %d value chunks (served: 1..%d)", nchunks,
                    CP_MAX_CHUNKS);
        DAB_REQUIRE(ctx, cuts && chunk_ptrs, DAB_ERR_ARG, "dab_expand: null value table");
        DAB_REQUIRE(ctx, cuts[0] == 0, DAB_ERR_ARG, "dab_expand: the first cut is not 0");
        s.nchunks = nchunks;
        for (int c = 0; c <= nchunks; ++c) {
            DAB_REQUIRE(ctx, c == 0 || cuts[c] >= cuts[c - 1], DAB_ERR_ARG, "dab_expand: cuts decrease");
            s.cuts[c] = cuts[c];
        }
        for (int c = 0; c < nchunks; ++c) {
            DAB_REQUIRE(ctx, cuts[c + 1] == cuts[c] || chunk_ptrs[c], DAB_ERR_ARG, "dab_expand: null pointer for non-empty chunk %d", c);
            DAB_REQUIRE(ctx, (uintptr_t)chunk_ptrs[c] % es == 0, DAB_ERR_ARG, "dab_expand: chunk %d misaligned", c);
            s.chunks[c] = (char*)chunk_ptrs[c];
        }
    }
    if (run_len == 0 || runs == 0) return DAB_OK;
    DAB_REQUIRE(ctx, mask && dst && (scalar || (tile_incl && run_info)), DAB_ERR_ARG, "dab_expand: null pointer");
    DAB_REQUIRE(ctx, (uintptr_t)dst % es == 0 && (uintptr_t)tile_incl % 8 == 0 && (uintptr_t)run_info % 8 == 0, DAB_ERR_ARG,
                "dab_expand: misaligned dst / tile_incl / run_info");
    unsigned tpr = 0, tiles = 0;
    const int32_t st = check_tiles(ctx, "dab_expand", run_len, runs, &tpr, &tiles);
    if (st != DAB_OK) return st;
    const long long* ti = (const long long*)tile_incl;
    const long long* ri = (const long long*)run_info;
    switch (elem_bytes) {
        case 1: return launch_expand<uint8_t>(ctx, mask, dst, run_len, tpr, tiles, ti, ri, s, scalar);
        case 4: return launch_expand<uint32_t>(ctx, mask, dst, run_len, tpr, tiles, ti, ri, s, scalar);
        case 8: return launch_expand<unsigned long long>(ctx, mask, dst, run_len, tpr, tiles, ti, ri, s, scalar);
        default: return launch_expand<int4>(ctx, mask, dst, run_len, tpr, tiles, ti, ri, s, scalar);
    }
}

}  // extern "C"
