// dab_compact.cu -- K23: stream compaction behind  d[mask::DArray{Bool}],  findall(mask)  and  filter(f, d)  (row f13).
//
// Replaces Base's generic getindex(A, I::AbstractArray{Bool}) / findall / filter on a DArray, which the reference would serve by one
// scalar remote read per element.  The selected elements of the whole array appear in column-major order, so every chunk is cut into
// RUNS, stretches that are contiguous in the global linear order: with k the first dimension whose grid is split, a run of a chunk
// holds all of dims 1..k-1 and the chunk's range along dim k, at one set of coordinates along dims k+1.. (DESIGN.md §3.10).  The runs
// of one chunk all have the same length run_len and lie back to back in its column-major storage, so a chunk is a regular
// (tiles_per_run x runs) table of tiles of CP_TILE elements; no tile straddles a run.
//
//   dab_compact_count  counts[b] = nonzero bytes of mask tile b                                     (reads the mask once)
//   (host)             dab_scan along each run of the table gives tile offsets, dab_scan_totals the run totals; the host gathers the
//                      run totals of every chunk and lays out the global output offsets of the runs (run_info)
//   dab_compact        each tile ranks its flags with a CTA-local scan, then writes its selected elements to the contiguous output
//                      segment [run_info[2r] + tile offset, + tile count) through the destination table  (reads the mask again)
//
// No CTA waits on another: both launches are flat grids of independent tiles.  The output is a 1-D DArray described by its cuts and
// one pointer per chunk (local or a CUDA-IPC peer mapping), passed by value in a __grid_constant__ parameter block as in K22.
// Values are moved as bytes (1, 4, 8 or 16), so NaN payloads and -0.0 are kept; index mode writes the Int64 1-based linear index.
// Indexing is 64-bit throughout.
#include "dab_compact_core.cuh"

namespace {

__global__ void __launch_bounds__(CP_THREADS) compact_count_kernel(const uint8_t* __restrict__ mask, unsigned long long run_len, unsigned tpr,
                                                                   int* __restrict__ counts) {
    __shared__ int warp_tot[CP_WARPS];
    unsigned r, t;
    unsigned long long base;
    int len;
    cp_tile(run_len, tpr, r, t, base, len);
    const int c = __reduce_add_sync(0xffffffffu, __popc(cp_flags(mask, base, len)));
    if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
#pragma unroll
        for (int w = 0; w < CP_WARPS; ++w) s += warp_tot[w];
        counts[blockIdx.x] = s;
    }
}

// U: the moved word (INDEX: long long, the 1-based linear index run_info[2r + 1] + position in run + 1).  tile_incl: inclusive scan
// of the tile counts along each run; run_info[2r]: the run's first output position.
template <typename U, bool INDEX>
__global__ void __launch_bounds__(CP_THREADS) compact_kernel(const uint8_t* __restrict__ mask, const U* __restrict__ src,
                                                             unsigned long long run_len, unsigned tpr, const long long* __restrict__ tile_incl,
                                                             const long long* __restrict__ run_info, const __grid_constant__ CompactDst dst) {
    __shared__ unsigned short pos[CP_TILE];      // tile positions of the selected elements, in rank order
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
    const unsigned long long out_len = dst.cuts[dst.nchunks];
    const int c0 = cp_search(dst.cuts, dst.nchunks, q0);
    const unsigned long long lo0 = dst.cuts[c0], hi0 = dst.cuts[c0 + 1];
    char* const chunk0 = dst.chunks[c0];
    const long long first_index = INDEX ? run_info[2 * (size_t)r + 1] + (long long)t * CP_TILE + 1 : 0;
    for (int i = threadIdx.x; i < total; i += CP_THREADS) {
        const unsigned long long q = q0 + i;
        if (q >= out_len) break;                 // a plan inconsistent with the mask: never write past the output
        const int p = pos[i];
        U v;
        if constexpr (INDEX) {
            v = first_index + p;
        } else {
            v = __ldg(src + base + p);          // d's own chunk: read-only for the whole launch
        }
        char* at;
        if (q < hi0) {
            at = chunk0 + (size_t)(q - lo0) * sizeof(U);
        } else {                                 // the segment crosses into later chunks of the output
            const int cq = cp_search(dst.cuts, dst.nchunks, q);
            at = dst.chunks[cq] + (size_t)(q - dst.cuts[cq]) * sizeof(U);
        }
        *reinterpret_cast<U*>(at) = v;
    }
}

template <typename U, bool INDEX>
int32_t launch_compact(dab_ctx* ctx, const void* mask, const void* src, size_t run_len, unsigned tpr, unsigned tiles,
                       const long long* tile_incl, const long long* run_info, const CompactDst& d) {
    compact_kernel<U, INDEX><<<tiles, CP_THREADS, 0, ctx->stream>>>((const uint8_t*)mask, (const U*)src, run_len, tpr, tile_incl, run_info, d);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_compact_count(dab_ctx* ctx, const void* mask, size_t run_len, size_t runs, int32_t* counts) {
    DAB_ENTER(ctx);
    if (run_len == 0 || runs == 0) return DAB_OK;
    DAB_REQUIRE(ctx, mask && counts, DAB_ERR_ARG, "dab_compact_count: null pointer");
    DAB_REQUIRE(ctx, (uintptr_t)counts % 4 == 0, DAB_ERR_ARG, "dab_compact_count: misaligned counts");
    unsigned tpr = 0, tiles = 0;
    const int32_t st = check_tiles(ctx, "dab_compact_count", run_len, runs, &tpr, &tiles);
    if (st != DAB_OK) return st;
    compact_count_kernel<<<tiles, CP_THREADS, 0, ctx->stream>>>((const uint8_t*)mask, run_len, tpr, counts);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

int32_t dab_compact(dab_ctx* ctx, int32_t elem_bytes, const void* mask, const void* src, size_t run_len, size_t runs, const int64_t* tile_incl,
                    const int64_t* run_info, int32_t nchunks, const size_t* cuts, void* const* chunk_ptrs) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, elem_bytes == DAB_COMPACT_INDEX || elem_bytes == 1 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "dab_compact: elem_bytes %d (served: 1, 4, 8, 16, or DAB_COMPACT_INDEX)", elem_bytes);
    DAB_REQUIRE(ctx, nchunks >= 1 && nchunks <= CP_MAX_CHUNKS, DAB_ERR_UNSUPPORTED, "dab_compact: %d output chunks (served: 1..%d)", nchunks,
                CP_MAX_CHUNKS);
    DAB_REQUIRE(ctx, cuts && chunk_ptrs, DAB_ERR_ARG, "dab_compact: null destination table");
    const size_t es = elem_bytes == DAB_COMPACT_INDEX ? 8 : (size_t)elem_bytes;
    CompactDst d;
    memset(&d, 0, sizeof(d));
    d.nchunks = nchunks;
    DAB_REQUIRE(ctx, cuts[0] == 0, DAB_ERR_ARG, "dab_compact: the first cut is not 0");
    for (int c = 0; c <= nchunks; ++c) {
        DAB_REQUIRE(ctx, c == 0 || cuts[c] >= cuts[c - 1], DAB_ERR_ARG, "dab_compact: cuts decrease");
        d.cuts[c] = cuts[c];
    }
    for (int c = 0; c < nchunks; ++c) {
        DAB_REQUIRE(ctx, cuts[c + 1] == cuts[c] || chunk_ptrs[c], DAB_ERR_ARG, "dab_compact: null pointer for non-empty chunk %d", c);
        DAB_REQUIRE(ctx, (uintptr_t)chunk_ptrs[c] % es == 0, DAB_ERR_ARG, "dab_compact: chunk %d misaligned", c);
        d.chunks[c] = (char*)chunk_ptrs[c];
    }
    if (run_len == 0 || runs == 0) return DAB_OK;
    DAB_REQUIRE(ctx, mask && tile_incl && run_info && (elem_bytes == DAB_COMPACT_INDEX || src), DAB_ERR_ARG, "dab_compact: null pointer");
    DAB_REQUIRE(ctx, (uintptr_t)tile_incl % 8 == 0 && (uintptr_t)run_info % 8 == 0 && (uintptr_t)src % es == 0, DAB_ERR_ARG,
                "dab_compact: misaligned tile_incl / run_info / src");
    unsigned tpr = 0, tiles = 0;
    const int32_t st = check_tiles(ctx, "dab_compact", run_len, runs, &tpr, &tiles);
    if (st != DAB_OK) return st;
    const long long* ti = (const long long*)tile_incl;
    const long long* ri = (const long long*)run_info;
    switch (elem_bytes) {
        case DAB_COMPACT_INDEX: return launch_compact<long long, true>(ctx, mask, nullptr, run_len, tpr, tiles, ti, ri, d);
        case 1: return launch_compact<uint8_t, false>(ctx, mask, src, run_len, tpr, tiles, ti, ri, d);
        case 4: return launch_compact<uint32_t, false>(ctx, mask, src, run_len, tpr, tiles, ti, ri, d);
        case 8: return launch_compact<unsigned long long, false>(ctx, mask, src, run_len, tpr, tiles, ti, ri, d);
        default: return launch_compact<int4, false>(ctx, mask, src, run_len, tpr, tiles, ti, ri, d);
    }
}

}  // extern "C"
