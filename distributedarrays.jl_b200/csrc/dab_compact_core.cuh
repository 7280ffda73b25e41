// dab_compact_core.cuh -- K23's tile table (runs of run_len elements cut into CP_TILE tiles), its flag loads, its destination table and
// the launch-size check, shared by the compaction of dab_compact.cu (K23) and the expansion of dab_expand.cu (K25).
#pragma once
#include "dab_common.cuh"

namespace {

constexpr int CP_THREADS = 256;
constexpr int CP_ITEMS = 16;                     // mask bytes per thread: one 16-byte load when aligned
constexpr int CP_TILE = CP_THREADS * CP_ITEMS;   // must equal DAB_COMPACT_TILE
constexpr int CP_WARPS = CP_THREADS / 32;
constexpr int CP_MAX_CHUNKS = 1024;
static_assert(CP_TILE == DAB_COMPACT_TILE, "tile size differs from the header's");

struct CompactDst {
    unsigned long long cuts[CP_MAX_CHUNKS + 1];  // 0-based first output position of each chunk, then the output length
    char* chunks[CP_MAX_CHUNKS];                 // NULL for an empty chunk
    int nchunks;
};
static_assert(sizeof(CompactDst) <= 32764, "kernel parameter block exceeds the 32764-byte limit");

// Tile b of the (tiles_per_run x runs) table: its first chunk element and its length.
__device__ __forceinline__ void cp_tile(unsigned long long run_len, unsigned tpr, unsigned& r, unsigned& t, unsigned long long& base,
                                        int& len) {
    r = blockIdx.x / tpr;
    t = blockIdx.x - r * tpr;
    const unsigned long long in_run = (unsigned long long)t * CP_TILE;
    base = (unsigned long long)r * run_len + in_run;
    const unsigned long long left = run_len - in_run;
    len = left < (unsigned long long)CP_TILE ? (int)left : CP_TILE;
}

// Bit j of the result: tile element threadIdx.x * CP_ITEMS + j is selected (its mask byte is nonzero).  16-byte loads when the tile
// starts 16-byte aligned (a CTA-uniform choice), byte loads otherwise and for a partial group at the tile's end.
__device__ __forceinline__ unsigned cp_flags(const uint8_t* __restrict__ mask, unsigned long long base, int len) {
    const uint8_t* p = mask + base;
    const int first = threadIdx.x * CP_ITEMS;
    unsigned bits = 0;
    if (((uintptr_t)p & 15) == 0 && first + CP_ITEMS <= len) {
        const uint4 w = *reinterpret_cast<const uint4*>(p + first);
        const unsigned words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const unsigned ne = __vcmpne4(words[q], 0u);   // 0xff in every nonzero byte
#pragma unroll
            for (int j = 0; j < 4; ++j) bits |= ((ne >> (8 * j)) & 1u) << (4 * q + j);
        }
    } else {
#pragma unroll
        for (int j = 0; j < CP_ITEMS; ++j)
            if (first + j < len && p[first + j]) bits |= 1u << j;
    }
    return bits;
}

// largest c in [0, n) with cuts[c] <= q (the cuts live in the parameter block; q is the same for every thread at the call sites
// that matter, so the loads are broadcasts)
__device__ __forceinline__ int cp_search(const unsigned long long* cuts, int n, unsigned long long q) {
    int lo = 0;
    while (n > 1) {
        const int half = n >> 1;
        if (cuts[lo + half] <= q) {
            lo += half;
            n -= half;
        } else {
            n = half;
        }
    }
    return lo;
}

int32_t check_tiles(dab_ctx* ctx, const char* name, size_t run_len, size_t runs, unsigned* tpr, unsigned* tiles) {
    const unsigned long long t = (run_len + CP_TILE - 1) / CP_TILE;
    if (t > 0x7fffffffull || (t && runs > 0x7fffffffull / t))
        return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "%s: %zu runs of %zu elements exceed one launch", name, runs, run_len);
    *tpr = (unsigned)t;
    *tiles = (unsigned)(t * runs);
    return DAB_OK;
}

}  // namespace
