// dab_take_core.cuh -- K22's description of a chunked array (dims, per-dimension cuts, one pointer per chunk) and the addressing of
// a 1-based linear index in it, shared by the gather of dab_take.cu (K22) and the scatter of dab_scatter.cu (K24).
#pragma once
#include "dab_common.cuh"

namespace {

constexpr int TK_MAXD = 8;
constexpr int TK_MAX_CHUNKS = 1024;
// sum over dims of grid[k] + 1: for integers g >= 1, g1 + g2 <= g1 * g2 + 1, so sum(grid) <= prod(grid) + ndim - 1 and the cuts of
// any grid of at most TK_MAX_CHUNKS chunks fit (1039 for grid (1024, 1, ..., 1) over 8 dims)
constexpr int TK_MAX_CUTS = TK_MAX_CHUNKS + 2 * TK_MAXD - 1;

struct TakeSrc {
    unsigned long long dims[TK_MAXD];
    unsigned long long inv[TK_MAXD];             // floor((2^64 - 1) / dims[k]): division by a multiply-high (tk_divmod)
    unsigned long long len;                      // prod(dims)
    int ndim, nchunks, ncuts;
    int grid[TK_MAXD];
    int cut_off[TK_MAXD];                        // dim k's grid[k] + 1 cuts start at cuts[cut_off[k]]
    unsigned long long cuts[TK_MAX_CUTS];        // 0-based first element of each chunk along the dim, then dims[k]
    const char* chunks[TK_MAX_CHUNKS];           // column-major grid order; NULL for an empty chunk
};
static_assert(sizeof(TakeSrc) <= 32764, "kernel parameter block exceeds the 32764-byte limit");

// largest c in [0, n) with cuts[c] <= x (cuts[0] == 0 <= x): skips empty chunks, whose cut equals the next one
__device__ __forceinline__ int tk_search(const unsigned long long* cuts, int n, unsigned long long x) {
    int lo = 0;
    while (n > 1) {
        const int half = n >> 1;
        if (cuts[lo + half] <= x) {
            lo += half;
            n -= half;
        } else {
            n = half;
        }
    }
    return lo;
}

// q = x / d, x -= q * d, inline (the 64-bit division subroutine would spill around its call).  inv = floor((2^64 - 1) / d)
// makes x * inv / 2^64 exceed x / d - 1, so the estimate is at most 1 short.
__device__ __forceinline__ unsigned long long tk_divmod(unsigned long long& x, unsigned long long d, unsigned long long inv) {
    unsigned long long q = __umul64hi(x, inv);
    x -= q * d;
    while (x >= d) {
        x -= d;
        ++q;
    }
    return q;
}

// Chunk of source element g (0-based linear, < len) in column-major grid order, and g's column-major offset inside that chunk.
// ND == false: the 1-D source, no division.
template <bool ND>
__device__ __forceinline__ int tk_locate(const TakeSrc& s, const unsigned long long* cuts, unsigned long long g, unsigned long long& off) {
    if (!ND) {
        const int c = tk_search(cuts, s.grid[0], g);
        off = g - cuts[c];
        return c;
    }
    unsigned long long rem = g, mult = 1;
    int chunk = 0, cstride = 1;
    off = 0;
#pragma unroll
    for (int k = 0; k < TK_MAXD; ++k) {
        if (k < s.ndim) {
            unsigned long long x = rem;
            if (k + 1 < s.ndim) rem = tk_divmod(x, s.dims[k], s.inv[k]);
            const unsigned long long* ck = cuts + s.cut_off[k];
            const int c = tk_search(ck, s.grid[k], x);
            off += (x - ck[c]) * mult;
            mult *= ck[c + 1] - ck[c];
            chunk += c * cstride;
            cstride *= s.grid[k];
        }
    }
    return chunk;
}

// Address of source element g (0-based linear, < len).  The same walk as tk_locate, kept separate so that K22's code stays as built.
template <bool ND>
__device__ __forceinline__ const char* tk_addr(const TakeSrc& s, const unsigned long long* cuts, const char* const* chunks,
                                               unsigned long long g, int es) {
    if (!ND) {
        const int c = tk_search(cuts, s.grid[0], g);
        return chunks[c] + (size_t)(g - cuts[c]) * es;
    }
    unsigned long long rem = g, off = 0, mult = 1;
    int chunk = 0, cstride = 1;
#pragma unroll
    for (int k = 0; k < TK_MAXD; ++k) {
        if (k < s.ndim) {
            unsigned long long x = rem;
            if (k + 1 < s.ndim) rem = tk_divmod(x, s.dims[k], s.inv[k]);
            const unsigned long long* ck = cuts + s.cut_off[k];
            const int c = tk_search(ck, s.grid[k], x);
            off += (x - ck[c]) * mult;
            mult *= ck[c + 1] - ck[c];
            chunk += c * cstride;
            cstride *= s.grid[k];
        }
    }
    return chunks[chunk] + (size_t)off * es;
}

template <int W> struct Word;
template <> struct Word<1> { using T = uint8_t; };
template <> struct Word<2> { using T = uint16_t; };
template <> struct Word<4> { using T = uint32_t; };
template <> struct Word<8> { using T = unsigned long long; };
template <> struct Word<16> { using T = int4; };

// Fills *s from the C ABI's description of a chunked array (see dab_index_gather in include/dab200.h) after checking it: grid sizes,
// at most TK_MAX_CHUNKS chunks and TK_MAX_CUTS cuts, cuts that span 0..dims[k] without decreasing, a pointer for every non-empty chunk,
// each aligned to `align` bytes.  `name` prefixes the error messages.
inline int32_t tk_fill_src(dab_ctx* ctx, const char* name, int32_t ndim, const size_t* dims, const int32_t* grid, const size_t* cuts,
                           const void* const* chunk_ptrs, size_t align, TakeSrc* out) {
    DAB_REQUIRE(ctx, ndim >= 1 && ndim <= TK_MAXD, DAB_ERR_UNSUPPORTED, "%s: %d source dimensions (served: 1..%d)", name, ndim, TK_MAXD);
    DAB_REQUIRE(ctx, dims && grid && cuts && chunk_ptrs, DAB_ERR_ARG, "%s: null source table", name);
    TakeSrc& s = *out;
    memset(&s, 0, sizeof(s));
    s.ndim = ndim;
    s.len = 1;
    int nchunks = 1, ncuts = 0;
    for (int k = 0; k < ndim; ++k) {
        DAB_REQUIRE(ctx, grid[k] >= 1, DAB_ERR_ARG, "%s: grid[%d] = %d", name, k, grid[k]);
        DAB_REQUIRE(ctx, nchunks <= TK_MAX_CHUNKS / grid[k], DAB_ERR_UNSUPPORTED, "%s: more than %d source chunks", name, TK_MAX_CHUNKS);
        nchunks *= grid[k];
        s.dims[k] = dims[k];
        s.inv[k] = dims[k] ? ~0ull / dims[k] : 0;
        s.grid[k] = grid[k];
        s.cut_off[k] = ncuts;
        DAB_REQUIRE(ctx, ncuts + grid[k] + 1 <= TK_MAX_CUTS, DAB_ERR_UNSUPPORTED, "%s: more than %d cuts", name, TK_MAX_CUTS);
        const size_t* ck = cuts + ncuts;
        DAB_REQUIRE(ctx, ck[0] == 0 && ck[grid[k]] == dims[k], DAB_ERR_ARG, "%s: cuts of dim %d do not span 0..%zu", name, k, dims[k]);
        for (int c = 0; c <= grid[k]; ++c) {
            DAB_REQUIRE(ctx, c == 0 || ck[c] >= ck[c - 1], DAB_ERR_ARG, "%s: cuts of dim %d decrease", name, k);
            s.cuts[ncuts + c] = ck[c];
        }
        ncuts += grid[k] + 1;
        DAB_REQUIRE(ctx, dims[k] == 0 || s.len <= ~0ull / dims[k], DAB_ERR_ARG, "%s: source length overflows", name);
        s.len *= dims[k];
    }
    s.nchunks = nchunks;
    s.ncuts = ncuts;
    // a non-empty chunk must have a pointer (an empty one is never addressed: the cut search skips it)
    for (int c = 0; c < nchunks; ++c) {
        int r = c;
        bool empty = false;
        for (int k = 0; k < ndim; ++k) {
            const int ci = r % grid[k];
            r /= grid[k];
            empty = empty || s.cuts[s.cut_off[k] + ci + 1] == s.cuts[s.cut_off[k] + ci];
        }
        DAB_REQUIRE(ctx, empty || chunk_ptrs[c], DAB_ERR_ARG, "%s: null pointer for non-empty chunk %d", name, c);
        DAB_REQUIRE(ctx, (uintptr_t)chunk_ptrs[c] % align == 0, DAB_ERR_ARG, "%s: chunk %d misaligned", name, c);
        s.chunks[c] = (const char*)chunk_ptrs[c];
    }
    return DAB_OK;
}

}  // namespace
