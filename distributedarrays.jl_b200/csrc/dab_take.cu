// dab_take.cu -- K22: R[k] = d[I[k]], the gather behind  d[I::DArray{<:Integer}]  (row f12).
//
// Replaces Base's generic getindex(A, I::AbstractArray) on a DArray: similar(d, axes(I)) (reference src/darray.jl:238) filled by
// scalar reads d[I[k]], which the reference cannot serve on the devices.  One launch fills one localpart of R from the matching
// block of I: every I[k] is a 1-based column-major LINEAR index into the whole source d, which may be spread over many chunks (local
// pointers or CUDA-IPC peer mappings).  The source table (dims, per-dimension cuts, one pointer per chunk) is passed by value in a
// __grid_constant__ parameter block and copied to shared memory by each CTA; no per-call device allocation.
//
// Memory-level parallelism: a random gather is latency-bound, so each thread keeps TK_ITEMS independent source loads in flight.
// Index loads are 16 bytes wide (and the V = 16 / sizeof(I) elements each vector carries are stored as one contiguous run) when the
// index block and the output are 16-byte aligned; otherwise a warp-strided scalar path.  Output stores are coalesced in both.  Source
// loads are plain global loads, as in dab_gather_box: the source may be a peer mapping.  Algorithmic bytes: n * (idx_bytes +
// 2 * elem_bytes) -- read the index, read the element, write the element.  The kernel only moves bytes (NaN payloads, -0.0 intact).
//
// Bounds: an index outside [1, length(d)] stores nothing and atomicMin's its position k (0-based, in the block) into *bad_pos.
#include "dab_common.cuh"

namespace {

constexpr int TK_THREADS = 256;
constexpr int TK_ITEMS = 8;                     // indices per thread, all loads issued before the first store
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

// Address of source element g (0-based linear, < len).  ND == false: the 1-D source, no division.
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

// V consecutive elements at a (V * sizeof(U))-aligned address (capped at 16 bytes per store)
template <typename U, int V>
__device__ __forceinline__ void tk_store_run(U* dst, const U (&v)[V], const bool (&ok)[V]) {
    bool all = true;
#pragma unroll
    for (int j = 0; j < V; ++j) all = all && ok[j];
    constexpr int BYTES = V * (int)sizeof(U);
    constexpr int W = BYTES < 16 ? BYTES : 16;
    using Wd = typename Word<W>::T;
    if (all) {
        struct alignas(W) Run { U e[V]; } r;
#pragma unroll
        for (int j = 0; j < V; ++j) r.e[j] = v[j];
#pragma unroll
        for (int w = 0; w < BYTES / W; ++w) reinterpret_cast<Wd*>(dst)[w] = reinterpret_cast<const Wd*>(&r)[w];
    } else {
#pragma unroll
        for (int j = 0; j < V; ++j)
            if (ok[j]) dst[j] = v[j];
    }
}

// Flat grid: CTA b fills out[b * TILE, (b + 1) * TILE).  VEC: thread t loads the 16-byte index vectors b * TILE / V + u * 256 + t
// (u < TK_ITEMS / V); otherwise it takes the single indices b * TILE + u * 256 + t (u < TK_ITEMS).
template <typename U, typename IDX, bool ND, bool VEC>
__global__ void __launch_bounds__(TK_THREADS) take_kernel(U* __restrict__ out, const IDX* __restrict__ idx, unsigned long long n,
                                                          const __grid_constant__ TakeSrc src, unsigned long long* __restrict__ bad_pos) {
    extern __shared__ unsigned long long tk_smem[];
    unsigned long long* cuts = tk_smem;
    const char** chunks = reinterpret_cast<const char**>(tk_smem + src.ncuts);
    for (int i = threadIdx.x; i < src.ncuts; i += TK_THREADS) cuts[i] = src.cuts[i];
    for (int i = threadIdx.x; i < src.nchunks; i += TK_THREADS) chunks[i] = src.chunks[i];
    __syncthreads();

    constexpr int TILE = TK_THREADS * TK_ITEMS;
    constexpr int V = VEC ? 16 / (int)sizeof(IDX) : 1;
    constexpr int NV = TK_ITEMS / V;
    const unsigned long long tile = (unsigned long long)blockIdx.x * TILE;
    unsigned long long bad = ~0ull;
    U v[NV][V];
    bool ok[NV][V];
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const unsigned long long k0 = tile + (unsigned long long)(u * TK_THREADS + threadIdx.x) * V;
        IDX iv[V];
        if (VEC && k0 + V <= n) {
            const int4 w = *reinterpret_cast<const int4*>(idx + k0);
            memcpy(iv, &w, 16);
        } else {
#pragma unroll
            for (int j = 0; j < V; ++j) iv[j] = k0 + j < n ? idx[k0 + j] : (IDX)1;
        }
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const unsigned long long g = (unsigned long long)(long long)iv[j] - 1ull;   // Int32 widened before the subtraction
            ok[u][j] = false;
            if (k0 + j >= n) continue;
            if (g >= src.len) {
                bad = min(bad, k0 + j);
                continue;
            }
            ok[u][j] = true;
            v[u][j] = *reinterpret_cast<const U*>(tk_addr<ND>(src, cuts, chunks, g, (int)sizeof(U)));
        }
    }
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const unsigned long long k0 = tile + (unsigned long long)(u * TK_THREADS + threadIdx.x) * V;
        if (k0 >= n) continue;
        tk_store_run<U, V>(out + k0, v[u], ok[u]);
    }
    if (bad != ~0ull) atomicMin(bad_pos, bad);
}

template <typename U, typename IDX, bool ND, bool VEC>
int32_t launch_take(dab_ctx* ctx, void* out, const void* idx, size_t n, const TakeSrc& s, unsigned long long* bad_pos) {
    const unsigned long long blocks = (n + TK_THREADS * TK_ITEMS - 1) / (TK_THREADS * TK_ITEMS);
    if (blocks > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_index_gather: %zu indices exceed one launch", n);
    const size_t smem = (size_t)s.ncuts * 8 + (size_t)s.nchunks * sizeof(void*);
    take_kernel<U, IDX, ND, VEC><<<(unsigned)blocks, TK_THREADS, smem, ctx->stream>>>((U*)out, (const IDX*)idx, n, s, bad_pos);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename U, typename IDX>
int32_t take_dispatch(dab_ctx* ctx, void* out, const void* idx, size_t n, const TakeSrc& s, unsigned long long* bad_pos) {
    const bool vec = ((uintptr_t)idx % 16 == 0) && ((uintptr_t)out % 16 == 0);
    if (s.ndim == 1)
        return vec ? launch_take<U, IDX, false, true>(ctx, out, idx, n, s, bad_pos) : launch_take<U, IDX, false, false>(ctx, out, idx, n, s, bad_pos);
    return vec ? launch_take<U, IDX, true, true>(ctx, out, idx, n, s, bad_pos) : launch_take<U, IDX, true, false>(ctx, out, idx, n, s, bad_pos);
}

template <typename U>
int32_t take_idx(dab_ctx* ctx, int32_t idx_dtype, void* out, const void* idx, size_t n, const TakeSrc& s, unsigned long long* bad_pos) {
    if (idx_dtype == DAB_I32) return take_dispatch<U, int32_t>(ctx, out, idx, n, s, bad_pos);
    return take_dispatch<U, long long>(ctx, out, idx, n, s, bad_pos);
}

}  // namespace

extern "C" {

int32_t dab_index_gather(dab_ctx* ctx, int32_t elem_bytes, void* out, const void* idx, int32_t idx_dtype, size_t n, int32_t ndim,
                         const size_t* dims, const int32_t* grid, const size_t* cuts, const void* const* chunk_ptrs,
                         unsigned long long* bad_pos) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, elem_bytes == 1 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "dab_index_gather: elem_bytes %d (served: 1, 4, 8, 16)", elem_bytes);
    DAB_REQUIRE(ctx, idx_dtype == DAB_I32 || idx_dtype == DAB_I64, DAB_ERR_ARG, "dab_index_gather: index dtype %d (served: I32, I64)", idx_dtype);
    DAB_REQUIRE(ctx, ndim >= 1 && ndim <= TK_MAXD, DAB_ERR_UNSUPPORTED, "dab_index_gather: %d source dimensions (served: 1..%d)", ndim, TK_MAXD);
    DAB_REQUIRE(ctx, dims && grid && cuts && chunk_ptrs, DAB_ERR_ARG, "dab_index_gather: null source table");
    if (n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, out && idx && bad_pos, DAB_ERR_ARG, "dab_index_gather: null pointer");
    const size_t ib = idx_dtype == DAB_I32 ? 4 : 8;
    DAB_REQUIRE(ctx, (uintptr_t)out % elem_bytes == 0 && (uintptr_t)idx % ib == 0 && (uintptr_t)bad_pos % 8 == 0, DAB_ERR_ARG,
                "dab_index_gather: misaligned out / idx / bad_pos");
    TakeSrc s;
    memset(&s, 0, sizeof(s));
    s.ndim = ndim;
    s.len = 1;
    int nchunks = 1, ncuts = 0;
    for (int k = 0; k < ndim; ++k) {
        DAB_REQUIRE(ctx, grid[k] >= 1, DAB_ERR_ARG, "dab_index_gather: grid[%d] = %d", k, grid[k]);
        DAB_REQUIRE(ctx, nchunks <= TK_MAX_CHUNKS / grid[k], DAB_ERR_UNSUPPORTED, "dab_index_gather: more than %d source chunks", TK_MAX_CHUNKS);
        nchunks *= grid[k];
        s.dims[k] = dims[k];
        s.inv[k] = dims[k] ? ~0ull / dims[k] : 0;
        s.grid[k] = grid[k];
        s.cut_off[k] = ncuts;
        DAB_REQUIRE(ctx, ncuts + grid[k] + 1 <= TK_MAX_CUTS, DAB_ERR_UNSUPPORTED, "dab_index_gather: more than %d cuts", TK_MAX_CUTS);
        const size_t* ck = cuts + ncuts;
        DAB_REQUIRE(ctx, ck[0] == 0 && ck[grid[k]] == dims[k], DAB_ERR_ARG, "dab_index_gather: cuts of dim %d do not span 0..%zu", k, dims[k]);
        for (int c = 0; c <= grid[k]; ++c) {
            DAB_REQUIRE(ctx, c == 0 || ck[c] >= ck[c - 1], DAB_ERR_ARG, "dab_index_gather: cuts of dim %d decrease", k);
            s.cuts[ncuts + c] = ck[c];
        }
        ncuts += grid[k] + 1;
        DAB_REQUIRE(ctx, dims[k] == 0 || s.len <= ~0ull / dims[k], DAB_ERR_ARG, "dab_index_gather: source length overflows");
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
        DAB_REQUIRE(ctx, empty || chunk_ptrs[c], DAB_ERR_ARG, "dab_index_gather: null pointer for non-empty chunk %d", c);
        DAB_REQUIRE(ctx, (uintptr_t)chunk_ptrs[c] % elem_bytes == 0, DAB_ERR_ARG, "dab_index_gather: chunk %d misaligned", c);
        s.chunks[c] = (const char*)chunk_ptrs[c];
    }
    switch (elem_bytes) {
        case 1: return take_idx<uint8_t>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        case 4: return take_idx<uint32_t>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        case 8: return take_idx<unsigned long long>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        default: return take_idx<int4>(ctx, idx_dtype, out, idx, n, s, bad_pos);
    }
}

}  // extern "C"
