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
#include "dab_take_core.cuh"

namespace {

constexpr int TK_THREADS = 256;
constexpr int TK_ITEMS = 8;                     // indices per thread, all loads issued before the first store

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
    const int32_t st = tk_fill_src(ctx, "dab_index_gather", ndim, dims, grid, cuts, chunk_ptrs, (size_t)elem_bytes, &s);
    if (st != DAB_OK) return st;
    switch (elem_bytes) {
        case 1: return take_idx<uint8_t>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        case 4: return take_idx<uint32_t>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        case 8: return take_idx<unsigned long long>(ctx, idx_dtype, out, idx, n, s, bad_pos);
        default: return take_idx<int4>(ctx, idx_dtype, out, idx, n, s, bad_pos);
    }
}

}  // extern "C"
