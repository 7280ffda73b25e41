// dab_slab.cu -- K8: the "halo" read.  Copies an up-to-4-D box out of a (possibly PEER) chunk into a local dense array.
//
// Replaces, per intersecting chunk, the owner-side  localpart(d)[idxs...]  + Julia serialisation + TCP + a[idxs...] = ...
// of setindex!(a::Array, s::SubDArray, I...) (reference src/darray.jl:798-820), chunk(d, pid) (:458) and the non-local branch
// of makelocal (:361-366).  The reference's read is pull-style and one-sided from the reader's point of view; so is this:
// the READER launches the kernel and loads straight from the owner's HBM (peer mapping / CUDA IPC) over NVLink 5, UNROLL
// independent loads in flight per thread, and stores into its own HBM.  Roofline: NVLink (peer) or HBM (local): elem_bytes moved
// once per element.
//
// Vector width: loads are the scarce resource on the peer path (NVLink request rate), so the LOAD unit is made as wide as the
// source geometry allows (16 B when source base / pitches / row length are 16-byte multiples); when the destination is less
// aligned than the source the value is stored in smaller pieces (local HBM stores are cheap).  A contiguous slab whose source
// start is not 16-byte aligned is split on the host into head (< 16 B) + 16-byte-aligned body + tail.
#include "dab_common.cuh"

namespace {

struct BoxGeom {
    unsigned long long upr;         // load units per row
    unsigned long long e1, e2, e3;  // rows along dims 1..3
    long long sp1, sp2, sp3;        // src pitches in bytes
    long long dp1, dp2, dp3;        // dst pitches in bytes
};

template <typename U, typename S>
__device__ __forceinline__ void store_as(char* dst, const U& v) {
    constexpr int N = sizeof(U) / sizeof(S);
    const S* p = reinterpret_cast<const S*>(&v);
#pragma unroll
    for (int k = 0; k < N; ++k) reinterpret_cast<S*>(dst)[k] = p[k];
}

// U = load unit, S = store unit (sizeof(S) <= sizeof(U)), I = index type
template <typename U, typename S, typename I, int UNROLL>
__global__ void __launch_bounds__(256) copy_box_kernel(char* __restrict__ dst, const char* __restrict__ src, BoxGeom g, I total) {
    // flat grid: CTA b moves the 256*UNROLL consecutive units starting at b*256*UNROLL (UNROLL independent loads per thread in
    // flight); the block scheduler issues CTAs in address order, which keeps the owner's (possibly remote) DRAM pages a compact window
    const I base = (I)blockIdx.x * (I)(256 * UNROLL) + threadIdx.x;
    const I upr = (I)g.upr, e1 = (I)g.e1, e2 = (I)g.e2;
    const bool flat = (g.e1 == 1 && g.e2 == 1 && g.e3 == 1);
    U v[UNROLL];
    size_t doff[UNROLL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
        const I id = base + (I)(u * 256);
        ok[u] = id < total;
        if (!ok[u]) continue;
        size_t soff;
        if (flat) {
            soff = doff[u] = (size_t)id * sizeof(U);
        } else {
            I row = id / upr, col = id - row * upr;
            I j = row % e1, t = row / e1;
            I k = t % e2, l = t / e2;
            soff = (size_t)col * sizeof(U) + (size_t)j * g.sp1 + (size_t)k * g.sp2 + (size_t)l * g.sp3;
            doff[u] = (size_t)col * sizeof(U) + (size_t)j * g.dp1 + (size_t)k * g.dp2 + (size_t)l * g.dp3;
        }
        v[u] = *reinterpret_cast<const U*>(src + soff);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
        if (ok[u]) store_as<U, S>(dst + doff[u], v[u]);
}

constexpr int COPY_UNROLL = 8;

template <typename U, typename S>
int32_t launch_copy(dab_ctx* ctx, char* dst, const char* src, const BoxGeom& g) {
    unsigned long long total = g.upr * g.e1 * g.e2 * g.e3;
    if (total == 0) return DAB_OK;
    const size_t work = (size_t)((total + 256ull * COPY_UNROLL - 1) / (256ull * COPY_UNROLL));
    if (work > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_ARG, "box too large for one launch");
    if (total < (1ull << 31))
        copy_box_kernel<U, S, unsigned int, COPY_UNROLL><<<(unsigned)work, 256, 0, ctx->stream>>>(dst, src, g, (unsigned int)total);
    else
        copy_box_kernel<U, S, unsigned long long, COPY_UNROLL><<<(unsigned)work, 256, 0, ctx->stream>>>(dst, src, g, total);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename U>
int32_t launch_copy_s(dab_ctx* ctx, char* dst, const char* src, const BoxGeom& g, size_t svec) {
    if (svec >= sizeof(U)) return launch_copy<U, U>(ctx, dst, src, g);
    if constexpr (sizeof(U) > 8)
        if (svec == 8) return launch_copy<U, long long>(ctx, dst, src, g);
    if constexpr (sizeof(U) > 4)
        if (svec == 4) return launch_copy<U, int>(ctx, dst, src, g);
    if constexpr (sizeof(U) > 2)
        if (svec == 2) return launch_copy<U, short>(ctx, dst, src, g);
    if constexpr (sizeof(U) > 1) return launch_copy<U, char>(ctx, dst, src, g);
    return launch_copy<U, U>(ctx, dst, src, g);
}

size_t pow2_align(size_t bits) {
    size_t v = 16;
    while (v > 1 && (bits & (v - 1))) v >>= 1;
    return v;
}

// rows of row_bytes bytes; e[] rows with pitches; load unit from the source geometry, store unit from the destination's
int32_t copy_rows(dab_ctx* ctx, char* t, const char* s, size_t row_bytes, const size_t e[3], const long long spp[3], const long long dpp[3]) {
    size_t sbits = (size_t)(uintptr_t)s | row_bytes, dbits = (size_t)(uintptr_t)t | row_bytes;
    for (int d = 0; d < 3; ++d)
        if (e[d] > 1) {
            sbits |= (size_t)spp[d];
            dbits |= (size_t)dpp[d];
        }
    const size_t lvec = pow2_align(sbits), svec = pow2_align(dbits);
    BoxGeom g;
    g.upr = row_bytes / lvec;
    g.e1 = e[0];
    g.e2 = e[1];
    g.e3 = e[2];
    g.sp1 = spp[0]; g.sp2 = spp[1]; g.sp3 = spp[2];
    g.dp1 = dpp[0]; g.dp2 = dpp[1]; g.dp3 = dpp[2];
    switch (lvec) {
        case 16: return launch_copy_s<int4>(ctx, t, s, g, svec);
        case 8: return launch_copy_s<long long>(ctx, t, s, g, svec);
        case 4: return launch_copy_s<int>(ctx, t, s, g, svec);
        case 2: return launch_copy_s<short>(ctx, t, s, g, svec);
        default: return launch_copy_s<char>(ctx, t, s, g, svec);
    }
}


// ---- strided / vector-indexed views: gather ------------------------------------------------------------------------------------------
// The piece of  Array(d[I...])  that lives in one chunk when some index is a StepRange or a Vector{Int} (reference src/darray.jl:661,
// 798-820 with indexin_mask / restrict_indices :706-781).  Per dimension k the element offset of coordinate t is either affine
// (t * stride[k]) or read from an index table (table[k][t]); source and destination each have their own.  Up to 8 dimensions.
constexpr int GB_MAXD = 8;
struct GatherGeom {
    unsigned long long extent[GB_MAXD];
    long long dst_stride[GB_MAXD], src_stride[GB_MAXD];          // elements; src may be negative (reversed StepRange)
    const long long* dst_index[GB_MAXD];                          // device tables of element offsets, or nullptr
    const long long* src_index[GB_MAXD];
    int ndim;
};

template <typename U>
__global__ void __launch_bounds__(256) gather_box_kernel(U* __restrict__ dst, const U* __restrict__ src, GatherGeom g, unsigned long long total) {
    for (unsigned long long id = (unsigned long long)blockIdx.x * 256 + threadIdx.x; id < total; id += (unsigned long long)gridDim.x * 256) {
        unsigned long long r = id;
        long long doff = 0, soff = 0;
#pragma unroll
        for (int k = 0; k < GB_MAXD; ++k) {
            if (k < g.ndim) {
                const unsigned long long t = r % g.extent[k];
                r /= g.extent[k];
                doff += g.dst_index[k] ? g.dst_index[k][t] : (long long)t * g.dst_stride[k];
                soff += g.src_index[k] ? g.src_index[k][t] : (long long)t * g.src_stride[k];
            }
        }
        dst[doff] = src[soff];
    }
}

template <typename U>
int32_t launch_gather(dab_ctx* ctx, void* dst, const void* src, const GatherGeom& g, unsigned long long total) {
    const int grid = dab_grid_for(ctx, (size_t)((total + 255) / 256), 16);
    gather_box_kernel<U><<<grid, 256, 0, ctx->stream>>>((U*)dst, (const U*)src, g, total);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_copy_box(dab_ctx* ctx, int32_t elem_bytes, void* dst, const size_t dst_shape[4], const size_t dst_off[4], const void* src,
                     const size_t src_shape[4], const size_t src_off[4], const size_t extent[4]) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dst && src && dst_shape && dst_off && src_shape && src_off && extent, DAB_ERR_ARG, "dab_copy_box: null pointer");
    DAB_REQUIRE(ctx, elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "dab_copy_box: elem_bytes %d", elem_bytes);
    for (int d = 0; d < 4; ++d) {
        if (extent[d] == 0) return DAB_OK;
        DAB_REQUIRE(ctx, src_off[d] + extent[d] <= src_shape[d] && dst_off[d] + extent[d] <= dst_shape[d], DAB_ERR_DIM_MISMATCH,
                    "dab_copy_box: box exceeds array in dim %d (BoundsError)", d);
    }
    // byte geometry
    size_t es = (size_t)elem_bytes;
    size_t sp[4], dp[4];  // pitch (bytes) of one step along dim d
    sp[0] = dp[0] = es;
    for (int d = 1; d < 4; ++d) {
        sp[d] = sp[d - 1] * src_shape[d - 1];
        dp[d] = dp[d - 1] * dst_shape[d - 1];
    }
    const char* s = (const char*)src;
    char* t = (char*)dst;
    for (int d = 0; d < 4; ++d) {
        s += src_off[d] * sp[d];
        t += dst_off[d] * dp[d];
    }
    // collapse: a dim that spans both arrays entirely merges into the run below it
    size_t row_bytes = extent[0] * es;
    size_t e[3] = {extent[1], extent[2], extent[3]};
    long long spp[3] = {(long long)sp[1], (long long)sp[2], (long long)sp[3]};
    long long dpp[3] = {(long long)dp[1], (long long)dp[2], (long long)dp[3]};
    int nd = 3;
    while (nd > 0 && ((size_t)spp[0] == row_bytes && (size_t)dpp[0] == row_bytes || e[0] == 1)) {
        if (e[0] > 1) row_bytes *= e[0];
        for (int d = 0; d + 1 < nd; ++d) {
            e[d] = e[d + 1];
            spp[d] = spp[d + 1];
            dpp[d] = dpp[d + 1];
        }
        e[nd - 1] = 1;
        spp[nd - 1] = 0;
        dpp[nd - 1] = 0;
        --nd;
    }
    if (nd == 0 && row_bytes >= 4096) {
        // contiguous slab: peel so that the SOURCE body is 16-byte aligned (peer loads stay 16 B wide)
        size_t head = (16 - ((uintptr_t)s & 15)) & 15;
        head -= head % es;  // stay on element boundaries (es divides 16)
        if (head) {
            int32_t st = copy_rows(ctx, t, s, head, e, spp, dpp);
            if (st != DAB_OK) return st;
        }
        size_t body = (row_bytes - head) & ~(size_t)15;
        if (body) {
            int32_t st = copy_rows(ctx, t + head, s + head, body, e, spp, dpp);
            if (st != DAB_OK) return st;
        }
        size_t tail = row_bytes - head - body;
        if (tail) return copy_rows(ctx, t + head + body, s + head + body, tail, e, spp, dpp);
        return DAB_OK;
    }
    return copy_rows(ctx, t, s, row_bytes, e, spp, dpp);
}

int32_t dab_gather_box(dab_ctx* ctx, int32_t elem_bytes, int32_t ndim, void* dst, const long long* dst_strides, const void* const* dst_index,
                       const void* src, const long long* src_strides, const void* const* src_index, const size_t* extent) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dst && src && extent && dst_strides && src_strides, DAB_ERR_ARG, "dab_gather_box: null pointer");
    DAB_REQUIRE(ctx, ndim >= 1 && ndim <= GB_MAXD, DAB_ERR_UNSUPPORTED, "dab_gather_box: %d dimensions (served: 1..%d)", ndim, GB_MAXD);
    GatherGeom g;
    memset(&g, 0, sizeof(g));
    g.ndim = ndim;
    unsigned long long total = 1;
    for (int k = 0; k < ndim; ++k) {
        if (extent[k] == 0) return DAB_OK;
        g.extent[k] = extent[k];
        g.dst_stride[k] = dst_strides[k];
        g.src_stride[k] = src_strides[k];
        g.dst_index[k] = dst_index ? (const long long*)dst_index[k] : nullptr;
        g.src_index[k] = src_index ? (const long long*)src_index[k] : nullptr;
        total *= extent[k];
    }
    switch (elem_bytes) {
        case 1: return launch_gather<uint8_t>(ctx, dst, src, g, total);
        case 2: return launch_gather<uint16_t>(ctx, dst, src, g, total);
        case 4: return launch_gather<uint32_t>(ctx, dst, src, g, total);
        case 8: return launch_gather<unsigned long long>(ctx, dst, src, g, total);
        case 16: return launch_gather<int4>(ctx, dst, src, g, total);
        default: return dab_fail(ctx, DAB_ERR_ARG, "dab_gather_box: elem_bytes %d", elem_bytes);
    }
}

}  // extern "C"
