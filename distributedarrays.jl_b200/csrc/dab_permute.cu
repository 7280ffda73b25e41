// dab_permute.cu -- K28: one piece of permutedims(A, perm) / permutedims!(dest, src, perm) (row f18).
//
// dst[sum_k t_k * dst_strides[k]] = src[sum_k t_k * src_strides[k]] for every coordinate t of the box, where dimension 0 is contiguous
// in the destination and one other dimension q is contiguous in the source.  dab_gather_box computes the same thing one element per
// thread, so one side of every warp access is strided; here each CTA moves one tile of the (0, q) plane through padded shared memory:
// reads run along q, writes along 0, both coalesced.  The remaining dimensions are a batch index decoded once per tile.
//
// Tiles hold NT elements (16 KiB for 4- and 16-byte elements, 8 KiB for 2- and 8-byte ones, 4 / 16 KiB for 1-byte scalar / vector);
// a plane dimension shorter than the square edge takes a narrower tile (down to one 32-byte sector per row segment) and the other
// side grows, so short dimensions do not leave the CTA idle.  When both operands, every stride outside the plane and both plane
// extents allow it, global accesses are 16 bytes wide on both sides (V elements each); otherwise one element per access.  Loads are
// plain global loads with the streaming hint, valid on a CUDA-IPC peer mapping, as in dab_transpose_box.
#include <type_traits>

#include "dab_common.cuh"

namespace {

constexpr int PB_MAXD = 8;
constexpr int PB_THREADS = 256;

struct PermGeom {
    unsigned long long e0, eq;                 // plane extents: dim 0 (contiguous in dst), dim q (contiguous in src)
    long long s0, dq;                          // src stride of dim 0, dst stride of dim q (elements)
    unsigned long long tiles_q, tiles_0, ntiles;
    int lq, l0;                                // log2 of the tile extents along q and along 0
    int nb;                                    // batch dimensions
    unsigned long long be[PB_MAXD - 2];        // batch extents, then their strides (elements)
    long long bs[PB_MAXD - 2], bd[PB_MAXD - 2];
};

template <int V> struct LogOf { static constexpr int value = 1 + LogOf<V / 2>::value; };
template <> struct LogOf<1> { static constexpr int value = 0; };

// V elements of U in one global access: uint4 when V > 1 (16 bytes), U itself when V == 1
template <typename U, int V> union Pack {
    typename std::conditional<V == 1, U, uint4>::type w;
    U e[V];
};

template <typename U, int V, int NT>
__global__ void __launch_bounds__(PB_THREADS) permute_box_kernel(U* __restrict__ dst, const U* __restrict__ src, PermGeom g) {
    extern __shared__ __align__(16) unsigned char pb_smem[];
    U* tile = reinterpret_cast<U*>(pb_smem);
    constexpr int LV = LogOf<V>::value;
    constexpr int PER = NT / V / PB_THREADS;   // global accesses per thread and side
    static_assert(PER >= 1 && PER * V * PB_THREADS == NT, "tile size");
    using W = decltype(Pack<U, V>::w);
    const int pitch = (1 << g.lq) + 1;         // padded tile row (one row per dim-0 coordinate)
    const int lqv = g.lq - LV, l0v = g.l0 - LV;
    for (unsigned long long id = blockIdx.x; id < g.ntiles; id += gridDim.x) {
        unsigned long long r = id;
        const unsigned long long q0 = (r % g.tiles_q) << g.lq;   // consecutive CTAs walk along q: source address order
        r /= g.tiles_q;
        const unsigned long long p0 = (r % g.tiles_0) << g.l0;
        r /= g.tiles_0;
        long long sb = 0, db = 0;
        for (int k = 0; k < g.nb; ++k) {
            const unsigned long long t = r % g.be[k];
            r /= g.be[k];
            sb += (long long)t * g.bs[k];
            db += (long long)t * g.bd[k];
        }
        Pack<U, V> v[PER];
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int idx = threadIdx.x + k * PB_THREADS;
            const int iq = (idx & ((1 << lqv) - 1)) << LV, i0 = idx >> lqv;
            const unsigned long long q = q0 + iq, p = p0 + i0;
            v[k].w = W{};
            if (q < g.eq && p < g.e0) v[k].w = __ldcs(reinterpret_cast<const W*>(src + sb + (long long)p * g.s0 + (long long)q));
        }
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int idx = threadIdx.x + k * PB_THREADS;
            const int iq = (idx & ((1 << lqv) - 1)) << LV, i0 = idx >> lqv;
#pragma unroll
            for (int j = 0; j < V; ++j) tile[i0 * pitch + iq + j] = v[k].e[j];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int idx = threadIdx.x + k * PB_THREADS;
            const int i0 = (idx & ((1 << l0v) - 1)) << LV, iq = idx >> l0v;
            const unsigned long long q = q0 + iq, p = p0 + i0;
            if (q < g.eq && p < g.e0) {
                Pack<U, V> o;
#pragma unroll
                for (int j = 0; j < V; ++j) o.e[j] = tile[(i0 + j) * pitch + iq];
                __stcs(reinterpret_cast<W*>(dst + db + (long long)p + (long long)q * g.dq), o.w);
            }
        }
        __syncthreads();                       // the tile is refilled by the next iteration
    }
}

int ceil_log2(unsigned long long x) {
    int l = 0;
    while ((1ull << l) < x) ++l;
    return l;
}

// Tile shape: square (2^(LNT/2) per side) when both plane extents reach the edge; otherwise the shorter plane dimension takes the
// smallest power of two that covers it, at least one 32-byte sector (and one access) per row segment, and the other side the rest.
template <typename U, int V, int NT>
int32_t launch_permute(dab_ctx* ctx, void* dst, const void* src, PermGeom g) {
    constexpr int LNT = LogOf<NT>::value, LE = LNT / 2;
    constexpr int SEG = 32 / (int)sizeof(U) > V ? 32 / (int)sizeof(U) : (V > 1 ? V : 1);
    const int lmin = LogOf<SEG>::value;
    const int lq = ceil_log2(g.eq), l0 = ceil_log2(g.e0);
    if (lq >= LE && l0 >= LE) {
        g.lq = g.l0 = LE;
    } else if (lq <= l0) {
        g.lq = lq > lmin ? lq : lmin;
        g.l0 = LNT - g.lq;
    } else {
        g.l0 = l0 > lmin ? l0 : lmin;
        g.lq = LNT - g.l0;
    }
    g.tiles_q = (g.eq + (1ull << g.lq) - 1) >> g.lq;
    g.tiles_0 = (g.e0 + (1ull << g.l0) - 1) >> g.l0;
    unsigned long long batch = 1;
    for (int k = 0; k < g.nb; ++k) batch *= g.be[k];
    g.ntiles = g.tiles_q * g.tiles_0 * batch;
    const size_t smem = (size_t)(1ull << g.l0) * (size_t)((1ull << g.lq) + 1) * sizeof(U);
    const unsigned grid = (unsigned)(g.ntiles < 0x7fffffffull ? g.ntiles : 0x7fffffffull);
    permute_box_kernel<U, V, NT><<<grid, PB_THREADS, smem, ctx->stream>>>((U*)dst, (const U*)src, g);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

bool multiple_of(long long x, int v) { return (x < 0 ? -x : x) % v == 0; }

// the 16-byte path: V elements of U per access, every access V-aligned on both sides
template <typename U, int V, int NTV, int NT1>
int32_t dispatch_width(dab_ctx* ctx, void* dst, const void* src, const PermGeom& g) {
    if constexpr (V > 1) {
        bool vec = (uintptr_t)dst % 16 == 0 && (uintptr_t)src % 16 == 0 && g.eq % V == 0 && g.e0 % V == 0 && multiple_of(g.s0, V) &&
                   multiple_of(g.dq, V);
        for (int k = 0; k < g.nb; ++k) vec = vec && multiple_of(g.bs[k], V) && multiple_of(g.bd[k], V);
        if (vec) return launch_permute<U, V, NTV>(ctx, dst, src, g);
    }
    return launch_permute<U, 1, NT1>(ctx, dst, src, g);
}

}  // namespace

extern "C" int32_t dab_permute_box(dab_ctx* ctx, int32_t elem_bytes, int32_t ndim, void* dst, const long long* dst_strides, const void* src,
                                   const long long* src_strides, const size_t* extent) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dst && src && dst_strides && src_strides && extent, DAB_ERR_ARG, "dab_permute_box: null pointer");
    DAB_REQUIRE(ctx, ndim >= 2 && ndim <= PB_MAXD, DAB_ERR_ARG, "dab_permute_box: %d dimensions (served: 2..%d)", ndim, PB_MAXD);
    DAB_REQUIRE(ctx, elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8 || elem_bytes == 16, DAB_ERR_ARG,
                "dab_permute_box: elem_bytes %d", elem_bytes);
    DAB_REQUIRE(ctx, dst_strides[0] == 1, DAB_ERR_ARG, "dab_permute_box: dimension 0 must have destination stride 1");
    int q = -1, nq = 0;
    for (int k = 1; k < ndim; ++k)
        if (src_strides[k] == 1) {
            q = k;
            ++nq;
        }
    DAB_REQUIRE(ctx, nq == 1, DAB_ERR_ARG, "dab_permute_box: %d dimensions other than 0 have source stride 1 (need exactly one)", nq);
    for (int k = 0; k < ndim; ++k)
        if (extent[k] == 0) return DAB_OK;
    PermGeom g;
    memset(&g, 0, sizeof(g));
    g.e0 = extent[0];
    g.eq = extent[q];
    g.s0 = src_strides[0];
    g.dq = dst_strides[q];
    for (int k = 1; k < ndim; ++k)
        if (k != q) {
            g.be[g.nb] = extent[k];
            g.bs[g.nb] = src_strides[k];
            g.bd[g.nb] = dst_strides[k];
            ++g.nb;
        }
    switch (elem_bytes) {
        case 1: return dispatch_width<uint8_t, 16, 16384, 4096>(ctx, dst, src, g);
        case 2: return dispatch_width<uint16_t, 8, 4096, 4096>(ctx, dst, src, g);
        case 4: return dispatch_width<uint32_t, 4, 4096, 4096>(ctx, dst, src, g);
        case 8: return dispatch_width<unsigned long long, 2, 1024, 1024>(ctx, dst, src, g);
        default: return dispatch_width<uint4, 1, 1024, 1024>(ctx, dst, src, g);
    }
}
