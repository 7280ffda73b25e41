// dab_reduce_traits.cuh -- reduction traits, map functors, block-level reduction and the launch plumbing shared by the reduction
// kernels (dab_reduce.cu, dab_reducedim.cu, dab_findminmax.cu; dab_scan.cu uses the traits)
#pragma once
#include <type_traits>

#include "dab_scalar_ops.cuh"

namespace {

constexpr int RD_THREADS = 256;
constexpr int RD_UNROLL = 4;  // 16-byte loads in flight per thread in the flat-grid kernels

// ---- flat grid of the whole-chunk kernels (reduce_kernel, findminmax_kernel) ----------------------------------------------------
// x[0, head) is the misaligned head, then tiles of RD_THREADS * RD_UNROLL 16-byte vectors.  CTA b owns the tiles_per_cta consecutive
// tiles from b * tiles_per_cta: 32 KiB of input per CTA (2 tiles), more once the grid would exceed DAB_MAX_REDUCE_BLOCKS, which is
// what keeps one partial per CTA inside ctx->block_partials.
struct FlatGrid {
    size_t head, grid;
    int tiles_per_cta;
};
template <typename T>
FlatGrid flat_grid(const T* x, size_t n) {
    constexpr int VPT = 16 / sizeof(T);
    size_t head = ((16 - ((uintptr_t)x & 15)) & 15) / sizeof(T);
    if (head > n) head = n;
    const size_t tiles = (n - head) / ((size_t)VPT * RD_THREADS * RD_UNROLL);
    size_t k = 2;
    if ((tiles + k - 1) / k > (size_t)DAB_MAX_REDUCE_BLOCKS) k = (tiles + DAB_MAX_REDUCE_BLOCKS - 1) / DAB_MAX_REDUCE_BLOCKS;
    size_t grid = (tiles + k - 1) / k;
    if (grid < 1) grid = 1;
    return FlatGrid{head, grid, (int)k};
}

// ---- split count of the dims kernels (dab_reducedim.cu, dab_findminmax.cu) ------------------------------------------------------
// Splits of the reduced extent that bring `have` work units up to `target`: ceil(target / have) when have < target, at most
// max_split (taken as >= 1) and 1024.  The partials of the splits go to ctx->dim_scratch.
inline int dim_nsplit(size_t have, size_t target, size_t max_split) {
    if (max_split < 1) max_split = 1;
    const size_t want = have >= target ? 1 : (target + have - 1) / have;
    const int nsplit = (int)(want < max_split ? want : max_split);
    return nsplit > 1024 ? 1024 : nsplit;
}

// ---------------------------------------------------------------------------------------------------------------
// Reduce "traits": V = value type after the map, W = value type inside a tile step, A = accumulator carried across tiles /
// threads / CTAs.
//   pre(V) -> W right after the map, tile(W, W) -> W combine inside a tile step, lift(W) -> A, comb(A, A) -> A (associative up
//   to rounding).
// W is V except for Int32 sums and products, which widen to Int64 before the first add or multiply (Base.add_sum /
// Base.mul_prod): a tile of 16 Int32 values would otherwise wrap at 32 bits before it reaches the Int64 accumulator.
// ---------------------------------------------------------------------------------------------------------------
template <typename V>
using WideInt32 = typename std::conditional<std::is_same<V, int32_t>::value, long long, V>::type;
template <typename V>
struct SumTraits {
    using A = typename std::conditional<std::is_floating_point<V>::value, double, long long>::type;
    using W = WideInt32<V>;
    __device__ static __forceinline__ A identity() { return (A)0; }
    __device__ static __forceinline__ W pre(V v) { return (W)v; }
    __device__ static __forceinline__ W tile(W a, W b) { return jl::add(a, b); }
    __device__ static __forceinline__ A lift(W v) { return (A)v; }
    __device__ static __forceinline__ A comb(A a, A b) { return jl::add(a, b); }
};
template <typename V>
struct ProdTraits {
    using A = typename std::conditional<std::is_floating_point<V>::value, double, long long>::type;
    using W = WideInt32<V>;
    __device__ static __forceinline__ A identity() { return (A)1; }
    __device__ static __forceinline__ W pre(V v) { return (W)v; }
    __device__ static __forceinline__ W tile(W a, W b) { return jl::mul(a, b); }
    __device__ static __forceinline__ A lift(W v) { return (A)v; }
    __device__ static __forceinline__ A comb(A a, A b) { return jl::mul(a, b); }
};
template <typename V>
__device__ __forceinline__ V lowest_of() {
    if constexpr (std::is_same<V, float>::value) return -__int_as_float(0x7f800000);
    else if constexpr (std::is_same<V, double>::value) return -__longlong_as_double(0x7ff0000000000000ll);
    else if constexpr (std::is_same<V, int32_t>::value) return (int32_t)0x80000000;
    else if constexpr (std::is_same<V, uint8_t>::value) return (uint8_t)0;
    else return (long long)0x8000000000000000ll;
}
template <typename V>
__device__ __forceinline__ V highest_of() {
    if constexpr (std::is_same<V, float>::value) return __int_as_float(0x7f800000);
    else if constexpr (std::is_same<V, double>::value) return __longlong_as_double(0x7ff0000000000000ll);
    else if constexpr (std::is_same<V, int32_t>::value) return (int32_t)0x7fffffff;
    else if constexpr (std::is_same<V, uint8_t>::value) return (uint8_t)0xff;
    else return (long long)0x7fffffffffffffffll;
}
template <typename V>
struct MaxTraits {  // Julia max: NaN-propagating, +0.0 > -0.0; -Inf is a true identity under those rules
    using A = V;
    using W = V;
    __device__ static __forceinline__ A identity() { return lowest_of<V>(); }
    __device__ static __forceinline__ W pre(V v) { return v; }
    __device__ static __forceinline__ V tile(V a, V b) { return jl::max(a, b); }
    __device__ static __forceinline__ A lift(V v) { return v; }
    __device__ static __forceinline__ A comb(A a, A b) { return jl::max(a, b); }
};
template <typename V>
struct MinTraits {
    using A = V;
    using W = V;
    __device__ static __forceinline__ A identity() { return highest_of<V>(); }
    __device__ static __forceinline__ W pre(V v) { return v; }
    __device__ static __forceinline__ V tile(V a, V b) { return jl::min(a, b); }
    __device__ static __forceinline__ A lift(V v) { return v; }
    __device__ static __forceinline__ A comb(A a, A b) { return jl::min(a, b); }
};
// extrema(localpart) in ONE pass (reference src/mapreduce.jl:124-131): the accumulator is the (min, max) pair
template <typename T>
struct Pair {
    T lo, hi;
};
template <typename T>
struct ExtremaTraits {
    using A = Pair<T>;
    using W = Pair<T>;
    __device__ static __forceinline__ A identity() { return A{highest_of<T>(), lowest_of<T>()}; }
    __device__ static __forceinline__ W pre(W v) { return v; }
    __device__ static __forceinline__ A tile(A a, A b) { return A{jl::min(a.lo, b.lo), jl::max(a.hi, b.hi)}; }
    __device__ static __forceinline__ A lift(A v) { return v; }
    __device__ static __forceinline__ A comb(A a, A b) { return tile(a, b); }
};
template <typename T>
struct ExtMapF {
    using V = Pair<T>;
    T p;
    __device__ __forceinline__ V operator()(T x) const { return V{x, x}; }
};
struct CountTraits {  // V = int (0/1) ; all / any / count all reduce to "number of trues"
    using A = long long;
    using W = int;
    __device__ static __forceinline__ A identity() { return 0; }
    __device__ static __forceinline__ W pre(int v) { return v; }
    __device__ static __forceinline__ int tile(int a, int b) { return a + b; }
    __device__ static __forceinline__ A lift(int v) { return (A)v; }
    __device__ static __forceinline__ A comb(A a, A b) { return a + b; }
};

// ---- map functors: T -> V -----------------------------------------------------------------------
// Int32 -x for the reduce kernels: the same bits as jl::neg, written as a 64-bit negate truncated to 32 bits.  Given jl::neg, ptxas
// (CUDA 12.9, sm_90a) folds the 32-bit negations into the operands of a three-input VIMNMX3 and drops one of them, so that
// maximum(-, d) of Int32 picked the wrong element; it leaves this form alone.  That is how this ptxas schedules it, not a guarantee:
// tests/test_gpu_reduce_exact.py runs Int32 max / min with -x through every reduce kernel and catches a toolkit that folds it again.
__device__ __forceinline__ int32_t neg_for_minmax(int32_t a) {
    int32_t r;
    asm("{.reg .s64 t; cvt.s64.s32 t, %1; neg.s64 t, t; cvt.u32.u64 %0, t;}" : "=r"(r) : "r"(a));
    return r;
}
template <typename T, int FN>
struct MapF {
    using V = T;
    T p;
    __device__ __forceinline__ V operator()(T x) const {
        if constexpr (FN == DAB_MAP_ABS) return jl::abs(x);
        else if constexpr (FN == DAB_MAP_ABS2) return jl::mul(x, x);
        else if constexpr (FN == DAB_MAP_NEG && std::is_same<T, int32_t>::value) return neg_for_minmax(x);
        else if constexpr (FN == DAB_MAP_NEG) return jl::neg(x);
        else return x;
    }
};
template <typename T, int FN>
struct PredF {
    using V = int;
    T p;
    __device__ __forceinline__ V operator()(T x) const {
        if constexpr (FN == DAB_MAP_EQ) return x == p;
        else if constexpr (FN == DAB_MAP_NE) return x != p;
        else if constexpr (FN == DAB_MAP_LT) return x < p;
        else if constexpr (FN == DAB_MAP_LE) return x <= p;
        else if constexpr (FN == DAB_MAP_GT) return x > p;
        else if constexpr (FN == DAB_MAP_GE) return x >= p;
        else if constexpr (FN == DAB_MAP_ISNAN) return x != x;
        else return x != (T)0;  // NONZERO / identity on Bool
    }
};

// ---- one 16-byte vector of mapped values folded into a widened accumulator ----------------------------------------------------
// The kernels' register tree works in the element type.  When the tile type is wider (Int32 sums and products) they fold each
// value straight into the Int64 accumulator instead: integer results do not depend on the grouping, and the chain keeps one Int64
// live instead of one per element.
template <typename R, typename T, typename Map>
__device__ __forceinline__ typename R::A fold_into(typename R::A acc, const Pack<T>& p, const Map& map) {
#pragma unroll
    for (int k = 0; k < 16 / (int)sizeof(T); ++k) acc = R::comb(acc, R::lift(R::pre(map(p.v[k]))));
    return acc;
}

// ---- shuffles for 4- and 8-byte accumulators -------------------------------------------------------
template <typename A>
__device__ __forceinline__ A shfl_down(A v, int d) {
    if constexpr (sizeof(A) == 16) {
        int w[4];
        memcpy(w, &v, 16);
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = __shfl_down_sync(0xffffffffu, w[k], d);
        A r;
        memcpy(&r, w, 16);
        return r;
    } else if constexpr (sizeof(A) == 8) {
        long long x;
        memcpy(&x, &v, 8);
        int lo = __shfl_down_sync(0xffffffffu, (int)(x & 0xffffffffll), d);
        int hi = __shfl_down_sync(0xffffffffu, (int)(x >> 32), d);
        x = ((long long)hi << 32) | (unsigned int)lo;
        A r;
        memcpy(&r, &x, 8);
        return r;
    } else if constexpr (sizeof(A) == 4) {
        int x;
        memcpy(&x, &v, 4);
        x = __shfl_down_sync(0xffffffffu, x, d);
        A r;
        memcpy(&r, &x, 4);
        return r;
    } else {
        int x = (int)v;
        x = __shfl_down_sync(0xffffffffu, x, d);
        return (A)x;
    }
}

template <typename R>
__device__ __forceinline__ typename R::A block_reduce(typename R::A acc, typename R::A* smem) {
    using A = typename R::A;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc = R::comb(acc, shfl_down<A>(acc, d));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();  // smem may still be read from a previous call
    if (lane == 0) smem[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < (RD_THREADS / 32) ? smem[lane] : R::identity();
#pragma unroll
        for (int d = 4; d > 0; d >>= 1) acc = R::comb(acc, shfl_down<A>(acc, d));
    }
    return acc;  // valid in thread 0
}

// ---- two-level "last one out" combine of the flat-grid kernels: deterministic, no second launch ---------------------------------
//  level 1: CTAs form groups of RD_THREADS; the last CTA of a group to finish folds the group's partials (one per thread);
//  level 2: the last group to finish folds the <= DAB_MAX_REDUCE_BLOCKS / RD_THREADS group partials.
// partials is ctx->block_partials: DAB_MAX_REDUCE_BLOCKS CTA partials, then the group partials.  counter is ctx->counter: [0] counts
// the groups, [1 + g] the CTAs of group g; the last CTA zeroes them again for the next launch on the stream.  acc is this CTA's
// block_reduce result (valid in thread 0); smem and is_last are the kernel's shared scratch (a __shared__ flag declared here instead
// changes the SASS of every caller).  Returns true in the last CTA only, where thread 0 holds the combined value in fin.
template <typename R>
__device__ __forceinline__ bool last_cta_out(typename R::A acc, typename R::A* partials, unsigned int* counter, typename R::A* smem, bool& is_last,
                                             typename R::A& fin) {
    using A = typename R::A;
    A* gpartials = partials + DAB_MAX_REDUCE_BLOCKS;
    const unsigned int ngroups = (gridDim.x + RD_THREADS - 1) / RD_THREADS;
    const unsigned int g = blockIdx.x / RD_THREADS;
    const unsigned int gsize = (g == ngroups - 1) ? gridDim.x - g * RD_THREADS : RD_THREADS;
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = acc;
        __threadfence();
        const unsigned int ticket = atomicAdd(counter + 1 + g, 1u);
        is_last = (ticket == gsize - 1);
    }
    __syncthreads();
    if (!is_last) return false;
    __threadfence();
    A v = threadIdx.x < gsize ? partials[(size_t)g * RD_THREADS + threadIdx.x] : R::identity();
    v = block_reduce<R>(v, smem);
    if (threadIdx.x == 0) {
        counter[1 + g] = 0;
        gpartials[g] = v;
        __threadfence();
        const unsigned int ticket = atomicAdd(counter, 1u);
        is_last = (ticket == ngroups - 1);
    }
    __syncthreads();
    if (!is_last) return false;
    __threadfence();
    A f = R::identity();
    for (unsigned int i = threadIdx.x; i < ngroups; i += RD_THREADS) f = R::comb(f, gpartials[i]);
    fin = block_reduce<R>(f, smem);
    if (threadIdx.x == 0) *counter = 0;
    return true;
}

// ---- complex element types: Cplx<T> (ComplexF32 / ComplexF64) -------------------------------------------------------------------
template <typename Z>
struct is_cplx : std::false_type {};
template <typename T>
struct is_cplx<Cplx<T>> : std::true_type {};

// Julia's complex + is componentwise; * is (ac - bd, ad + bc) with every operation rounded separately (never contracted).
template <typename T>
__device__ __forceinline__ Cplx<T> cadd(Cplx<T> a, Cplx<T> b) { return {jl::add(a.re, b.re), jl::add(a.im, b.im)}; }
template <typename T>
__device__ __forceinline__ Cplx<T> cmul(Cplx<T> a, Cplx<T> b) {
    return {jl::sub(jl::mul(a.re, b.re), jl::mul(a.im, b.im)), jl::add(jl::mul(a.re, b.im), jl::mul(a.im, b.re))};
}
template <typename T>
__device__ __forceinline__ Cplx<double> cwiden(Cplx<T> v) { return {(double)v.re, (double)v.im}; }

// sum: each component added in T inside a tile step (like the real kernel's register tree), carried in fp64
template <typename T>
struct CSumTraits {
    using A = Cplx<double>;
    using W = Cplx<T>;
    __device__ static __forceinline__ A identity() { return {0.0, 0.0}; }
    __device__ static __forceinline__ W pre(W v) { return v; }
    __device__ static __forceinline__ W tile(W a, W b) { return cadd(a, b); }
    __device__ static __forceinline__ A lift(W v) { return cwiden(v); }
    __device__ static __forceinline__ A comb(A a, A b) { return cadd(a, b); }
};
// product: every value widened to the complex fp64 carrier first, rounded once to T at the end
template <typename T>
struct CProdTraits {
    using A = Cplx<double>;
    using W = Cplx<double>;
    __device__ static __forceinline__ A identity() { return {1.0, 0.0}; }
    __device__ static __forceinline__ W pre(Cplx<T> v) { return cwiden(v); }
    __device__ static __forceinline__ W tile(W a, W b) { return cmul(a, b); }
    __device__ static __forceinline__ A lift(W v) { return v; }
    __device__ static __forceinline__ A comb(A a, A b) { return cmul(a, b); }
};

// abs(z) = hypot(re, im): Float32 through exact fp64 squares (one rounding for the sum, one for the root, one back to Float32), Inf when
// either component is infinite even if the other is NaN; Float64 with CUDA's hypot (<= 2 ulp, no intermediate overflow, same Inf rule)
__device__ __forceinline__ float cabs(Cplx<float> z) {
    if (isinf(z.re) || isinf(z.im)) return __int_as_float(0x7f800000);  // hypot(Inf, NaN) = Inf, as Julia's hypot
    const double x = z.re, y = z.im;
    return (float)__dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
}
__device__ __forceinline__ double cabs(Cplx<double> z) { return hypot(z.re, z.im); }

template <typename T, int FN>
struct CMapF {  // Complex{T} -> Complex{T} (identity, -z) or T (abs, abs2)
    using V = typename std::conditional<FN == DAB_MAP_ABS || FN == DAB_MAP_ABS2, T, Cplx<T>>::type;
    T p;
    __device__ __forceinline__ V operator()(Cplx<T> z) const {
        if constexpr (FN == DAB_MAP_ABS) return cabs(z);
        else if constexpr (FN == DAB_MAP_ABS2) return jl::add(jl::mul(z.re, z.re), jl::mul(z.im, z.im));
        else if constexpr (FN == DAB_MAP_NEG) return Cplx<T>{jl::neg(z.re), jl::neg(z.im)};
        else return z;
    }
};
template <typename T, int FN>
struct CPredF {  // Complex{T} -> Bool: !iszero(z), isnan(z)
    using V = int;
    T p;
    __device__ __forceinline__ V operator()(Cplx<T> z) const {
        if constexpr (FN == DAB_MAP_ISNAN) return (z.re != z.re) || (z.im != z.im);
        else return (z.re != (T)0) || (z.im != (T)0);  // NONZERO
    }
};

// ---- Float16 element type: Half ------------------------------------------------------------------------------------------------------
// Each value is widened to Float32 (exact) as it leaves the 16-byte vector; the map, the tile tree and the traits then work in Float32
// (SumTraits<float> etc.: fp32 inside a tile step, fp64 carrier), and the result is rounded once to Float16.  abs2 rounds x*x to
// Float16 first, as Julia's Float16 * does.
template <int FN>
struct HMapF {
    using V = float;
    Half p;
    __device__ __forceinline__ V operator()(Half h) const {
        const float x = (float)h;
        if constexpr (FN == DAB_MAP_ABS) return fabsf(x);
        else if constexpr (FN == DAB_MAP_ABS2) return (float)Half(jl::mul(x, x));   // x*x is exact in Float32: one rounding
        else if constexpr (FN == DAB_MAP_NEG) return -x;
        else return x;
    }
};
template <int FN>
struct HPredF {  // Float16 -> Bool, compared in Float32 (exact for Float16 operands)
    using V = int;
    Half p;
    __device__ __forceinline__ V operator()(Half h) const { return PredF<float, FN>{(float)p}((float)h); }
};

}  // namespace
