// dab_findminmax.cu -- K20: findmax / findmin / argmax / argmin of a chunk as index-carrying streaming sm_90a kernels.
//
// Replaces Base's generic findmax(f, A) / findmin(f, A) (_findmax: mapfoldl over pairs(A), one scalar getindex per element on a DArray)
// and findminmax!(f, op, Rval, Rind, A) (the dims form) on one localpart.
//
// Order.  Julia replaces the current best (v, i) of findmax by a later (x, k) when isless(v, x), and that of findmin when isgreater(v, x).
// Both make NaN the winner (the first NaN is kept) and keep the earlier index on ties; findmax prefers +0.0 to -0.0 and findmin -0.0 to
// +0.0.  So the result is the maximal element under "larger order key, then smaller linear index", where the order key is
// SortKey<T>::enc of the mapped value (dab_sort_key.cuh: Julia's isless order), every NaN canonicalised to the top key, and for findmin
// the non-NaN keys reversed.  That comparison is associative and commutative: threads, CTAs, splits and chunks combine in any order and
// give Julia's answer.
//
// Roofline: HBM, sizeof(T) bytes read per element (the whole-chunk form); the dims form also writes sizeof(T) + 8 bytes per output.
//   * dab_findminmax: the flat grid of reduce_kernel (32 KiB tiles, four 16-byte evict-first loads in flight per thread).  Each thread
//     walks its tiles in DESCENDING index order, so "key >= best" keeps the smaller index on ties with one compare per element.  Warp
//     shuffles, a CTA tree, then the self-resetting two-level last-CTA-out ticket combine.  The last CTA re-reads x[idx] and applies the
//     map, so the returned value is the element itself (a NaN keeps its payload).
//   * dab_findminmax_dim: (inner, red, outer) as in dab_reducedim.cu; a sub-warp group per contiguous run (inner == 1) or a thread per
//     output walking red in ascending order (inner > 1; VPT outputs per thread with 16-byte loads when they form whole aligned vectors); red is split when there are too few outputs to fill the GPU, and the splits'
//     (value, index) pairs are folded by a second small kernel.  Indices leave as 1-based GLOBAL linear indices of the DArray.
#include <type_traits>

#include "dab_reduce_traits.cuh"
#include "dab_sort_key.cuh"

namespace {

constexpr unsigned long long FM_NONE = ~0ull;  // "no element yet": loses every tie against a real index

template <typename T> struct FmEnc;
template <> struct FmEnc<float> { using S = SortKey<float>; };
template <> struct FmEnc<double> { using S = SortKey<double>; };
template <> struct FmEnc<int32_t> { using S = SortKey<int32_t>; };
template <> struct FmEnc<long long> { using S = SortKey<int64_t>; };

template <typename T> struct FmKeyT { using U = typename FmEnc<T>::S::U; };
template <> struct FmKeyT<uint8_t> { using U = uint32_t; };
template <typename T> using FmKey = typename FmKeyT<T>::U;

// The order key of a mapped value: a larger key is the better element for both functions.
template <typename T, bool MIN>
__host__ __device__ __forceinline__ FmKey<T> order_key(T v) {
    if constexpr (std::is_same<T, uint8_t>::value) {  // Bool: false < true
        const uint32_t k = v ? 1u : 0u;
        return MIN ? ~k : k;
    } else {
        using S = typename FmEnc<T>::S;
        using U = typename S::U;
        U bits;
        memcpy(&bits, &v, sizeof(U));
        const U k = S::enc(bits);
        if constexpr (std::is_floating_point<T>::value) {
            if (v != v) return ~(U)0;                 // every NaN is the top key, for findmax and findmin alike
            return MIN ? (U)(~k - (U)1) : k;           // reversed for findmin, strictly below the NaN key (enc(-Inf) == 0)
        } else {
            return MIN ? (U)~k : k;
        }
    }
}

// Strict in the index: of two entries with equal key and index (index inputs that carry one index twice) the accumulator keeps the one
// it holds, so a walk or fold in position order keeps the earlier one.
template <typename U>
__host__ __device__ __forceinline__ bool fm_better(U ka, unsigned long long ia, U kb, unsigned long long ib) {
    return ka > kb || (ka == kb && ia < ib);
}

// (key, index) accumulator of the whole-chunk kernel, with the shuffle and CTA tree of dab_reduce_traits.cuh
template <typename U>
struct FmBest {
    U key;
    unsigned long long idx;
};
template <typename U>
struct FmTraits {
    using A = FmBest<U>;
    __device__ static __forceinline__ A identity() { return A{(U)0, FM_NONE}; }
    __device__ static __forceinline__ A comb(A a, A b) { return fm_better(b.key, b.idx, a.key, a.idx) ? b : a; }
};

// Bool: abs and abs2 are the identity (abs(b) === b, b * b === b).  Float abs clears the sign bit, as Julia's abs_float does: an FP
// instruction would turn a NaN into the canonical NaN and lose the payload.  abs2 is x * x (MapF), whose NaN is the GPU's canonical one.
template <typename T, int FN>
struct FmMap {
    using F = MapF<T, std::is_same<T, uint8_t>::value ? DAB_MAP_ID : FN>;
    __device__ __forceinline__ T operator()(T x) const {
        if constexpr (std::is_same<T, uint8_t>::value) {
            return x;
        } else if constexpr (FN == DAB_MAP_ABS && std::is_same<T, float>::value) {
            return __int_as_float(__float_as_int(x) & 0x7fffffff);
        } else if constexpr (FN == DAB_MAP_ABS && std::is_same<T, double>::value) {
            return __longlong_as_double(__double_as_longlong(x) & 0x7fffffffffffffffll);
        } else {
            return F{(T)0}(x);
        }
    }
};

// ---- whole chunk -----------------------------------------------------------------------------------------------------------------
// 48 registers (5 CTAs of 256 threads per SM): the per-element (key, 64-bit index) update of four 16-byte vectors does not fit the 32
// of reduce_kernel without spilling for 8-byte T.  1280 threads per SM with four 16-byte loads each in flight cover HBM latency.
template <typename T, int FN, bool MIN>
__global__ void __launch_bounds__(RD_THREADS, 5) findminmax_kernel(const T* __restrict__ x, size_t n, size_t head, FmBest<FmKey<T>>* partials,
                                                                  unsigned int* counter, void* out, int tiles_per_cta) {
    using U = FmKey<T>;
    using R = FmTraits<U>;
    using A = FmBest<U>;
    constexpr int VPT = 16 / sizeof(T);
    __shared__ A smem[RD_THREADS / 32];
    __shared__ bool is_last;
    const FmMap<T, FN> map;

    const size_t nvec = (n - head) / VPT;
    const int4* xv = reinterpret_cast<const int4*>(x + head);
    constexpr size_t TILE = (size_t)RD_THREADS * RD_UNROLL;
    const size_t ntiles = nvec / TILE;
    U bk = 0;
    unsigned long long bi = FM_NONE;
    const size_t t_beg = (size_t)blockIdx.x * (size_t)tiles_per_cta;
    size_t t_end = t_beg + (size_t)tiles_per_cta;
    if (t_end > ntiles) t_end = ntiles;
    // descending walk: of two equal keys the one seen later has the smaller index, so ">=" keeps Julia's earlier index (and replaces the
    // identity's FM_NONE even for key 0)
#pragma unroll 1
    for (size_t t = t_end; t > t_beg;) {
        --t;
        const size_t base = t * TILE + threadIdx.x;
        int4 r[RD_UNROLL];
#pragma unroll
        for (int u = 0; u < RD_UNROLL; ++u) r[u] = ld_stream(xv + base + (size_t)u * RD_THREADS);
#pragma unroll
        for (int u = RD_UNROLL - 1; u >= 0; --u) {
            const Pack<T> p = as_pack<T>(r[u]);
            const unsigned long long i0 = head + (base + (size_t)u * RD_THREADS) * VPT;
#pragma unroll
            for (int k = VPT - 1; k >= 0; --k) {
                const U key = order_key<T, MIN>(map(p.v[k]));
                if (key >= bk) {
                    bk = key;
                    bi = i0 + k;
                }
            }
        }
    }
    A acc{bk, bi};
    if (blockIdx.x == gridDim.x - 1) {  // remainder vectors, unaligned head, tail: any order, full comparison
        for (size_t i = ntiles * TILE + threadIdx.x; i < nvec; i += RD_THREADS) {
            const Pack<T> p = as_pack<T>(ld_stream(xv + i));
#pragma unroll
            for (int k = 0; k < VPT; ++k) acc = R::comb(acc, A{order_key<T, MIN>(map(p.v[k])), head + i * VPT + k});
        }
        for (size_t i = threadIdx.x; i < head; i += RD_THREADS) acc = R::comb(acc, A{order_key<T, MIN>(map(x[i])), i});
        for (size_t i = head + nvec * VPT + threadIdx.x; i < n; i += RD_THREADS) acc = R::comb(acc, A{order_key<T, MIN>(map(x[i])), i});
    }
    acc = block_reduce<R>(acc, smem);
    // the ticket counters and partials of reduce_kernel (same stream, so never concurrent)
    A fin;
    if (!last_cta_out<R>(acc, partials, counter, smem, is_last, fin)) return;
    if (threadIdx.x == 0) {
        const T val = map(x[fin.idx]);  // the element itself, mapped: NaN payloads survive
        memset(out, 0, 16);
        memcpy(out, &val, sizeof(T));
        const long long li = (long long)fin.idx;
        memcpy((char*)out + 8, &li, 8);
    }
}

template <typename T, int FN, bool MIN>
int32_t launch_findminmax(dab_ctx* ctx, const T* x, size_t n, void* out) {
    const FlatGrid fg = flat_grid(x, n);
    findminmax_kernel<T, FN, MIN><<<(unsigned)fg.grid, RD_THREADS, 0, ctx->stream>>>(x, n, fg.head, (FmBest<FmKey<T>>*)ctx->block_partials,
                                                                                      ctx->counter, out, fg.tiles_per_cta);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// ---- dims ------------------------------------------------------------------------------------------------------------------------
// Chunk-local linear position -> 1-based global linear index of the DArray: column-major unravel in the chunk's dims, plus the chunk's
// 0-based global offsets, ravel in the global dims.  Applied once per output.  nd == 0: the position itself (plus one).
struct FmGlobal {
    int nd;
    long long cdims[8], off[8], gdims[8];
    __device__ __forceinline__ long long operator()(unsigned long long pos) const {
        unsigned long long g = 0, stride = 1;
        if (nd == 0) return (long long)pos + 1;
#pragma unroll
        for (int d = 0; d < 8; ++d) {  // static indices: the parameter arrays stay in the constant bank, no local copy
            if (d >= nd) break;
            const unsigned long long c = pos % (unsigned long long)cdims[d];
            pos /= (unsigned long long)cdims[d];
            g += (c + (unsigned long long)off[d]) * stride;
            stride *= (unsigned long long)gdims[d];
        }
        return (long long)g + 1;
    }
};

// running best of one lane / thread: key, raw index (chunk-local position, or the 1-based global index read from idx_in), mapped value
template <typename T>
struct FmRun {
    FmKey<T> key;
    unsigned long long idx;
    T val;
};
// an index input of -1 (FM_NONE) marks "no element": the slab of a chunk that is empty along the reduced dims
template <typename T, bool MIN, bool IDX>
__device__ __forceinline__ void fm_take(FmRun<T>& b, T v, unsigned long long idx) {
    if (IDX && idx == FM_NONE) return;
    const FmKey<T> key = order_key<T, MIN>(v);
    if (fm_better(key, idx, b.key, b.idx)) b = FmRun<T>{key, idx, v};
}
template <typename T>
__device__ __forceinline__ FmRun<T> fm_shfl_down(const FmRun<T>& b, int d) {
    FmRun<T> r;
    r.key = shfl_down(b.key, d);
    r.idx = shfl_down(b.idx, d);
    r.val = shfl_down(b.val, d);
    return r;
}

// the result of one (run, split): the final output, or a partial for fmdim_finish_kernel
template <typename T, bool IDX>
__device__ __forceinline__ void fm_store(const FmRun<T>& b, size_t k, size_t part, int nsplit, const FmGlobal& gl, T* pv, unsigned long long* pi,
                                         T* out_v, long long* out_i) {
    if (nsplit == 1) {
        out_v[k] = b.val;
        out_i[k] = IDX ? (long long)b.idx : gl(b.idx);
    } else {
        pv[part] = b.val;
        pi[part] = b.idx;
    }
}

// inner == 1: a group of G lanes per contiguous run of `red` elements (split in nsplit pieces), 4 loads in flight per lane
template <typename T, int FN, bool MIN, bool IDX, int G>
__global__ void __launch_bounds__(RD_THREADS) fmdim_lead_kernel(const T* __restrict__ x, const long long* __restrict__ idx_in, size_t red,
                                                                size_t outer, int nsplit, FmGlobal gl, T* pv, unsigned long long* pi,
                                                                T* __restrict__ out_v, long long* __restrict__ out_i) {
    constexpr int GROUPS = RD_THREADS / G;
    const FmMap<T, FN> map;
    const int lane = threadIdx.x % G;
    const size_t work = outer * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
#pragma unroll 1
    for (size_t w0 = (size_t)blockIdx.x * GROUPS; w0 < work; w0 += (size_t)gridDim.x * GROUPS) {  // uniform over the CTA: full-mask shuffles
        const size_t w = w0 + threadIdx.x / G;
        const bool active = w < work;
        const size_t seg = active ? w / nsplit : 0, sp = active ? w % nsplit : 0;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        if (!active) hi = lo;
        const size_t base = seg * red;
        FmRun<T> b{(FmKey<T>)0, FM_NONE, (T)0};
        size_t r = lo + lane;
        for (; r + 3 * G < hi; r += 4 * G) {
            T v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = __ldcs(x + base + r + (size_t)u * G);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const size_t pos = base + r + (size_t)u * G;
                fm_take<T, MIN, IDX>(b, map(v[u]), IDX ? (unsigned long long)idx_in[pos] : pos);
            }
        }
        for (; r < hi; r += G) fm_take<T, MIN, IDX>(b, map(__ldcs(x + base + r)), IDX ? (unsigned long long)idx_in[base + r] : base + r);
#pragma unroll
        for (int d = G / 2; d > 0; d >>= 1) {
            const FmRun<T> o = fm_shfl_down(b, d);
            if (fm_better(o.key, o.idx, b.key, b.idx)) b = o;
        }
        if (active && lane == 0) fm_store<T, IDX>(b, seg, seg * (size_t)nsplit + sp, nsplit, gl, pv, pi, out_v, out_i);
    }
}

// inner > 1: a thread per output k = i + inner*o (coalesced along i), walking its split of red in ascending order, 8 loads in flight
template <typename T, int FN, bool MIN, bool IDX>
__global__ void __launch_bounds__(RD_THREADS) fmdim_strided_kernel(const T* __restrict__ x, const long long* __restrict__ idx_in, size_t inner,
                                                                   size_t red, size_t outer, int nsplit, FmGlobal gl, T* pv,
                                                                   unsigned long long* pi, T* __restrict__ out_v, long long* __restrict__ out_i) {
    constexpr int UNROLL = 8;
    const FmMap<T, FN> map;
    const size_t nout = inner * outer;
    const size_t kblocks = (nout + RD_THREADS - 1) / RD_THREADS;
    const size_t work = kblocks * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
#pragma unroll 1
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const size_t kb = w % kblocks, sp = w / kblocks;
        const size_t k = kb * RD_THREADS + threadIdx.x;
        if (k >= nout) continue;
        const size_t o = k / inner, i = k - o * inner;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        const size_t base = i + inner * (o * red);
        FmRun<T> b{(FmKey<T>)0, FM_NONE, (T)0};
        size_t r = lo;
        for (; r + UNROLL <= hi; r += UNROLL) {
            T v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = __ldcs(x + base + (r + u) * inner);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const size_t pos = base + (r + u) * inner;
                fm_take<T, MIN, IDX>(b, map(v[u]), IDX ? (unsigned long long)idx_in[pos] : pos);
            }
        }
        for (; r < hi; ++r) {
            const size_t pos = base + r * inner;
            fm_take<T, MIN, IDX>(b, map(__ldcs(x + pos)), IDX ? (unsigned long long)idx_in[pos] : pos);
        }
        fm_store<T, IDX>(b, k, sp * nout + k, nsplit, gl, pv, pi, out_v, out_i);
    }
}

// inner > 1, 16-byte: each thread owns VPT consecutive outputs along i and walks its split of red with 16-byte loads (512 bytes per warp
// load, four in flight).  Needs inner % VPT == 0, a 16-byte aligned base and 4- or 8-byte T; no index input.
template <typename T, int FN, bool MIN>
__global__ void __launch_bounds__(RD_THREADS) fmdim_strided_vec_kernel(const T* __restrict__ x, size_t inner, size_t red, size_t outer, int nsplit,
                                                                       FmGlobal gl, T* pv, unsigned long long* pi, T* __restrict__ out_v,
                                                                       long long* __restrict__ out_i) {
    constexpr int VPT = 16 / sizeof(T);
    constexpr int UNROLL = 4;
    const FmMap<T, FN> map;
    const size_t nout = inner * outer;
    const size_t nvout = nout / VPT, ivec = inner / VPT;
    const size_t kblocks = (nvout + RD_THREADS - 1) / RD_THREADS;
    const size_t work = kblocks * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
#pragma unroll 1
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const size_t kb = w % kblocks, sp = w / kblocks;
        const size_t kv = kb * RD_THREADS + threadIdx.x;
        if (kv >= nvout) continue;
        const size_t o = kv / ivec, iv = kv - o * ivec;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        const size_t base = iv * VPT + inner * (o * red);  // element position of (i = iv * VPT, r = 0, o)
        const int4* p = reinterpret_cast<const int4*>(x + base);
        FmRun<T> b[VPT];
#pragma unroll
        for (int k = 0; k < VPT; ++k) b[k] = FmRun<T>{(FmKey<T>)0, FM_NONE, (T)0};
        size_t r = lo;
        for (; r + UNROLL <= hi; r += UNROLL) {
            int4 v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = ld_stream(p + (r + u) * ivec);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const Pack<T> pk = as_pack<T>(v[u]);
#pragma unroll
                for (int k = 0; k < VPT; ++k) fm_take<T, MIN, false>(b[k], map(pk.v[k]), base + (r + u) * inner + k);
            }
        }
        for (; r < hi; ++r) {
            const Pack<T> pk = as_pack<T>(ld_stream(p + r * ivec));
#pragma unroll
            for (int k = 0; k < VPT; ++k) fm_take<T, MIN, false>(b[k], map(pk.v[k]), base + r * inner + k);
        }
        const size_t k0 = kv * VPT;
#pragma unroll
        for (int k = 0; k < VPT; ++k) fm_store<T, false>(b[k], k0 + k, sp * nout + k0 + k, nsplit, gl, pv, pi, out_v, out_i);
    }
}

// fold of the split partials: thread per output, (value, index) pairs combined under the same order; a split that held no element keeps
// FM_NONE and is skipped
template <typename T, bool MIN, bool IDX>
__global__ void __launch_bounds__(RD_THREADS) fmdim_finish_kernel(const T* __restrict__ pv, const unsigned long long* __restrict__ pi, size_t nout,
                                                                  int nsplit, size_t stride_out, size_t stride_split, FmGlobal gl,
                                                                  T* __restrict__ out_v, long long* __restrict__ out_i) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < nout; k += stride) {
        FmRun<T> b{(FmKey<T>)0, FM_NONE, (T)0};
        for (int s = 0; s < nsplit; ++s) {
            const size_t q = k * stride_out + (size_t)s * stride_split;
            fm_take<T, MIN, true>(b, pv[q], pi[q]);
        }
        out_v[k] = b.val;
        out_i[k] = IDX ? (long long)b.idx : gl(b.idx);
    }
}

// one output from the whole-chunk slot (a dims reduction that is one run: inner == outer == 1)
template <typename T>
__global__ void fm_slot_to_out_kernel(const void* __restrict__ slot, FmGlobal gl, T* __restrict__ out_v, long long* __restrict__ out_i) {
    T v;
    long long i;
    memcpy(&v, slot, sizeof(T));
    memcpy(&i, (const char*)slot + 8, 8);
    *out_v = v;
    *out_i = gl((unsigned long long)i);
}

template <typename T, int FN, bool MIN, bool IDX>
int32_t launch_fmdim(dab_ctx* ctx, const T* x, const long long* idx_in, size_t inner, size_t red, size_t outer, const FmGlobal& gl, T* out_v,
                     long long* out_i) {
    const size_t nout = inner * outer;
    const size_t target_ctas = (size_t)ctx->sm_count * 8;
    if (!IDX && inner == 1 && outer == 1 && red >= (1u << 16)) {  // one long run: the whole-chunk kernel, then the slot to the outputs
        int32_t st = launch_findminmax<T, FN, MIN>(ctx, x, red, ctx->result_slot);
        if (st != DAB_OK) return st;
        fm_slot_to_out_kernel<T><<<1, 1, 0, ctx->stream>>>(ctx->result_slot, gl, out_v, out_i);
        DAB_LAUNCHED(ctx);
        return DAB_OK;
    }
    // the 16-byte strided kernel: whole vectors of outputs, an aligned base, 4- or 8-byte T, no index input, enough vectors to fill the GPU
    constexpr int VPT = 16 / sizeof(T);
    const bool vec = !IDX && sizeof(T) >= 4 && inner > 1 && inner % VPT == 0 && ((uintptr_t)x & 15) == 0 && nout / VPT >= 4096;
    int nsplit;
    if (inner == 1) {
        const int G = red >= 64 ? 32 : 4;
        nsplit = dim_nsplit(outer, target_ctas * (RD_THREADS / G), red / ((size_t)G * 64));  // every lane keeps >= 64 elements of its split
    } else {
        const size_t base_ctas = vec ? (nout / VPT + RD_THREADS - 1) / RD_THREADS : (nout + RD_THREADS - 1) / RD_THREADS;
        nsplit = dim_nsplit(base_ctas, 4 * target_ctas, red / 256);
    }
    T* pv = nullptr;
    unsigned long long* pi = nullptr;
    if (nsplit > 1) {
        const size_t parts = nout * (size_t)nsplit;
        int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, parts * 16, false);
        if (st != DAB_OK) return st;
        pi = (unsigned long long*)ctx->dim_scratch;
        pv = (T*)(pi + parts);
    }
    if (inner == 1) {
        if (red >= 64) {
            auto kern = fmdim_lead_kernel<T, FN, MIN, IDX, 32>;
            const int grid = dab_persistent_grid(ctx, kern, RD_THREADS, (outer * (size_t)nsplit + RD_THREADS / 32 - 1) / (RD_THREADS / 32));
            kern<<<grid, RD_THREADS, 0, ctx->stream>>>(x, idx_in, red, outer, nsplit, gl, pv, pi, out_v, out_i);
        } else {
            auto kern = fmdim_lead_kernel<T, FN, MIN, IDX, 4>;
            const int grid = dab_persistent_grid(ctx, kern, RD_THREADS, (outer * (size_t)nsplit + RD_THREADS / 4 - 1) / (RD_THREADS / 4));
            kern<<<grid, RD_THREADS, 0, ctx->stream>>>(x, idx_in, red, outer, nsplit, gl, pv, pi, out_v, out_i);
        }
    } else {
        if constexpr (!IDX && sizeof(T) >= 4) {
            if (vec) {
                auto kern = fmdim_strided_vec_kernel<T, FN, MIN>;
                const int grid = dab_persistent_grid(ctx, kern, RD_THREADS, (nout / VPT + RD_THREADS - 1) / RD_THREADS * (size_t)nsplit);
                kern<<<grid, RD_THREADS, 0, ctx->stream>>>(x, inner, red, outer, nsplit, gl, pv, pi, out_v, out_i);
            }
        }
        if (!vec) {
            auto kern = fmdim_strided_kernel<T, FN, MIN, IDX>;
            const int grid = dab_persistent_grid(ctx, kern, RD_THREADS, (nout + RD_THREADS - 1) / RD_THREADS * (size_t)nsplit);
            kern<<<grid, RD_THREADS, 0, ctx->stream>>>(x, idx_in, inner, red, outer, nsplit, gl, pv, pi, out_v, out_i);
        }
    }
    DAB_LAUNCHED(ctx);
    if (nsplit > 1) {
        const int g2 = dab_grid_for(ctx, (nout + RD_THREADS - 1) / RD_THREADS, 8);
        const size_t so = inner == 1 ? (size_t)nsplit : 1, ss = inner == 1 ? 1 : nout;
        fmdim_finish_kernel<T, MIN, IDX><<<g2, RD_THREADS, 0, ctx->stream>>>(pv, pi, nout, nsplit, so, ss, gl, out_v, out_i);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

// (map, which) dispatch; the optional Int64 index input serves the identity map only (the values it goes with are already mapped)
template <typename T>
int32_t fm_dispatch(dab_ctx* ctx, int32_t which, int32_t map, const void* x, size_t n, void* out) {
    const T* p = (const T*)x;
    const bool mn = which == DAB_FINDMIN;
    if constexpr (!std::is_same<T, uint8_t>::value) {
        if (map == DAB_MAP_ABS) return mn ? launch_findminmax<T, DAB_MAP_ABS, true>(ctx, p, n, out) : launch_findminmax<T, DAB_MAP_ABS, false>(ctx, p, n, out);
        if (map == DAB_MAP_ABS2)
            return mn ? launch_findminmax<T, DAB_MAP_ABS2, true>(ctx, p, n, out) : launch_findminmax<T, DAB_MAP_ABS2, false>(ctx, p, n, out);
    }
    return mn ? launch_findminmax<T, DAB_MAP_ID, true>(ctx, p, n, out) : launch_findminmax<T, DAB_MAP_ID, false>(ctx, p, n, out);
}

template <typename T, int FN>
int32_t fmdim_which(dab_ctx* ctx, int32_t which, const T* x, const long long* idx_in, size_t inner, size_t red, size_t outer, const FmGlobal& gl,
                    T* out_v, long long* out_i) {
    if (idx_in) {
        if constexpr (FN == DAB_MAP_ID) {
            return which == DAB_FINDMIN ? launch_fmdim<T, FN, true, true>(ctx, x, idx_in, inner, red, outer, gl, out_v, out_i)
                                        : launch_fmdim<T, FN, false, true>(ctx, x, idx_in, inner, red, outer, gl, out_v, out_i);
        } else {
            return dab_fail(ctx, DAB_ERR_ARG, "dab_findminmax_dim: an index input goes with already mapped values (map must be DAB_MAP_ID)");
        }
    }
    return which == DAB_FINDMIN ? launch_fmdim<T, FN, true, false>(ctx, x, nullptr, inner, red, outer, gl, out_v, out_i)
                                : launch_fmdim<T, FN, false, false>(ctx, x, nullptr, inner, red, outer, gl, out_v, out_i);
}

template <typename T>
int32_t fmdim_dispatch(dab_ctx* ctx, int32_t which, int32_t map, const void* x, const long long* idx_in, size_t inner, size_t red, size_t outer,
                       const FmGlobal& gl, void* out_v, long long* out_i) {
    const T* p = (const T*)x;
    T* ov = (T*)out_v;
    if constexpr (!std::is_same<T, uint8_t>::value) {
        if (map == DAB_MAP_ABS) return fmdim_which<T, DAB_MAP_ABS>(ctx, which, p, idx_in, inner, red, outer, gl, ov, out_i);
        if (map == DAB_MAP_ABS2) return fmdim_which<T, DAB_MAP_ABS2>(ctx, which, p, idx_in, inner, red, outer, gl, ov, out_i);
    }
    return fmdim_which<T, DAB_MAP_ID>(ctx, which, p, idx_in, inner, red, outer, gl, ov, out_i);
}

// the checks every entry makes before it touches the context
int32_t fm_check(int32_t dtype, int32_t which, int32_t map, const char* who) {
    if (dtype == DAB_C64 || dtype == DAB_C128)
        return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "%s: complex numbers are not ordered (isless has no complex method)", who);
    if (dtype != DAB_F32 && dtype != DAB_F64 && dtype != DAB_I32 && dtype != DAB_I64 && dtype != DAB_U8)
        return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "%s: dtype %d is not served (Float32, Float64, Int32, Int64 and Bool are)", who, dtype);
    if (which != DAB_FINDMAX && which != DAB_FINDMIN) return dab_fail(nullptr, DAB_ERR_ARG, "%s: bad which %d", who, which);
    if (map != DAB_MAP_ID && map != DAB_MAP_ABS && map != DAB_MAP_ABS2)
        return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "%s: map %d is not served (identity, abs and abs2 are)", who, map);
    return DAB_OK;
}

template <typename T, bool MIN>
void fm_combine(const unsigned char* rec, size_t count, unsigned char* out) {
    size_t best = 0;
    FmKey<T> bk = 0;
    long long bi = 0;
    for (size_t j = 0; j < count; ++j) {
        T v;
        long long i;
        memcpy(&v, rec + 16 * j, sizeof(T));
        memcpy(&i, rec + 16 * j + 8, 8);
        const FmKey<T> k = order_key<T, MIN>(v);
        if (j == 0 || fm_better(k, (unsigned long long)i, bk, (unsigned long long)bi)) {
            best = j;
            bk = k;
            bi = i;
        }
    }
    memcpy(out, rec + 16 * best, 16);
}

}  // namespace

extern "C" {

int32_t dab_findminmax(dab_ctx* ctx, int32_t dtype, int32_t which, int32_t map, const void* map_param, const void* x, size_t n, void* out_dev) {
    (void)map_param;
    int32_t st = fm_check(dtype, which, map, "dab_findminmax");
    if (st != DAB_OK) return st;
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, out_dev && x, DAB_ERR_ARG, "dab_findminmax: null pointer");
    DAB_REQUIRE(ctx, (uintptr_t)x % dab_dtype_size(dtype) == 0, DAB_ERR_ARG, "dab_findminmax: x is not aligned to its element size");
    if (n == 0) return dab_fail(ctx, DAB_ERR_EMPTY, "reducing over an empty collection is not allowed");
    switch (dtype) {
        case DAB_F32: return fm_dispatch<float>(ctx, which, map, x, n, out_dev);
        case DAB_F64: return fm_dispatch<double>(ctx, which, map, x, n, out_dev);
        case DAB_I32: return fm_dispatch<int32_t>(ctx, which, map, x, n, out_dev);
        case DAB_I64: return fm_dispatch<long long>(ctx, which, map, x, n, out_dev);
        default: return fm_dispatch<uint8_t>(ctx, which, map, x, n, out_dev);  // DAB_U8 (Bool)
    }
}

int32_t dab_findminmax_dim(dab_ctx* ctx, int32_t dtype, int32_t which, int32_t map, const void* x, const int64_t* idx_in, size_t inner,
                           size_t reduce, size_t outer, int32_t nd, const int64_t* chunk_dims, const int64_t* offsets,
                           const int64_t* global_dims, void* out_vals, int64_t* out_idx) {
    int32_t st = fm_check(dtype, which, map, "dab_findminmax_dim");
    if (st != DAB_OK) return st;
    if (nd < 0 || nd > 8 || (nd > 0 && (!chunk_dims || !offsets || !global_dims)))
        return dab_fail(nullptr, DAB_ERR_ARG, "dab_findminmax_dim: nd = %d (0..8, with all three dimension arrays)", nd);
    DAB_ENTER(ctx);
    if (inner * outer == 0) return DAB_OK;
    if (reduce == 0) return dab_fail(ctx, DAB_ERR_EMPTY, "collection slices must be non-empty");
    DAB_REQUIRE(ctx, x && out_vals && out_idx, DAB_ERR_ARG, "dab_findminmax_dim: null pointer");
    DAB_REQUIRE(ctx, (uintptr_t)x % dab_dtype_size(dtype) == 0, DAB_ERR_ARG, "dab_findminmax_dim: x is not aligned to its element size");
    FmGlobal gl;
    memset(&gl, 0, sizeof(gl));
    gl.nd = nd;
    for (int d = 0; d < nd; ++d) {
        DAB_REQUIRE(ctx, chunk_dims[d] > 0 && offsets[d] >= 0 && global_dims[d] >= offsets[d] + chunk_dims[d], DAB_ERR_ARG,
                    "dab_findminmax_dim: dimension %d does not fit its global extent", d + 1);
        gl.cdims[d] = chunk_dims[d];
        gl.off[d] = offsets[d];
        gl.gdims[d] = global_dims[d];
    }
    const long long* ii = (const long long*)idx_in;
    long long* oi = (long long*)out_idx;
    switch (dtype) {
        case DAB_F32: return fmdim_dispatch<float>(ctx, which, map, x, ii, inner, reduce, outer, gl, out_vals, oi);
        case DAB_F64: return fmdim_dispatch<double>(ctx, which, map, x, ii, inner, reduce, outer, gl, out_vals, oi);
        case DAB_I32: return fmdim_dispatch<int32_t>(ctx, which, map, x, ii, inner, reduce, outer, gl, out_vals, oi);
        case DAB_I64: return fmdim_dispatch<long long>(ctx, which, map, x, ii, inner, reduce, outer, gl, out_vals, oi);
        default: return fmdim_dispatch<uint8_t>(ctx, which, map, x, ii, inner, reduce, outer, gl, out_vals, oi);
    }
}

int32_t dab_combine_findminmax(int32_t dtype, int32_t which, const void* records, size_t count, void* out) {
    int32_t st = fm_check(dtype, which, DAB_MAP_ID, "dab_combine_findminmax");
    if (st != DAB_OK) return st;
    if (!records || !out) return dab_fail(nullptr, DAB_ERR_ARG, "dab_combine_findminmax: null pointer");
    if (count == 0) return dab_fail(nullptr, DAB_ERR_EMPTY, "reducing over an empty collection is not allowed");
    const unsigned char* r = (const unsigned char*)records;
    unsigned char* o = (unsigned char*)out;
    const bool mn = which == DAB_FINDMIN;
    switch (dtype) {
        case DAB_F32: mn ? fm_combine<float, true>(r, count, o) : fm_combine<float, false>(r, count, o); break;
        case DAB_F64: mn ? fm_combine<double, true>(r, count, o) : fm_combine<double, false>(r, count, o); break;
        case DAB_I32: mn ? fm_combine<int32_t, true>(r, count, o) : fm_combine<int32_t, false>(r, count, o); break;
        case DAB_I64: mn ? fm_combine<long long, true>(r, count, o) : fm_combine<long long, false>(r, count, o); break;
        default: mn ? fm_combine<uint8_t, true>(r, count, o) : fm_combine<uint8_t, false>(r, count, o); break;
    }
    return DAB_OK;
}

}  // extern "C"
