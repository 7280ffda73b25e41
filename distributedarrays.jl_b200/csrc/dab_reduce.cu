// dab_reduce.cu -- K4 / K7: whole-chunk mapreduce(f, op, localpart(d)) as one streaming sm_90a kernel.
//
// Replaces the per-worker Base.mapreduce / reduce / all / any / count at reference src/mapreduce.jl:23,31,100,109,118
// and the caller-side left fold reduce(op, results) at src/mapreduce.jl:26,34 (dab_combine_ordered).
//
// Roofline: HBM, 4 B/element read (sizeof(T)), output negligible.
// Design: flat grid, one CTA of 256 threads per 32 KiB of input; each thread keeps UNROLL independent 16-byte evict-first loads
// in flight, reduces the 16 values of a tile step with a register tree in the element type (Int32 sums and products instead fold
// each value, widened to Int64, straight into the accumulator), and carries the running
// value in a wide accumulator (fp64 for float sums/products, int64 for integers) -- one F2D + DADD per 16 elements, so the
// FP64 pipe is idle >90 % of the time and the result is far inside the 1e-6 tolerance.  Warp shuffle -> shared-memory
// tree -> one partial per CTA -> the LAST CTA to finish (ticket counter) folds the CTA partials in a fixed order, so the
// result is deterministic for a given (n, grid).  No atomics on data, no second launch.
//
// Fused map-store-reduce: when the reduced array is the y of a deferred dab_affine (y .= a.*x .+ b; dab_elementwise.cu) the
// same kernel reads x instead, stores y and reduces it -- 8 B/element of Float32 instead of 8 (broadcast) + 4 (reduce), and
// bit-identical to reducing the finished y (AffineStore below).
#include <type_traits>

#include <cmath>

#include "dab_reduce_traits.cuh"

namespace {

// What the reduce kernel does with each loaded value before the map.  NoStore: nothing (plain reduction of x).
struct NoStore {
    template <typename T>
    __device__ __forceinline__ void vec(Pack<T>&, size_t) const {}
    template <typename T>
    __device__ __forceinline__ T scalar(T v, size_t) const { return v; }
};
// AffineStore: the kernel consumes a deferred dab_affine -- x is the affine's input, each value becomes y = a*x + b, is stored
// to y (same index, same thread, so x == y in place is safe) and is then reduced.  The reduction sees exactly the values a
// plain reduce of the finished y would load, in the same order.
template <typename T>
struct AffineStore {
    AffineF<T> f;
    T* y;      // y[i] pairs with x[i]
    int4* yv;  // y + head as 16-byte vectors (x and y share their misalignment)
    __device__ __forceinline__ void vec(Pack<T>& p, size_t i) const {
#pragma unroll
        for (int k = 0; k < Pack<T>::N; ++k) p.v[k] = f(p.v[k]);
        st_stream(yv + i, as_int4(p));
    }
    __device__ __forceinline__ T scalar(T v, size_t i) const {
        v = f(v);
        y[i] = v;
        return v;
    }
};

// CTAs per SM the reduce kernel is compiled for: 8 (a 32-register budget) for the real element types; 6 (40 registers) for Complex{T},
// whose tile tree holds two components per value and would spill at 32; 4 (64 registers) for abs of ComplexF32, which computes hypot
// through fp64 squares.  Every choice keeps >= 1024 threads per SM, each with 4 x 16-byte loads in flight.
template <typename T, typename Map>
struct RdMinBlocks {
    static constexpr int value = !is_cplx<T>::value ? 8 : (std::is_same<Map, CMapF<float, DAB_MAP_ABS>>::value ? 4 : 6);
};

// Result slot layout (16 bytes at `out`): [0..8) the result in its result dtype, [8..16) the wide accumulator (fp64 for
// float SUM/PROD -- lets the host see the un-rounded carrier; tests use it).
template <typename T, typename Map, typename R, typename Out, typename St>
__global__ void __launch_bounds__(RD_THREADS, RdMinBlocks<T, Map>::value) reduce_kernel(const T* __restrict__ x, size_t n, size_t head, Map map,
                                                             typename R::A* __restrict__ partials, unsigned int* counter,
                                                             void* out, int finalize_mode, long long n_for_all, int tiles_per_cta,
                                                             FusedComm fc, St st) {
    using A = typename R::A;
    using W = typename R::W;
    constexpr int VPT = 16 / sizeof(T);
    __shared__ A smem[RD_THREADS / 32];
    __shared__ bool is_last;

    const size_t nvec = (n - head) / VPT;
    const int4* xv = reinterpret_cast<const int4*>(x + head);
    constexpr size_t TILE = (size_t)RD_THREADS * RD_UNROLL;
    const size_t ntiles = nvec / TILE;
    A acc = R::identity();
    // "flat" grid: CTA b owns the tiles_per_cta consecutive tiles starting at b*tiles_per_cta (fixed mapping -> deterministic
    // result); the block scheduler issues CTAs in address order, keeping the open DRAM pages a compact window (faster than a
    // persistent grid-stride loop when the kernel was designed).
    size_t t_end = ((size_t)blockIdx.x + 1) * (size_t)tiles_per_cta;
    if (t_end > ntiles) t_end = ntiles;
#pragma unroll 1
    for (size_t t = (size_t)blockIdx.x * (size_t)tiles_per_cta; t < t_end; ++t) {
        const size_t base = t * TILE + threadIdx.x;
        int4 r[RD_UNROLL];
#pragma unroll
        for (int u = 0; u < RD_UNROLL; ++u) r[u] = ld_stream(xv + base + (size_t)u * RD_THREADS);
        if constexpr (std::is_same<W, typename Map::V>::value) {
            W tv[RD_UNROLL];
#pragma unroll
            for (int u = 0; u < RD_UNROLL; ++u) {
                Pack<T> p = as_pack<T>(r[u]);
                st.vec(p, base + (size_t)u * RD_THREADS);
                W m[VPT];
#pragma unroll
                for (int k = 0; k < VPT; ++k) m[k] = map(p.v[k]);
#pragma unroll
                for (int w = VPT; w > 1; w >>= 1)  // register tree inside one 16-byte vector
#pragma unroll
                    for (int k = 0; k < w / 2; ++k) m[k] = R::tile(m[k], m[k + w / 2]);
                tv[u] = m[0];
            }
#pragma unroll
            for (int w = RD_UNROLL; w > 1; w >>= 1)
#pragma unroll
                for (int k = 0; k < w / 2; ++k) tv[k] = R::tile(tv[k], tv[k + w / 2]);
            acc = R::comb(acc, R::lift(tv[0]));
        } else {  // widened tile (Int32 sums and products)
#pragma unroll
            for (int u = 0; u < RD_UNROLL; ++u) {
                Pack<T> p = as_pack<T>(r[u]);
                st.vec(p, base + (size_t)u * RD_THREADS);
                acc = fold_into<R>(acc, p, map);
            }
        }
    }
    if (blockIdx.x == gridDim.x - 1) {  // remainder vectors, unaligned head, tail
        for (size_t i = ntiles * TILE + threadIdx.x; i < nvec; i += RD_THREADS) {
            Pack<T> p = as_pack<T>(ld_stream(xv + i));
            st.vec(p, i);
            W m = R::pre(map(p.v[0]));
#pragma unroll
            for (int k = 1; k < VPT; ++k) m = R::tile(m, R::pre(map(p.v[k])));
            acc = R::comb(acc, R::lift(m));
        }
        for (size_t i = threadIdx.x; i < head; i += RD_THREADS) acc = R::comb(acc, R::lift(R::pre(map(st.scalar(x[i], i)))));
        for (size_t i = head + nvec * VPT + threadIdx.x; i < n; i += RD_THREADS)
            acc = R::comb(acc, R::lift(R::pre(map(st.scalar(x[i], i)))));
    }
    acc = block_reduce<R>(acc, smem);
    // the last CTA to finish writes the result (tail latency of a few microseconds)
    A fin;
    if (!last_cta_out<R>(acc, partials, counter, smem, is_last, fin)) return;
    if (threadIdx.x == 0) {
        if constexpr (std::is_arithmetic<A>::value) {
            Out res;
            if (finalize_mode == 1) res = (Out)(fin == (A)n_for_all);  // ALL
            else if (finalize_mode == 2) res = (Out)(fin != (A)0);      // ANY
            else res = (Out)fin;
            memcpy(out, &res, sizeof(Out));
            if (sizeof(Out) < 8) memset((char*)out + sizeof(Out), 0, 8 - sizeof(Out));
            A wide = fin;
            memcpy((char*)out + 8, &wide, sizeof(A));
            if (sizeof(A) < 8) memset((char*)out + 8 + sizeof(A), 0, 8 - sizeof(A));
            if (fc.host_out && fc.nranks <= 1) {
                // single worker: the scalar goes straight into pinned host memory (zero-copy), no D2H memcpy launch
                unsigned long long bits = 0;
                memcpy(&bits, &res, sizeof(Out));
                volatile unsigned long long* h = reinterpret_cast<volatile unsigned long long*>(fc.host_out);
                h[0] = bits;
                h[1] = 0ull;
                __threadfence_system();
            }
        } else if constexpr (is_cplx<Out>::value) {  // complex sum / product: rounded once to Complex{T}, [0, 2*sizeof(T)) of the slot
            using CT = decltype(Out::re);
            const Out res{(CT)fin.re, (CT)fin.im};
            memset(out, 0, 16);
            memcpy(out, &res, sizeof(Out));
        } else {  // extrema: the (min, max) pair fills the slot (8 bytes for 4-byte T, 16 for 8-byte T)
            memset(out, 0, 16);
            memcpy(out, &fin, sizeof(A));
        }
    }
    if constexpr (!std::is_arithmetic<Out>::value) return;
    else {
    if (fc.nranks <= 1) return;
    // ---- fused cross-worker combine over NVLink peer memory (replaces remotecall_fetch + reduce(op, results), reference
    // src/mapreduce.jl:30-34, and an ncclAllGather + D2H copy): thread j of this last CTA PUSHES this rank's chunk result into
    // rank j's mailbox (16-byte payload, system fence, then the sequence flag), then polls its own mailbox slot j until rank j's
    // result for this call has landed; thread 0 folds the P results LEFT TO RIGHT in rank (= procs(d)) order in the result type
    // and writes the scalar straight into pinned host memory.  Two parity banks: a fast rank can be at most one call ahead.
    __shared__ unsigned long long pay[2];
    __shared__ unsigned long long got[DAB_MAX_RANKS];
    __shared__ int timed_out;
    if (threadIdx.x == 0) {
        memcpy(&pay[0], out, 8);
        memcpy(&pay[1], (char*)out + 8, 8);
        timed_out = 0;
    }
    __syncthreads();
    const size_t bank = (size_t)(fc.seq & 1ull) * DAB_MAX_RANKS * DAB_MBOX_SLOT;
    if (threadIdx.x < (unsigned)fc.nranks) {
        volatile unsigned long long* dst =
            reinterpret_cast<volatile unsigned long long*>((char*)fc.peers[threadIdx.x] + bank + (size_t)fc.rank * DAB_MBOX_SLOT);
        dst[0] = pay[0];
        dst[1] = pay[1];
        __threadfence_system();
        dst[2] = fc.seq;
        volatile unsigned long long* src =
            reinterpret_cast<volatile unsigned long long*>((char*)fc.peers[fc.rank] + bank + (size_t)threadIdx.x * DAB_MBOX_SLOT);
        // SPMD ranks are not in lockstep (a first-time NVRTC compile, a large H2D copy or GC can hold one back for seconds), so the
        // bound is generous wall-clock time (default 120 s, dab_set_option "combine_timeout_ms") and only exists so that a DEAD
        // peer surfaces as an error instead of a hung GPU; a timeout leaves the communicator unusable, like a failed collective.
        const unsigned long long t0 = dab_globaltimer_ns();
        unsigned int spins = 0;
        while (src[2] != fc.seq) {
            if ((++spins & 1023u) == 0 && dab_globaltimer_ns() - t0 > fc.timeout_ns) {
                timed_out = 1;
                break;
            }
        }
        __threadfence_system();
        got[threadIdx.x] = src[0];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Out a;
        memcpy(&a, &got[0], sizeof(Out));
        for (int j = 1; j < fc.nranks; ++j) {
            Out b;
            memcpy(&b, &got[j], sizeof(Out));
            switch (fc.op) {
                case DAB_SUM: case DAB_COUNT: a = jl::add(a, b); break;
                case DAB_PROD: a = jl::mul(a, b); break;
                case DAB_MAX: a = jl::max(a, b); break;
                case DAB_MIN: a = jl::min(a, b); break;
                case DAB_ALL: a = (Out)(a != (Out)0 && b != (Out)0); break;
                default: a = (Out)(a != (Out)0 || b != (Out)0); break;  // ANY
            }
        }
        unsigned long long bits = 0;
        memcpy(&bits, &a, sizeof(Out));
        volatile unsigned long long* h = reinterpret_cast<volatile unsigned long long*>(fc.host_out);
        h[0] = bits;
        h[1] = (unsigned long long)timed_out;
        __threadfence_system();
    }
    }  // arithmetic Out
}

template <typename T, typename Map, typename R, typename Out, typename St = NoStore>
int32_t launch_reduce(dab_ctx* ctx, const T* x, size_t n, Map map, void* out, int finalize_mode, St st = St()) {
    const FlatGrid fg = flat_grid(x, n);
    if constexpr (!std::is_same<St, NoStore>::value) st.yv = reinterpret_cast<int4*>(st.y + fg.head);
    FusedComm fc;
    memset(&fc, 0, sizeof(fc));
    if (ctx->fuse_op >= 0 && ctx->mbox_ranks > 1) {
        fc.peers = ctx->peer_mbox_dev;
        fc.host_out = ctx->host_slot;
        fc.seq = ++ctx->mbox_seq;
        fc.timeout_ns = (unsigned long long)ctx->opt_combine_timeout_ms * 1000000ull;
        fc.rank = ctx->rank;
        fc.nranks = ctx->mbox_ranks;
        fc.op = ctx->fuse_op;
    } else if (ctx->fuse_op >= 0) {
        fc.host_out = ctx->host_slot;  // one worker: zero-copy scalar to the host, nothing to combine
        fc.nranks = 1;
        fc.op = ctx->fuse_op;
    }
    reduce_kernel<T, Map, R, Out, St><<<(unsigned)fg.grid, RD_THREADS, 0, ctx->stream>>>(
        x, n, fg.head, map, (typename R::A*)ctx->block_partials, ctx->counter, out, finalize_mode, (long long)n, fg.tiles_per_cta, fc, st);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename T>
using ResultOfSum = typename std::conditional<std::is_floating_point<T>::value, T, long long>::type;

template <typename T, int FN>
int32_t reduce_arith(dab_ctx* ctx, int32_t op, const T* x, size_t n, void* out) {
    MapF<T, FN> map{(T)0};
    switch (op) {
        case DAB_SUM: return launch_reduce<T, MapF<T, FN>, SumTraits<T>, ResultOfSum<T>>(ctx, x, n, map, out, 0);
        case DAB_PROD: return launch_reduce<T, MapF<T, FN>, ProdTraits<T>, ResultOfSum<T>>(ctx, x, n, map, out, 0);
        case DAB_MAX: return launch_reduce<T, MapF<T, FN>, MaxTraits<T>, T>(ctx, x, n, map, out, 0);
        case DAB_MIN: return launch_reduce<T, MapF<T, FN>, MinTraits<T>, T>(ctx, x, n, map, out, 0);
        case DAB_EXTREMA:
            if constexpr (FN == DAB_MAP_ID) return launch_reduce<T, ExtMapF<T>, ExtremaTraits<T>, Pair<T>>(ctx, x, n, ExtMapF<T>{(T)0}, out, 0);
            else return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "extrema with a map is not served (no host fallback)");
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "reduce op %d needs a predicate map (no host fallback)", op);
    }
}

template <typename T, int FN>
int32_t reduce_pred(dab_ctx* ctx, int32_t op, const T* x, size_t n, const void* param, void* out) {
    PredF<T, FN> map{param ? *(const T*)param : (T)0};
    int mode;
    switch (op) {
        case DAB_ALL: mode = 1; break;
        case DAB_ANY: mode = 2; break;
        case DAB_COUNT:
        case DAB_SUM: mode = 0; break;  // sum of Bools == count
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "reduce op %d on a predicate map (no host fallback)", op);
    }
    return launch_reduce<T, PredF<T, FN>, CountTraits, long long>(ctx, x, n, map, out, mode);
}

template <typename T>
int32_t reduce_t(dab_ctx* ctx, int32_t op, int32_t map, const void* param, const T* x, size_t n, void* out) {
    switch (map) {
        case DAB_MAP_ID: return reduce_arith<T, DAB_MAP_ID>(ctx, op, x, n, out);
        case DAB_MAP_ABS: return reduce_arith<T, DAB_MAP_ABS>(ctx, op, x, n, out);
        case DAB_MAP_ABS2: return reduce_arith<T, DAB_MAP_ABS2>(ctx, op, x, n, out);
        case DAB_MAP_NEG: return reduce_arith<T, DAB_MAP_NEG>(ctx, op, x, n, out);
#define P(FN) \
    case FN: return reduce_pred<T, FN>(ctx, op, x, n, param, out)
            P(DAB_MAP_EQ);
            P(DAB_MAP_NE);
            P(DAB_MAP_LT);
            P(DAB_MAP_LE);
            P(DAB_MAP_GT);
            P(DAB_MAP_GE);
            P(DAB_MAP_ISNAN);
            P(DAB_MAP_NONZERO);
#undef P
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "map %d not served by a reduce kernel (no host fallback)", map);
    }
}

// Complex{T} chunks: the same kernel with Cplx<T> elements (a 16-byte load carries 2 ComplexF32 or 1 ComplexF64).
template <typename T>
int32_t reduce_c(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const Cplx<T>* x, size_t n, void* out) {
    using Z = Cplx<T>;
    if ((uintptr_t)x % sizeof(Z))
        return dab_fail(ctx, DAB_ERR_ARG, "dab_reduce: complex dtype %d needs %d-byte aligned data", dtype, (int)sizeof(Z));
    switch (map) {
        case DAB_MAP_ID:
            if (op == DAB_SUM) return launch_reduce<Z, CMapF<T, DAB_MAP_ID>, CSumTraits<T>, Z>(ctx, x, n, {(T)0}, out, 0);
            if (op == DAB_PROD) return launch_reduce<Z, CMapF<T, DAB_MAP_ID>, CProdTraits<T>, Z>(ctx, x, n, {(T)0}, out, 0);
            break;
        case DAB_MAP_NEG:
            if (op == DAB_SUM) return launch_reduce<Z, CMapF<T, DAB_MAP_NEG>, CSumTraits<T>, Z>(ctx, x, n, {(T)0}, out, 0);
            if (op == DAB_PROD) return launch_reduce<Z, CMapF<T, DAB_MAP_NEG>, CProdTraits<T>, Z>(ctx, x, n, {(T)0}, out, 0);
            break;
#define ABSMAP(FN)                                                                                                      \
    case FN:                                                                                                            \
        if (op == DAB_SUM) return launch_reduce<Z, CMapF<T, FN>, SumTraits<T>, T>(ctx, x, n, {(T)0}, out, 0);            \
        if (op == DAB_MAX) return launch_reduce<Z, CMapF<T, FN>, MaxTraits<T>, T>(ctx, x, n, {(T)0}, out, 0);            \
        if (op == DAB_MIN) return launch_reduce<Z, CMapF<T, FN>, MinTraits<T>, T>(ctx, x, n, {(T)0}, out, 0);            \
        break;
            ABSMAP(DAB_MAP_ABS)
            ABSMAP(DAB_MAP_ABS2)
#undef ABSMAP
#define PREDMAP(FN)                                                                                                     \
    case FN: {                                                                                                          \
        const int mode = op == DAB_ALL ? 1 : (op == DAB_ANY ? 2 : 0);                                                   \
        if (op == DAB_ALL || op == DAB_ANY || op == DAB_COUNT || op == DAB_SUM)                                         \
            return launch_reduce<Z, CPredF<T, FN>, CountTraits, long long>(ctx, x, n, {(T)0}, out, mode);               \
        break;                                                                                                          \
    }
            PREDMAP(DAB_MAP_NONZERO)
            PREDMAP(DAB_MAP_ISNAN)
#undef PREDMAP
        default: break;
    }
    return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reduce: op %d with map %d is not served for complex dtype %d (no host fallback)", op, map,
                    dtype);
}

// Float16 chunks: the same kernel with Half elements (a 16-byte load carries 8), each value widened to Float32 by the map (HMapF); Float16
// results for SUM / PROD / MAX / MIN (extrema of Float16 data is a MIN and a MAX reduction on the host side).
template <int FN>
int32_t reduce_h_arith(dab_ctx* ctx, int32_t op, const Half* x, size_t n, void* out) {
    using M = HMapF<FN>;
    const M map{};
    switch (op) {
        case DAB_SUM: return launch_reduce<Half, M, SumTraits<float>, Half>(ctx, x, n, map, out, 0);
        case DAB_PROD: return launch_reduce<Half, M, ProdTraits<float>, Half>(ctx, x, n, map, out, 0);
        case DAB_MAX: return launch_reduce<Half, M, MaxTraits<float>, Half>(ctx, x, n, map, out, 0);
        case DAB_MIN: return launch_reduce<Half, M, MinTraits<float>, Half>(ctx, x, n, map, out, 0);
        case DAB_EXTREMA: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reduce: EXTREMA is not served for Float16 (a MIN and a MAX reduction are)");
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "reduce op %d needs a predicate map (no host fallback)", op);
    }
}

template <int FN>
int32_t reduce_h_pred(dab_ctx* ctx, int32_t op, const Half* x, size_t n, const void* param, void* out) {
    HPredF<FN> map;
    map.p.bits = 0;
    if (param) memcpy(&map.p, param, 2);
    const int mode = op == DAB_ALL ? 1 : (op == DAB_ANY ? 2 : 0);
    if (op != DAB_ALL && op != DAB_ANY && op != DAB_COUNT && op != DAB_SUM)
        return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "reduce op %d on a predicate map (no host fallback)", op);
    return launch_reduce<Half, HPredF<FN>, CountTraits, long long>(ctx, x, n, map, out, mode);
}

int32_t reduce_h(dab_ctx* ctx, int32_t op, int32_t map, const void* param, const Half* x, size_t n, void* out) {
    if ((uintptr_t)x % 2) return dab_fail(ctx, DAB_ERR_ARG, "dab_reduce: Float16 data needs 2-byte alignment");
    switch (map) {
        case DAB_MAP_ID: return reduce_h_arith<DAB_MAP_ID>(ctx, op, x, n, out);
        case DAB_MAP_ABS: return reduce_h_arith<DAB_MAP_ABS>(ctx, op, x, n, out);
        case DAB_MAP_ABS2: return reduce_h_arith<DAB_MAP_ABS2>(ctx, op, x, n, out);
        case DAB_MAP_NEG: return reduce_h_arith<DAB_MAP_NEG>(ctx, op, x, n, out);
#define P(FN) \
    case FN: return reduce_h_pred<FN>(ctx, op, x, n, param, out)
            P(DAB_MAP_EQ);
            P(DAB_MAP_NE);
            P(DAB_MAP_LT);
            P(DAB_MAP_LE);
            P(DAB_MAP_GT);
            P(DAB_MAP_GE);
            P(DAB_MAP_ISNAN);
            P(DAB_MAP_NONZERO);
#undef P
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "map %d not served by a reduce kernel for Float16 (no host fallback)", map);
    }
}

// The deferred dab_affine y .= a.*x .+ b and the reduction of y as ONE kernel: reads x, writes y, reduces y (8 B/element of
// Float32 instead of 8 + 4).  Same CTA geometry, element-to-thread mapping and fold as reduce_arith<T, DAB_MAP_ID> on y.
template <typename T>
int32_t reduce_pending_affine(dab_ctx* ctx, int32_t op, const dab_pending_affine& p, void* out) {
    using M = MapF<T, DAB_MAP_ID>;
    AffineStore<T> st;
    memcpy(&st.f.a, p.a, sizeof(T));
    memcpy(&st.f.b, p.b, sizeof(T));
    st.y = (T*)p.y;
    st.yv = nullptr;  // set by launch_reduce from the head
    const T* x = (const T*)p.x;
    switch (op) {
        case DAB_SUM: return launch_reduce<T, M, SumTraits<T>, ResultOfSum<T>>(ctx, x, p.n, M{(T)0}, out, 0, st);
        case DAB_PROD: return launch_reduce<T, M, ProdTraits<T>, ResultOfSum<T>>(ctx, x, p.n, M{(T)0}, out, 0, st);
        case DAB_MAX: return launch_reduce<T, M, MaxTraits<T>, T>(ctx, x, p.n, M{(T)0}, out, 0, st);
        default: return launch_reduce<T, M, MinTraits<T>, T>(ctx, x, p.n, M{(T)0}, out, 0, st);  // DAB_MIN
    }
}

bool consumes_pending(const dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* x, size_t n) {
    const dab_pending_affine& p = ctx->pending;
    return p.active && x == p.y && n == p.n && dtype == p.dtype && map == DAB_MAP_ID &&
           (op == DAB_SUM || op == DAB_PROD || op == DAB_MAX || op == DAB_MIN);
}

int32_t reduce_u8(dab_ctx* ctx, int32_t op, int32_t map, const uint8_t* x, size_t n, void* out) {
    // Bool arrays: all(d) / any(d) / count(d) / sum(d) with the identity predicate; max/min on Bool.
    if (map != DAB_MAP_ID && map != DAB_MAP_NONZERO)
        return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "map %d on Bool not served (no host fallback)", map);
    if (op == DAB_MAX) return launch_reduce<uint8_t, MapF<uint8_t, DAB_MAP_ID>, MaxTraits<uint8_t>, uint8_t>(ctx, x, n, {0}, out, 0);
    if (op == DAB_MIN) return launch_reduce<uint8_t, MapF<uint8_t, DAB_MAP_ID>, MinTraits<uint8_t>, uint8_t>(ctx, x, n, {0}, out, 0);
    return reduce_pred<uint8_t, DAB_MAP_NONZERO>(ctx, op, x, n, nullptr, out);
}

// host-side write of the n == 0 result
int32_t empty_result(dab_ctx* ctx, int32_t dtype, int32_t op, void* out_dev) {
    unsigned char buf[16];
    memset(buf, 0, 16);
    bool flt = dtype == DAB_F32 || dtype == DAB_F64;
    switch (op) {
        case DAB_SUM:
        case DAB_ANY:
        case DAB_COUNT: break;
        case DAB_ALL: {
            long long one = 1;
            memcpy(buf, &one, 8);
            break;
        }
        case DAB_PROD:
            if (dtype == DAB_F32) {
                float one = 1.f;
                memcpy(buf, &one, 4);
            } else if (dtype == DAB_F64) {
                double one = 1.0;
                memcpy(buf, &one, 8);
            } else if (dtype == DAB_F16) {
                const unsigned short one = 0x3c00;
                memcpy(buf, &one, 2);
            } else if (dtype == DAB_C64) {
                const float one[2] = {1.f, 0.f};
                memcpy(buf, one, 8);
            } else if (dtype == DAB_C128) {
                const double one[2] = {1.0, 0.0};
                memcpy(buf, one, 16);
            } else {
                long long one = 1;
                memcpy(buf, &one, 8);
            }
            if (flt || dtype == DAB_F16) {
                double one = 1.0;
                memcpy(buf + 8, &one, 8);
            }
            break;
        default: return dab_fail(ctx, DAB_ERR_EMPTY, "reducing over an empty collection is not allowed");
    }
    // stream-ordered small copy from a stack buffer: use the pinned slot's tail to stay async-safe
    memcpy((char*)ctx->host_slot + DAB_MAX_RANKS * 16, buf, 16);
    DAB_CUDA(ctx, cudaMemcpyAsync(out_dev, (char*)ctx->host_slot + DAB_MAX_RANKS * 16, 16, cudaMemcpyHostToDevice, ctx->stream));
    DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_reduce_result_dtype(int32_t dtype, int32_t op, int32_t map, int32_t* out_dtype) {
    if (!out_dtype) return DAB_ERR_ARG;
    if (dtype == DAB_C64 || dtype == DAB_C128) {
        const int32_t comp = dtype == DAB_C64 ? DAB_F32 : DAB_F64;
        const bool id = map == DAB_MAP_ID || map == DAB_MAP_NEG, mag = map == DAB_MAP_ABS || map == DAB_MAP_ABS2;
        const bool pred = map == DAB_MAP_NONZERO || map == DAB_MAP_ISNAN;
        if (id && (op == DAB_SUM || op == DAB_PROD)) *out_dtype = dtype;
        else if (mag && (op == DAB_SUM || op == DAB_MAX || op == DAB_MIN)) *out_dtype = comp;
        else if (pred && (op == DAB_SUM || op == DAB_COUNT || op == DAB_ALL || op == DAB_ANY)) *out_dtype = DAB_I64;
        else return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "op %d with map %d is not served for complex dtype %d", op, map, dtype);
        return DAB_OK;
    }
    const bool pred = map >= DAB_MAP_EQ;  // predicate maps yield Bool: sum/count/all/any -> Int64
    switch (op) {
        case DAB_SUM:
        case DAB_PROD:
            *out_dtype = (!pred && (dtype == DAB_F32 || dtype == DAB_F64 || dtype == DAB_F16)) ? dtype : DAB_I64;
            return DAB_OK;
        case DAB_MAX:
        case DAB_MIN:
        case DAB_EXTREMA: *out_dtype = dtype; return DAB_OK;
        case DAB_ALL:
        case DAB_ANY:
        case DAB_COUNT: *out_dtype = DAB_I64; return DAB_OK;
        default: return DAB_ERR_ARG;
    }
}

// out_dev: 16 bytes (result + wide accumulator)
int32_t dab_reduce(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* map_param, const void* x, size_t n,
                   void* out_dev) {
    DAB_ENTER_NOFLUSH(ctx);
    if (out_dev && consumes_pending(ctx, dtype, op, map, x, n)) {
        const dab_pending_affine p = ctx->pending;
        ctx->pending.active = 0;
        switch (dtype) {
            case DAB_F32: return reduce_pending_affine<float>(ctx, op, p, out_dev);
            case DAB_F64: return reduce_pending_affine<double>(ctx, op, p, out_dev);
            case DAB_I32: return reduce_pending_affine<int32_t>(ctx, op, p, out_dev);
            default: return reduce_pending_affine<long long>(ctx, op, p, out_dev);  // DAB_I64
        }
    }
    DAB_FLUSH(ctx);
    DAB_REQUIRE(ctx, out_dev && (x || n == 0), DAB_ERR_ARG, "dab_reduce: null pointer");
    DAB_REQUIRE(ctx, op >= DAB_SUM && op <= DAB_EXTREMA, DAB_ERR_ARG, "dab_reduce: bad op %d", op);
    if (dtype == DAB_C64 || dtype == DAB_C128) {
        int32_t rdt;
        if (dab_reduce_result_dtype(dtype, op, map, &rdt) != DAB_OK)
            return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reduce: op %d with map %d is not served for complex dtype %d (no host fallback)", op,
                            map, dtype);
        if (n == 0) return empty_result(ctx, map == DAB_MAP_ABS || map == DAB_MAP_ABS2 ? rdt : dtype, op, out_dev);
        if (dtype == DAB_C64) return reduce_c<float>(ctx, dtype, op, map, (const Cplx<float>*)x, n, out_dev);
        return reduce_c<double>(ctx, dtype, op, map, (const Cplx<double>*)x, n, out_dev);
    }
    if (n == 0) return empty_result(ctx, dtype, op, out_dev);
    // predicate maps turn the value into a Bool: only SUM/ALL/ANY/COUNT make sense
    switch (dtype) {
        case DAB_F32: return reduce_t<float>(ctx, op, map, map_param, (const float*)x, n, out_dev);
        case DAB_F64: return reduce_t<double>(ctx, op, map, map_param, (const double*)x, n, out_dev);
        case DAB_I32: return reduce_t<int32_t>(ctx, op, map, map_param, (const int32_t*)x, n, out_dev);
        case DAB_I64: return reduce_t<long long>(ctx, op, map, map_param, (const long long*)x, n, out_dev);
        case DAB_U8: return reduce_u8(ctx, op, map, (const uint8_t*)x, n, out_dev);
        case DAB_F16: return reduce_h(ctx, op, map, map_param, (const Half*)x, n, out_dev);
        default: return dab_fail(ctx, DAB_ERR_ARG, "dab_reduce: bad dtype %d", dtype);
    }
}

int32_t dab_reduce_host(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* map_param, const void* x, size_t n,
                        void* out_host) {
    DAB_ENTER_NOFLUSH(ctx);  // dab_reduce consumes or flushes the deferred dab_affine
    if (!out_host) {
        DAB_FLUSH(ctx);
        return dab_fail(ctx, DAB_ERR_ARG, "dab_reduce_host: null out");
    }
    int32_t st = dab_reduce(ctx, dtype, op, map, map_param, x, n, ctx->result_slot);
    if (st != DAB_OK) return st;
    DAB_CUDA(ctx, cudaMemcpyAsync(ctx->host_slot, ctx->result_slot, 16, cudaMemcpyDeviceToHost, ctx->stream));
    DAB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(out_host, ctx->host_slot, 16);
    return DAB_OK;
}

// reduce(op, results) on the caller: plain left fold in procs(d) order, in the result dtype (src/mapreduce.jl:34).
int32_t dab_combine_ordered(int32_t rdt, int32_t op, const void* partials, size_t p, void* out) {
    if (!partials || !out) return dab_fail(nullptr, DAB_ERR_ARG, "dab_combine_ordered: null pointer");
    if (p == 0) return dab_fail(nullptr, DAB_ERR_EMPTY, "reducing over an empty collection is not allowed");
#define FOLD(T, EXPR)                          \
    {                                          \
        const T* v = (const T*)partials;       \
        T a = v[0];                            \
        for (size_t i = 1; i < p; ++i) {       \
            T b = v[i];                        \
            a = (EXPR);                        \
        }                                      \
        *(T*)out = a;                          \
        return DAB_OK;                         \
    }
    auto fmax_jl = [](auto a, auto b) {
        using T = decltype(a);
        if (a != a || b != b) return (T)NAN;
        if (a == b) return std::signbit(a) ? b : a;
        return a > b ? a : b;
    };
    auto fmin_jl = [](auto a, auto b) {
        using T = decltype(a);
        if (a != a || b != b) return (T)NAN;
        if (a == b) return std::signbit(a) ? a : b;
        return a < b ? a : b;
    };
    switch (rdt) {
        case DAB_F32:
            switch (op) {
                case DAB_SUM: {
                    // volatile: keep each partial sum rounded to fp32 (no x87 / contraction surprises)
                    const float* v = (const float*)partials;
                    volatile float a = v[0];
                    for (size_t i = 1; i < p; ++i) a = a + v[i];
                    *(float*)out = a;
                    return DAB_OK;
                }
                case DAB_PROD: {
                    const float* v = (const float*)partials;
                    volatile float a = v[0];
                    for (size_t i = 1; i < p; ++i) a = a * v[i];
                    *(float*)out = a;
                    return DAB_OK;
                }
                case DAB_MAX: FOLD(float, fmax_jl(a, b))
                case DAB_MIN: FOLD(float, fmin_jl(a, b))
                default: break;
            }
            break;
        case DAB_F64:
            switch (op) {
                case DAB_SUM: FOLD(double, a + b)
                case DAB_PROD: FOLD(double, a * b)
                case DAB_MAX: FOLD(double, fmax_jl(a, b))
                case DAB_MIN: FOLD(double, fmin_jl(a, b))
                default: break;
            }
            break;
        case DAB_I64:
            switch (op) {
                case DAB_SUM:
                case DAB_COUNT: FOLD(long long, (long long)((unsigned long long)a + (unsigned long long)b))
                case DAB_PROD: FOLD(long long, (long long)((unsigned long long)a * (unsigned long long)b))
                case DAB_MAX: FOLD(long long, a > b ? a : b)
                case DAB_MIN: FOLD(long long, a < b ? a : b)
                case DAB_ALL: FOLD(long long, (long long)(a && b))
                case DAB_ANY: FOLD(long long, (long long)(a || b))
                default: break;
            }
            break;
        case DAB_I32:
            switch (op) {
                case DAB_MAX: FOLD(int32_t, a > b ? a : b)
                case DAB_MIN: FOLD(int32_t, a < b ? a : b)
                default: break;
            }
            break;
        case DAB_U8:
            switch (op) {
                case DAB_MAX: FOLD(uint8_t, a > b ? a : b)
                case DAB_MIN: FOLD(uint8_t, a < b ? a : b)
                default: break;
            }
            break;
        case DAB_F16: {  // Float16 arithmetic: each operation widened to Float32 and rounded back to Float16, as Julia's Float16 methods
            const unsigned short* v = (const unsigned short*)partials;
            float a = dab_half_to_float(v[0]);
            for (size_t i = 1; i < p; ++i) {
                const float b = dab_half_to_float(v[i]);
                volatile float r;
                switch (op) {
                    case DAB_SUM: r = a + b; break;
                    case DAB_PROD: r = a * b; break;
                    case DAB_MAX: r = fmax_jl(a, b); break;
                    case DAB_MIN: r = fmin_jl(a, b); break;
                    default: return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "dab_combine_ordered: dtype %d (Float16) op %d", rdt, op);
                }
                a = dab_half_to_float(dab_float_to_half(r));
            }
            const unsigned short h = dab_float_to_half(a);
            memcpy(out, &h, 2);
            return DAB_OK;
        }
        case DAB_C64:
            if (op == DAB_SUM || op == DAB_PROD) {  // Float32 arithmetic, each operation rounded (volatile: no wider intermediates)
                const float* v = (const float*)partials;
                volatile float re = v[0], im = v[1];
                for (size_t i = 1; i < p; ++i) {
                    const float br = v[2 * i], bi = v[2 * i + 1];
                    if (op == DAB_SUM) {
                        re = re + br;
                        im = im + bi;
                    } else {
                        volatile float rr = re * br, ii = im * bi, ri = re * bi, ir = im * br;
                        re = rr - ii;
                        im = ri + ir;
                    }
                }
                ((float*)out)[0] = re;
                ((float*)out)[1] = im;
                return DAB_OK;
            }
            break;
        case DAB_C128:
            if (op == DAB_SUM || op == DAB_PROD) {
                const double* v = (const double*)partials;
                volatile double re = v[0], im = v[1];
                for (size_t i = 1; i < p; ++i) {
                    const double br = v[2 * i], bi = v[2 * i + 1];
                    if (op == DAB_SUM) {
                        re = re + br;
                        im = im + bi;
                    } else {
                        volatile double rr = re * br, ii = im * bi, ri = re * bi, ir = im * br;
                        re = rr - ii;
                        im = ri + ir;
                    }
                }
                ((double*)out)[0] = re;
                ((double*)out)[1] = im;
                return DAB_OK;
            }
            break;
        default: break;
    }
#undef FOLD
    return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "dab_combine_ordered: dtype %d op %d", rdt, op);
}

}  // extern "C"
