// dab_scan.cu -- K17: accumulate!(op, B, A; dims) / cumsum / cumprod on one chunk (Julia base/accumulate.jl), single pass over HBM.
//
// The chunk is collapsed to the column-major shape (inner, len, outer) around `dims`, as dab_reducedim does:
//   y[i + inner*(r + len*o)] = c[i + inner*o] (op) x[i + inner*o*len] (op) ... (op) x[i + inner*(r + len*o)]
// where c is the optional carry slab (the exclusive prefix contributed by init and by earlier chunks along dims) or nothing.
//   * inner == 1  (dims = 1, vectors): ONE flat-grid kernel over the whole chunk.  Persistent CTAs take 4096-element tiles by ticket
//     (address order), stage them in shared memory with 16-byte loads, and scan them as a SEGMENTED scan: a run starts every `len`
//     elements, so one long vector, columns of a few thousand elements and (10, 10^8) are the same kernel.  The prefix of a run that
//     crosses a tile boundary comes from a decoupled look-back over the earlier tiles' words; a tile that contains a run start
//     publishes its inclusive value at once, so the look-back never walks past the last run start.  8 bytes per Float32 element.
//     A misaligned x (y) is loaded (stored) with coalesced element accesses for the whole call: there is no head peel, and the host
//     runtime's own chunks are always 256-byte aligned.
//   * inner  > 1  (dims >= 2): each thread owns 16 bytes along `inner` (or one element when inner is not a multiple of a vector) and
//     walks `len` sequentially: coalesced, single pass, 8 bytes per Float32 element.  When inner*outer cannot fill ~4 waves of the
//     GPU, `len` is split into segments: pass 1 reduces each segment, the flat kernel above scans the segment totals (stored
//     segment-fastest, so every output's totals are one run), pass 2 scans each segment from its carry (12 bytes per Float32 element).
// Carriers: fp64 for Float32 / Float64 sums and products (rounded once per output), Int64 for integer and Bool sums and products
// (an Int32 result keeps the low 32 bits: Julia's wrap-around), the element type for max / min.  The operators are the reduce
// traits' (jl::add / jl::mul / jl::max / jl::min: Julia's NaN and signed-zero rules).
//
// Look-back words never need clearing: each flat launch gets a new epoch, and a word of an older launch reads as "not ready"
// (the scheme of K11, dab_sort.cu).  Tile tickets come from one 64-bit counter that is never reset either: every launch draws exactly
// ntiles + grid tickets, so the host knows where the next launch's tickets start.
#include "dab_reduce_traits.cuh"

namespace {

constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 16;                        // elements per thread of the flat kernel
constexpr int SC_TILE = SC_THREADS * SC_ITEMS;      // 4096 elements per tile
constexpr size_t SC_HEAD_BYTES = 256;               // ticket counter, ahead of the look-back words
constexpr unsigned long long LB_PARTIAL = 1ull << 62, LB_INCLUSIVE = 2ull << 62, LB_FLAGS = 3ull << 62;
constexpr unsigned long long LB_EPOCH_MASK = ((1ull << 30) - 1ull) << 32;

struct LookbackWord {   // one per tile; `agg` is written before a PARTIAL status, `incl` before an INCLUSIVE one
    unsigned long long status, agg, incl, pad;
};

// ---- the scan operator over the carrier, from the reduce traits ------------------------------------------------------------------
template <typename T, int OP>
struct ScanOp {
    using R = typename std::conditional<OP == DAB_SUM, SumTraits<T>,
              typename std::conditional<OP == DAB_PROD, ProdTraits<T>,
              typename std::conditional<OP == DAB_MAX, MaxTraits<T>, MinTraits<T>>::type>::type>::type;
    using A = typename R::A;
    static constexpr int op = OP;
    // -0.0 is the identity of a float sum (0.0 + -0.0 would lose the sign of a leading -0.0, which reduce_first keeps)
    __device__ static __forceinline__ A identity() {
        if constexpr (OP == DAB_SUM && std::is_floating_point<A>::value) return (A)-0.0;
        else return R::identity();
    }
    __device__ static __forceinline__ A comb(A a, A b) { return R::comb(a, b); }
    __device__ static __forceinline__ A lift(T v) { return (A)v; }
};

template <typename Out, typename A>
__device__ __forceinline__ Out narrow_out(A a) {
    if constexpr (std::is_same<Out, int32_t>::value && std::is_same<A, long long>::value) return (int32_t)(uint32_t)(unsigned long long)a;
    else return (Out)a;   // fp64 -> Float32 rounds to nearest; Bool products are 0 / 1
}

template <typename A>
__device__ __forceinline__ unsigned long long to_bits(A a) {
    unsigned long long u = 0;
    memcpy(&u, &a, sizeof(A));
    return u;
}
template <typename A>
__device__ __forceinline__ A from_bits(unsigned long long u) {
    A a;
    memcpy(&a, &u, sizeof(A));
    return a;
}
template <typename A>
__device__ __forceinline__ A shfl_up_a(A v, int d) {
    const unsigned long long u = to_bits(v);
    const int lo = __shfl_up_sync(0xffffffffu, (int)(u & 0xffffffffull), d);
    const int hi = __shfl_up_sync(0xffffffffu, (int)(u >> 32), d);
    return from_bits<A>(((unsigned long long)(unsigned)hi << 32) | (unsigned)lo);
}
template <typename A>
__device__ __forceinline__ A shfl_down_a(A v, int d) {
    const unsigned long long u = to_bits(v);
    const int lo = __shfl_down_sync(0xffffffffu, (int)(u & 0xffffffffull), d);
    const int hi = __shfl_down_sync(0xffffffffu, (int)(u >> 32), d);
    return from_bits<A>(((unsigned long long)(unsigned)hi << 32) | (unsigned)lo);
}

__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// segmented-scan element: value and "a run starts in here"; (a, fa) . (b, fb) = (fb ? b : a op b, fa | fb)
template <typename S>
struct Seg {
    typename S::A v;
    int f;
};
template <typename S>
__device__ __forceinline__ Seg<S> seg_comb(Seg<S> a, Seg<S> b) {
    return Seg<S>{b.f ? b.v : S::comb(a.v, b.v), a.f | b.f};
}

// ---- inner == 1: flat single-pass segmented scan with decoupled look-back ------------------------------------------------------
// y == nullptr: totals mode -- nothing is stored but totals[o] = the inclusive value at the end of run o.
template <typename T, typename Out, typename S>
__global__ void __launch_bounds__(SC_THREADS) scan_flat_kernel(const T* x, Out* y, size_t n, size_t len, const typename S::A* __restrict__ carry,
                                                               typename S::A* __restrict__ totals, LookbackWord* __restrict__ lb,
                                                               unsigned long long* __restrict__ ticket, unsigned long long ticket_base,
                                                               unsigned long long ep, unsigned long long ntiles) {
    using A = typename S::A;
    __shared__ __align__(16) unsigned char stage[SC_TILE * 8];   // the tile's input, then its output
    __shared__ Seg<S> s_warp[SC_THREADS / 32];
    __shared__ A s_prefix;
    __shared__ unsigned long long s_tile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool x_vec = ((uintptr_t)x & 15) == 0, y_vec = y && ((uintptr_t)y & 15) == 0;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(ticket, 1ull) - ticket_base;
        __syncthreads();
        const unsigned long long tile = s_tile;
        if (tile >= ntiles) return;
        const size_t tb = (size_t)tile * SC_TILE;
        const size_t cnt = (n - tb < (size_t)SC_TILE) ? n - tb : (size_t)SC_TILE;
        T* sin = reinterpret_cast<T*>(stage);
        if (cnt == (size_t)SC_TILE && x_vec) {
            constexpr int NV = SC_TILE * (int)sizeof(T) / 16;
            const int4* xv = reinterpret_cast<const int4*>(x + tb);
            int4* sv = reinterpret_cast<int4*>(stage);
            int4 r[NV / SC_THREADS];
#pragma unroll
            for (int k = 0; k < NV / SC_THREADS; ++k) r[k] = ld_stream(xv + k * SC_THREADS + tid);
#pragma unroll
            for (int k = 0; k < NV / SC_THREADS; ++k) sv[k * SC_THREADS + tid] = r[k];
        } else {   // misaligned base or ragged last tile: coalesced element loads
            for (size_t i = tid; i < cnt; i += SC_THREADS) sin[i] = x[tb + i];
        }
        __syncthreads();
        T v[SC_ITEMS];
        {
            Pack<T> pk[SC_ITEMS * sizeof(T) / 16];
            const int4* sv = reinterpret_cast<const int4*>(stage) + tid * (SC_ITEMS * (int)sizeof(T) / 16);
#pragma unroll
            for (int j = 0; j < SC_ITEMS * (int)sizeof(T) / 16; ++j) pk[j] = as_pack<T>(sv[j]);
            memcpy(v, pk, sizeof(v));
        }
        const size_t g0 = tb + (size_t)tid * SC_ITEMS;
        const int nmine = g0 >= tb + cnt ? 0 : (int)((tb + cnt - g0) < (size_t)SC_ITEMS ? (tb + cnt - g0) : SC_ITEMS);
        size_t o0 = 0, r0 = g0;
        if (len < n) {
            o0 = g0 / len;
            r0 = g0 - o0 * len;
        }
        // thread aggregate
        Seg<S> me{S::identity(), 0};
        {
            size_t r = r0, o = o0;
#pragma unroll
            for (int k = 0; k < SC_ITEMS; ++k) {
                if (k < nmine) {
                    const A xv = S::lift(v[k]);
                    if (r == 0) {
                        me.v = S::comb(carry ? carry[o] : S::identity(), xv);
                        me.f = 1;
                    } else {
                        me.v = S::comb(me.v, xv);
                    }
                    if (++r == len) {
                        r = 0;
                        ++o;
                    }
                }
            }
        }
        // block scan of the thread aggregates
        Seg<S> inc = me;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            Seg<S> up{shfl_up_a(inc.v, d), __shfl_up_sync(0xffffffffu, inc.f, d)};
            if (lane >= d) inc = seg_comb<S>(up, inc);
        }
        if (lane == 31) s_warp[warp] = inc;
        Seg<S> excl{shfl_up_a(inc.v, 1), __shfl_up_sync(0xffffffffu, inc.f, 1)};
        __syncthreads();
        Seg<S> wpre{S::identity(), 0}, tagg{S::identity(), 0};
#pragma unroll
        for (int w = 0; w < SC_THREADS / 32; ++w) {
            if (w < warp) wpre = seg_comb<S>(wpre, s_warp[w]);
            tagg = seg_comb<S>(tagg, s_warp[w]);
        }
        excl = lane == 0 ? wpre : seg_comb<S>(wpre, excl);
        // publish; a tile holding a run start knows its inclusive value already
        LookbackWord* mine = lb + tile;
        if (tid == 0) {
            if (tile == 0 || tagg.f) {
                *(volatile unsigned long long*)&mine->incl = to_bits(tagg.v);
                st_release(&mine->status, LB_INCLUSIVE | ep);
            } else {
                *(volatile unsigned long long*)&mine->agg = to_bits(tagg.v);
                st_release(&mine->status, LB_PARTIAL | ep);
            }
        }
        // look-back: only when the tile's first element continues a run of an earlier tile
        const bool need = tile > 0 && (tb % len) != 0;
        if (need && warp == 0) {
            A ex = S::identity();
            long long base = (long long)tile - 1;
            for (;;) {
                const long long p = base - lane;          // lane 0 = nearest predecessor
                A val = S::identity();
                int stop = 1;
                if (p >= 0) {
                    unsigned long long st;
                    do {
                        st = ld_acquire(&lb[p].status);
                    } while ((st & LB_FLAGS) == 0 || (st & LB_EPOCH_MASK) != ep);
                    stop = (st & LB_INCLUSIVE) != 0;
                    val = from_bits<A>(stop ? *(volatile unsigned long long*)&lb[p].incl : *(volatile unsigned long long*)&lb[p].agg);
                }
                const unsigned m = __ballot_sync(0xffffffffu, stop);
                const int first = m ? __ffs(m) - 1 : 32;
                if (lane > first) val = S::identity();
                // ordered fold of the window: a higher lane is an EARLIER tile
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const A earlier = shfl_down_a(val, d);
                    if (lane + d < 32) val = S::comb(earlier, val);
                }
                ex = S::comb(val, ex);                    // valid in lane 0
                if (m) break;
                base -= 32;
            }
            if (lane == 0) {
                s_prefix = ex;
                if (!tagg.f) {
                    *(volatile unsigned long long*)&mine->incl = to_bits(S::comb(ex, tagg.v));
                    st_release(&mine->status, LB_INCLUSIVE | ep);
                }
            }
        }
        __syncthreads();
        A acc = excl.f ? excl.v : S::comb(need ? s_prefix : S::identity(), excl.v);
        Out res[SC_ITEMS];
        {
            size_t r = r0, o = o0;
#pragma unroll
            for (int k = 0; k < SC_ITEMS; ++k) {
                if (k < nmine) {
                    const A xv = S::lift(v[k]);
                    acc = r == 0 ? S::comb(carry ? carry[o] : S::identity(), xv) : S::comb(acc, xv);
                    res[k] = narrow_out<Out>(acc);
                    if (totals && r + 1 == len) totals[o] = acc;
                    if (++r == len) {
                        r = 0;
                        ++o;
                    }
                }
            }
        }
        if (y) {
            Out* sout = reinterpret_cast<Out*>(stage);
            {
                int4* sv = reinterpret_cast<int4*>(stage) + tid * (SC_ITEMS * (int)sizeof(Out) / 16);
                int4 w[SC_ITEMS * sizeof(Out) / 16];
                memcpy(w, res, sizeof(w));
#pragma unroll
                for (int j = 0; j < SC_ITEMS * (int)sizeof(Out) / 16; ++j) sv[j] = w[j];
            }
            __syncthreads();
            if (cnt == (size_t)SC_TILE && y_vec) {
                constexpr int NV = SC_TILE * (int)sizeof(Out) / 16;
                int4* yv = reinterpret_cast<int4*>(y + tb);
                const int4* sv = reinterpret_cast<const int4*>(stage);
#pragma unroll 4
                for (int k = 0; k < NV / SC_THREADS; ++k) st_stream(yv + k * SC_THREADS + tid, sv[k * SC_THREADS + tid]);
            } else {
                for (size_t i = tid; i < cnt; i += SC_THREADS) y[tb + i] = sout[i];
            }
        }
        __syncthreads();   // stage and s_tile are reused by the next tile
    }
}

// ---- inner > 1: threads along inner, sequential walk along len ---------------------------------------------------------------------
// Work item t -> (unit u = t % nunits, segment s = t / nunits); a unit is VPT consecutive outputs along inner (VEC) or one output.
// Segment 0 of output k starts from carry[k], segment s > 0 from incl[k * nseg + s - 1], the inclusive scan of the segment totals;
// either pointer may be null (the identity: pass 1 of a split folds every segment from the identity).  y == nullptr: totals mode
// (totals[k * nseg + s] = fold of the segment, segment-fastest).
template <typename T, typename Out, typename S, bool VEC>
__global__ void __launch_bounds__(SC_THREADS) scan_strided_kernel(const T* x, Out* y, size_t inner, size_t len, size_t outer, size_t nseg,
                                                                  size_t seg_len, const typename S::A* __restrict__ carry,
                                                                  const typename S::A* __restrict__ incl, typename S::A* __restrict__ totals) {
    using A = typename S::A;
    constexpr int VPT = VEC ? 16 / (int)sizeof(T) : 1;
    const size_t nout = inner * outer;
    const size_t nunits = nout / VPT;
    const size_t ivec = inner / VPT;
    const size_t items = nunits * nseg;
    for (size_t t = (size_t)blockIdx.x * SC_THREADS + threadIdx.x; t < items; t += (size_t)gridDim.x * SC_THREADS) {
        const size_t u = t % nunits, s = t / nunits;
        const size_t o = u / ivec, iu = u - o * ivec;
        const size_t k0 = o * inner + iu * VPT;                    // first output index of the unit
        const size_t lo = s * seg_len;
        const size_t hi = lo + seg_len < len ? lo + seg_len : len;
        A acc[VPT];
#pragma unroll
        for (int q = 0; q < VPT; ++q)
            acc[q] = s > 0 ? (incl ? incl[(k0 + q) * nseg + s - 1] : S::identity()) : (carry ? carry[k0 + q] : S::identity());
        const size_t base = o * len * inner + iu * VPT;             // element (i, r = 0, o)
#pragma unroll 1
        for (size_t r = lo; r < hi; ++r) {
            const size_t e = base + r * inner;
            T vv[VPT];
            if constexpr (VEC) {
                Pack<T> pk = as_pack<T>(ld_stream(reinterpret_cast<const int4*>(x + e)));
                memcpy(vv, pk.v, sizeof(vv));
            } else {
                vv[0] = x[e];
            }
#pragma unroll
            for (int q = 0; q < VPT; ++q) acc[q] = S::comb(acc[q], S::lift(vv[q]));
            if (y) {
                struct alignas(16) { Out v[VPT]; } res;
#pragma unroll
                for (int q = 0; q < VPT; ++q) res.v[q] = narrow_out<Out>(acc[q]);
                if constexpr (VEC) {
#pragma unroll
                    for (int j = 0; j < (int)(VPT * sizeof(Out) / 16); ++j)
                        st_stream(reinterpret_cast<int4*>(y + e) + j, reinterpret_cast<const int4*>(&res)[j]);
                } else {
                    y[e] = res.v[0];
                }
            }
        }
        if (totals) {
#pragma unroll
            for (int q = 0; q < VPT; ++q) totals[(k0 + q) * nseg + s] = acc[q];
        }
    }
}

template <typename S>
__global__ void fill_identity_kernel(typename S::A* __restrict__ out, size_t n) {
    for (size_t k = (size_t)blockIdx.x * SC_THREADS + threadIdx.x; k < n; k += (size_t)gridDim.x * SC_THREADS) out[k] = S::identity();
}

template <typename T, typename Out, typename S>
int32_t launch_flat(dab_ctx* ctx, const T* x, Out* y, size_t n, size_t len, const typename S::A* carry, typename S::A* totals) {
    const unsigned long long ntiles = (n + SC_TILE - 1) / SC_TILE;
    const size_t need = SC_HEAD_BYTES + (size_t)ntiles * sizeof(LookbackWord);
    if (ctx->scan_dev_bytes < need) {
        // fresh words are zero (never ready); the ticket counter restarts at 0
        int32_t st = dab_scratch_grow(ctx, &ctx->scan_dev, &ctx->scan_dev_bytes, need + need / 4, true);
        if (st != DAB_OK) return st;
        ctx->scan_tickets = 0;
    }
    unsigned long long epoch = (++ctx->scan_epoch) & ((1ull << 30) - 1ull);
    if (epoch == 0) {   // wrapped (2^30 launches): clean words, new era
        DAB_CUDA(ctx, cudaMemsetAsync((char*)ctx->scan_dev + SC_HEAD_BYTES, 0, ctx->scan_dev_bytes - SC_HEAD_BYTES, ctx->stream));
        epoch = (++ctx->scan_epoch) & ((1ull << 30) - 1ull);
    }
    auto kern = scan_flat_kernel<T, Out, S>;
    const int grid = dab_persistent_grid(ctx, kern, SC_THREADS, (size_t)ntiles);
    kern<<<grid, SC_THREADS, 0, ctx->stream>>>(x, y, n, len, carry, totals, (LookbackWord*)((char*)ctx->scan_dev + SC_HEAD_BYTES),
                                               (unsigned long long*)ctx->scan_dev, ctx->scan_tickets, epoch << 32, ntiles);
    DAB_LAUNCHED(ctx);
    ctx->scan_tickets += ntiles + (unsigned long long)grid;   // every CTA draws one ticket past the last tile
    return DAB_OK;
}

template <typename T, typename Out, typename S>
int32_t launch_strided(dab_ctx* ctx, const T* x, Out* y, size_t inner, size_t len, size_t outer, const typename S::A* carry,
                       typename S::A* totals) {
    using A = typename S::A;
    constexpr int VPT = 16 / sizeof(T);
    const bool vec = inner % VPT == 0 && ((uintptr_t)x & 15) == 0 && (!y || ((uintptr_t)y & 15) == 0);
    const size_t nout = inner * outer;
    const size_t nunits = vec ? nout / VPT : nout;
    // split len when the units cannot fill ~4 waves of resident threads; every segment keeps >= 32 rows
    const size_t want_items = (size_t)ctx->sm_count * 2048 * 4;
    size_t nseg = nunits >= want_items ? 1 : (want_items + nunits - 1) / nunits;
    const size_t max_seg = len / 32 > 0 ? len / 32 : 1;
    if (nseg > max_seg) nseg = max_seg;
    const size_t seg_len = (len + nseg - 1) / nseg;
    nseg = (len + seg_len - 1) / seg_len;
    auto run = [&](Out* yy, const A* cy, const A* incl, A* tot) -> int32_t {
        if (vec) {
            auto k = scan_strided_kernel<T, Out, S, true>;
            const int grid = dab_persistent_grid(ctx, k, SC_THREADS, (nunits * nseg + SC_THREADS - 1) / SC_THREADS);
            k<<<grid, SC_THREADS, 0, ctx->stream>>>(x, yy, inner, len, outer, nseg, seg_len, cy, incl, tot);
        } else {
            auto k = scan_strided_kernel<T, Out, S, false>;
            const int grid = dab_persistent_grid(ctx, k, SC_THREADS, (nunits * nseg + SC_THREADS - 1) / SC_THREADS);
            k<<<grid, SC_THREADS, 0, ctx->stream>>>(x, yy, inner, len, outer, nseg, seg_len, cy, incl, tot);
        }
        DAB_LAUNCHED(ctx);
        return DAB_OK;
    };
    if (nseg == 1) return run(y, carry, nullptr, totals);
    int32_t st = dab_scratch_grow(ctx, &ctx->scan_scratch, &ctx->scan_scratch_bytes, nseg * nout * sizeof(A), false);
    if (st != DAB_OK) return st;
    A* segs = (A*)ctx->scan_scratch;
    st = run(nullptr, nullptr, nullptr, segs);                           // pass 1: segment totals from the identity, [nout][nseg]
    if (st != DAB_OK) return st;
    // the segment totals of output k are run k of length nseg: ONE flat scan over all of them, in parallel (seeded by carry[k]).
    // Totals mode keeps only the last inclusive value of each run.
    using SA = ScanOp<A, S::op>;
    if (!y) return launch_flat<A, A, SA>(ctx, segs, nullptr, nout * nseg, nseg, nullptr, totals);
    st = launch_flat<A, A, SA>(ctx, segs, segs, nout * nseg, nseg, carry, nullptr);
    if (st != DAB_OK) return st;
    return run(y, carry, segs, nullptr);                                 // pass 2: each segment from its carry
}

template <typename T, typename Out, int OP>
int32_t scan_typed(dab_ctx* ctx, const void* xv, void* yv, size_t inner, size_t len, size_t outer, const void* carry, void* totals) {
    using S = ScanOp<T, OP>;
    using A = typename S::A;
    const T* x = (const T*)xv;
    Out* y = (Out*)yv;
    if (len == 0) {   // empty fibres: nothing to store; their totals are the identity
        if (totals) {
            const size_t n = inner * outer;
            fill_identity_kernel<S><<<dab_grid_for(ctx, (n + SC_THREADS - 1) / SC_THREADS, 8), SC_THREADS, 0, ctx->stream>>>((A*)totals, n);
            DAB_LAUNCHED(ctx);
        }
        return DAB_OK;
    }
    if (inner == 1) return launch_flat<T, Out, S>(ctx, x, y, len * outer, len, (const A*)carry, (A*)totals);
    return launch_strided<T, Out, S>(ctx, x, y, inner, len, outer, (const A*)carry, (A*)totals);
}

template <typename T, typename Out>
int32_t scan_op(dab_ctx* ctx, int32_t op, const void* x, void* y, size_t inner, size_t len, size_t outer, const void* carry, void* totals) {
    // only the served triples are instantiated (scan_served has already refused the others): Bool sums give Int64, every other Bool
    // scan keeps Bool, and max / min keep the element type
    constexpr bool is_bool = std::is_same<T, uint8_t>::value, same = std::is_same<T, Out>::value;
    if constexpr (!(is_bool && same)) {
        if (op == DAB_SUM) return scan_typed<T, Out, DAB_SUM>(ctx, x, y, inner, len, outer, carry, totals);
    }
    if constexpr (!(is_bool && !same)) {
        if (op == DAB_PROD) return scan_typed<T, Out, DAB_PROD>(ctx, x, y, inner, len, outer, carry, totals);
    }
    if constexpr (same) {
        if (op == DAB_MAX) return scan_typed<T, Out, DAB_MAX>(ctx, x, y, inner, len, outer, carry, totals);
        if (op == DAB_MIN) return scan_typed<T, Out, DAB_MIN>(ctx, x, y, inner, len, outer, carry, totals);
    }
    return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_scan: op %d is not served for this element type", op);
}

// the (in_dtype, op, out_dtype) triples of the result-type table of include/dab200.h
bool scan_served(int32_t in, int32_t op, int32_t out) {
    if (op < DAB_SUM || op > DAB_MIN) return false;
    const bool sp = op == DAB_SUM || op == DAB_PROD;
    switch (in) {
        case DAB_F32: case DAB_F64: case DAB_I64: return out == in;
        case DAB_I32: return out == DAB_I32 || (sp && out == DAB_I64);
        case DAB_U8: return op == DAB_SUM ? out == DAB_I64 : out == DAB_U8;
        default: return false;
    }
}

int32_t scan_entry(dab_ctx* ctx, const char* name, int32_t in, int32_t op, int32_t out, const void* x, void* y, size_t inner, size_t len,
                   size_t outer, const void* carry, void* totals) {
    DAB_ENTER(ctx);
    if (!scan_served(in, op, out))
        return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "%s: in_dtype %d, op %d, out_dtype %d is not served (no host fallback)", name, in, op, out);
    const size_t n = inner * len * outer;
    if (inner * outer == 0) return DAB_OK;
    DAB_REQUIRE(ctx, (x || n == 0) && (y || totals), DAB_ERR_ARG, "%s: null pointer", name);
    DAB_REQUIRE(ctx, !y || (const void*)y != x || dab_dtype_size(in) == dab_dtype_size(out), DAB_ERR_ARG,
                "%s: in place needs equal element sizes", name);
    switch (in) {
        case DAB_F32: return scan_op<float, float>(ctx, op, x, y, inner, len, outer, carry, totals);
        case DAB_F64: return scan_op<double, double>(ctx, op, x, y, inner, len, outer, carry, totals);
        case DAB_I64: return scan_op<long long, long long>(ctx, op, x, y, inner, len, outer, carry, totals);
        case DAB_I32:
            if (out == DAB_I64) return scan_op<int32_t, long long>(ctx, op, x, y, inner, len, outer, carry, totals);
            return scan_op<int32_t, int32_t>(ctx, op, x, y, inner, len, outer, carry, totals);
        default:
            if (out == DAB_I64) return scan_op<uint8_t, long long>(ctx, op, x, y, inner, len, outer, carry, totals);
            return scan_op<uint8_t, uint8_t>(ctx, op, x, y, inner, len, outer, carry, totals);
    }
}

}  // namespace

extern "C" {

int32_t dab_scan(dab_ctx* ctx, int32_t in_dtype, int32_t op, int32_t out_dtype, const void* x, size_t inner, size_t len, size_t outer,
                 const void* carry, void* y) {
    if (ctx && !y && inner * outer != 0) return dab_fail(ctx, DAB_ERR_ARG, "dab_scan: null pointer");
    return scan_entry(ctx, "dab_scan", in_dtype, op, out_dtype, x, y, inner, len, outer, carry, nullptr);
}

int32_t dab_scan_totals(dab_ctx* ctx, int32_t in_dtype, int32_t op, int32_t out_dtype, const void* x, size_t inner, size_t len, size_t outer,
                        void* totals) {
    if (ctx && !totals && inner * outer != 0) return dab_fail(ctx, DAB_ERR_ARG, "dab_scan_totals: null pointer");
    return scan_entry(ctx, "dab_scan_totals", in_dtype, op, out_dtype, x, nullptr, inner, len, outer, nullptr, totals);
}

int32_t dab_scan_carrier_dtype(int32_t in_dtype, int32_t op, int32_t out_dtype, int32_t* carrier_dtype) {
    if (!carrier_dtype) return DAB_ERR_ARG;
    if (!scan_served(in_dtype, op, out_dtype)) return DAB_ERR_UNSUPPORTED;
    if (op == DAB_MAX || op == DAB_MIN) *carrier_dtype = in_dtype;
    else *carrier_dtype = (in_dtype == DAB_F32 || in_dtype == DAB_F64) ? DAB_F64 : DAB_I64;
    return DAB_OK;
}

}  // extern "C"
