// dab_reducedim.cu -- K5 / K6: mapreduce(f, op, localpart(A), dims=region) as streaming sm_90a kernels.
//
// Replaces the per-worker Base.mapreducedim! at reference src/mapreduce.jl:64 (phase 1, mapreducedim_within) and :77
// (phase 2, accumulation of the gathered partials onto localpart(R) in mapreducedim_between!).
//
// The chunk is collapsed to the column-major shape (inner, reduce, outer):  out[i + inner*o] = op_r f(x[i + inner*(r + reduce*o)]).
// Roofline: HBM, sizeof(T) bytes read per element + one output element per (i, o).
//   * inner == 1  ("leading dims", e.g. sum(A, dims=1)): every output is a CONTIGUOUS run of `reduce` elements.
//       - long runs : one CTA per (run, split); 16-byte evict-first loads, 4 in flight per thread, per-run head/tail peel
//         (run starts are not 16-byte aligned when reduce % (16/sizeof T) != 0); runs are split across CTAs when there are too
//         few of them to fill the SMs, and a tiny second kernel folds the splits in order (deterministic, no atomics).
//       - short / medium runs: a sub-warp group of G lanes per run (G = #16-byte vectors in the run, <= 32), so a warp streams
//         32/G consecutive runs with 512 contiguous bytes per load instruction; flat grid.
//   * inner  > 1  (reduce over a non-leading dim): threads map along i (coalesced), each walks r with 8 independent loads in
//     flight; r is split across CTAs when inner*outer alone cannot fill the machine, then folded in order.
// Accumulators are wide (fp64 / int64) exactly as in dab_reduce.cu; float results are rounded once at the end.
#include "dab_reduce_traits.cuh"

namespace {

template <typename A, typename Out>
__device__ __forceinline__ Out narrow(A a) {
    return (Out)a;
}

// ---- leading-dims, long runs: one CTA per (run, split) -----------------------------------------------------------------
template <typename T, typename Map, typename R, typename Out>
__global__ void __launch_bounds__(RD_THREADS) rdim_lead_cta_kernel(const T* __restrict__ x, size_t red, size_t outer, int nsplit,
                                                                    Map map, typename R::A* __restrict__ partials,
                                                                    Out* __restrict__ out, int accumulate) {
    using A = typename R::A;
    using W = typename R::W;
    constexpr int VPT = 16 / sizeof(T);
    constexpr int UNROLL = 4;
    __shared__ A smem[RD_THREADS / 32];
    const size_t work = outer * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const size_t seg = w / nsplit;
        const size_t sp = w % nsplit;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        A acc = R::identity();
        if (lo < hi) {
            const T* p = x + seg * red + lo;
            const size_t n = hi - lo;
            size_t head = ((16 - ((uintptr_t)p & 15)) & 15) / sizeof(T);
            if (head > n) head = n;
            const size_t nvec = (n - head) / VPT;
            const int4* pv = reinterpret_cast<const int4*>(p + head);
            size_t i = threadIdx.x;
            for (; i + (size_t)(UNROLL - 1) * RD_THREADS < nvec; i += (size_t)UNROLL * RD_THREADS) {
                int4 r[UNROLL];
#pragma unroll
                for (int u = 0; u < UNROLL; ++u) r[u] = ld_stream(pv + i + (size_t)u * RD_THREADS);
                if constexpr (std::is_same<W, typename Map::V>::value) {
                    W tv[UNROLL];
#pragma unroll
                    for (int u = 0; u < UNROLL; ++u) {
                        Pack<T> pk = as_pack<T>(r[u]);
                        W m[VPT];
#pragma unroll
                        for (int k = 0; k < VPT; ++k) m[k] = map(pk.v[k]);
#pragma unroll
                        for (int ww = VPT; ww > 1; ww >>= 1)
#pragma unroll
                            for (int k = 0; k < ww / 2; ++k) m[k] = R::tile(m[k], m[k + ww / 2]);
                        tv[u] = m[0];
                    }
#pragma unroll
                    for (int ww = UNROLL; ww > 1; ww >>= 1)
#pragma unroll
                        for (int k = 0; k < ww / 2; ++k) tv[k] = R::tile(tv[k], tv[k + ww / 2]);
                    acc = R::comb(acc, R::lift(tv[0]));
                } else {  // widened tile (Int32 sums and products)
#pragma unroll
                    for (int u = 0; u < UNROLL; ++u) acc = fold_into<R>(acc, as_pack<T>(r[u]), map);
                }
            }
            for (; i < nvec; i += RD_THREADS) {
                Pack<T> pk = as_pack<T>(ld_stream(pv + i));
                W m = R::pre(map(pk.v[0]));
#pragma unroll
                for (int k = 1; k < VPT; ++k) m = R::tile(m, R::pre(map(pk.v[k])));
                acc = R::comb(acc, R::lift(m));
            }
            for (size_t j = threadIdx.x; j < head; j += RD_THREADS) acc = R::comb(acc, R::lift(R::pre(map(p[j]))));
            for (size_t j = head + nvec * VPT + threadIdx.x; j < n; j += RD_THREADS) acc = R::comb(acc, R::lift(R::pre(map(p[j]))));
        }
        acc = block_reduce<R>(acc, smem);
        if (threadIdx.x == 0) {
            if (nsplit == 1) {
                if (accumulate) acc = R::comb((A)out[seg], acc);
                out[seg] = narrow<A, Out>(acc);
            } else {
                partials[seg * nsplit + sp] = acc;
            }
        }
    }
}

// ---- leading-dims, short / medium runs: one sub-warp GROUP of G lanes per run --------------------------------------------------
// G lanes cooperate on one contiguous run; a warp therefore streams 32/G consecutive runs per step, i.e. 32 lanes x 16 B = 512
// contiguous bytes per load instruction when the runs are 16-byte aligned multiples of a vector (VEC == true), 128 B otherwise.
// Flat grid: CTA b owns groups_per_cta * KRUNS consecutive runs (fixed mapping, deterministic).
template <typename T, typename Map, typename R, typename Out, int G, bool VEC>
__global__ void __launch_bounds__(RD_THREADS) rdim_lead_group_kernel(const T* __restrict__ x, size_t red, size_t outer, Map map,
                                                                      Out* __restrict__ out, int accumulate, int kruns) {
    using A = typename R::A;
    using W = typename R::W;
    constexpr int VPT = 16 / sizeof(T);
    constexpr int GROUPS = RD_THREADS / G;
    const int gl = threadIdx.x % G;           // lane inside the group
    const int grp = threadIdx.x / G;          // group inside the CTA
    const size_t first = ((size_t)blockIdx.x * GROUPS + grp) * (size_t)kruns;
    if (VEC && red / VPT <= (size_t)G && kruns == 4) {
        // very short runs (at most one 16-byte vector per lane): issue the loads of all 4 runs of this group before reducing any
        // of them, so that 4 independent requests per lane are in flight instead of one load -> shuffle chain at a time
        const size_t nvec = red / VPT;
        int4 r[4];
        bool act[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const size_t seg = first + u;
            act[u] = seg < outer && (size_t)gl < nvec;
            if (act[u]) r[u] = ld_stream(reinterpret_cast<const int4*>(x + seg * red) + gl);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            A acc = R::identity();
            if (act[u]) {
                Pack<T> pk = as_pack<T>(r[u]);
                W m = R::pre(map(pk.v[0]));
#pragma unroll
                for (int k = 1; k < VPT; ++k) m = R::tile(m, R::pre(map(pk.v[k])));
                acc = R::lift(m);
            }
#pragma unroll
            for (int d = G / 2; d > 0; d >>= 1) acc = R::comb(acc, shfl_down<A>(acc, d));
            const size_t seg = first + u;
            if (gl == 0 && seg < outer) {
                if (accumulate) acc = R::comb((A)out[seg], acc);
                out[seg] = narrow<A, Out>(acc);
            }
        }
        return;
    }
#pragma unroll 1
    for (int kk = 0; kk < kruns; ++kk) {
        const size_t seg = first + kk;
        // groups past the last run stay in the loop with an empty run: the full-mask shuffles below need every lane of the warp
        const bool active = seg < outer;
        const size_t nred = active ? red : 0;
        const T* p = x + (active ? seg : 0) * red;
        A acc = R::identity();
        if (VEC) {
            const int4* pv = reinterpret_cast<const int4*>(p);
            const size_t nvec = nred / VPT;
            size_t j = gl;
            for (; j + 3 * G < nvec; j += 4 * G) {   // 4 independent 16-byte loads in flight
                int4 r[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) r[u] = ld_stream(pv + j + (size_t)u * G);
                W tv[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    Pack<T> pk = as_pack<T>(r[u]);
                    W m = R::pre(map(pk.v[0]));
#pragma unroll
                    for (int k = 1; k < VPT; ++k) m = R::tile(m, R::pre(map(pk.v[k])));
                    tv[u] = m;
                }
                acc = R::comb(acc, R::lift(R::tile(R::tile(tv[0], tv[1]), R::tile(tv[2], tv[3]))));
            }
            for (; j < nvec; j += G) {
                Pack<T> pk = as_pack<T>(ld_stream(pv + j));
                W m = R::pre(map(pk.v[0]));
#pragma unroll
                for (int k = 1; k < VPT; ++k) m = R::tile(m, R::pre(map(pk.v[k])));
                acc = R::comb(acc, R::lift(m));
            }
        } else {
            size_t j = gl;
            for (; j + 3 * G < nred; j += 4 * G) {
                T a0 = p[j], a1 = p[j + G], a2 = p[j + 2 * G], a3 = p[j + 3 * G];
                acc = R::comb(acc, R::lift(R::tile(R::tile(R::pre(map(a0)), R::pre(map(a1))), R::tile(R::pre(map(a2)), R::pre(map(a3))))));
            }
            for (; j < nred; j += G) acc = R::comb(acc, R::lift(R::pre(map(p[j]))));
        }
#pragma unroll
        for (int d = G / 2; d > 0; d >>= 1) acc = R::comb(acc, shfl_down<A>(acc, d));  // stays inside the G-lane group
        if (active && gl == 0) {
            if (accumulate) acc = R::comb((A)out[seg], acc);
            out[seg] = narrow<A, Out>(acc);
        }
    }
}

template <typename T, typename Map, typename R, typename Out, int G>
int32_t launch_group(dab_ctx* ctx, const T* x, size_t red, size_t outer, Map map, Out* out, int accumulate) {
    constexpr int VPT = 16 / sizeof(T);
    const bool vec = (red % VPT == 0) && (((uintptr_t)x & 15) == 0);
    const int groups = RD_THREADS / G;
    int kruns = 4;
    size_t grid = (outer + (size_t)groups * kruns - 1) / ((size_t)groups * kruns);
    if (grid > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_ARG, "too many runs for one launch");
    if (vec) rdim_lead_group_kernel<T, Map, R, Out, G, true><<<(unsigned)grid, RD_THREADS, 0, ctx->stream>>>(x, red, outer, map, out, accumulate, kruns);
    else rdim_lead_group_kernel<T, Map, R, Out, G, false><<<(unsigned)grid, RD_THREADS, 0, ctx->stream>>>(x, red, outer, map, out, accumulate, kruns);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// ---- non-leading dim: threads along i, loop over r --------------------------------------------------------------------------
template <typename T, typename Map, typename R, typename Out>
__global__ void __launch_bounds__(RD_THREADS) rdim_strided_kernel(const T* __restrict__ x, size_t inner, size_t red, size_t outer,
                                                                   int nsplit, Map map, typename R::A* __restrict__ partials,
                                                                   Out* __restrict__ out, int accumulate) {
    using A = typename R::A;
    constexpr int UNROLL = 8;
    // threads cover the flattened output index k = i + inner*o (i fastest): full CTAs even when `inner` is small
    const size_t nout = inner * outer;
    const size_t kblocks = (nout + RD_THREADS - 1) / RD_THREADS;
    const size_t work = kblocks * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const size_t kb = w % kblocks;
        const size_t sp = w / kblocks;
        const size_t k = kb * RD_THREADS + threadIdx.x;
        if (k >= nout) continue;
        const size_t o = k / inner;
        const size_t i = k - o * inner;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        const T* p = x + i + inner * (o * red);
        A acc = R::identity();
        size_t r = lo;
        for (; r + UNROLL <= hi; r += UNROLL) {
            T v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = __ldcs(p + (r + u) * inner);
            typename R::W m[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) m[u] = R::pre(map(v[u]));
#pragma unroll
            for (int ww = UNROLL; ww > 1; ww >>= 1)
#pragma unroll
                for (int q = 0; q < ww / 2; ++q) m[q] = R::tile(m[q], m[q + ww / 2]);
            acc = R::comb(acc, R::lift(m[0]));
        }
        for (; r < hi; ++r) acc = R::comb(acc, R::lift(R::pre(map(__ldcs(p + r * inner)))));
        if (nsplit == 1) {
            if (accumulate) acc = R::comb((A)out[k], acc);
            out[k] = narrow<A, Out>(acc);
        } else {
            partials[sp * nout + k] = acc;
        }
    }
}

// ---- non-leading dim, vectorised: each thread owns 16 bytes (VPT consecutive outputs along `inner`) and walks r with 16-byte loads
// (512 contiguous bytes per warp load instruction); needs inner % VPT == 0 and a 16-byte aligned base
template <typename T, typename Map, typename R, typename Out>
__global__ void __launch_bounds__(RD_THREADS) rdim_strided_vec_kernel(const T* __restrict__ x, size_t inner, size_t red, size_t outer,
                                                                       int nsplit, Map map, typename R::A* __restrict__ partials,
                                                                       Out* __restrict__ out, int accumulate) {
    using A = typename R::A;
    constexpr int VPT = 16 / sizeof(T);
    constexpr int UNROLL = 4;
    const size_t nout = inner * outer;
    const size_t nvout = nout / VPT;                 // vectors of outputs
    const size_t ivec = inner / VPT;                 // vectors per column
    const size_t kblocks = (nvout + RD_THREADS - 1) / RD_THREADS;
    const size_t work = kblocks * (size_t)nsplit;
    const size_t split_len = (red + nsplit - 1) / nsplit;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const size_t kb = w % kblocks;
        const size_t sp = w / kblocks;
        const size_t kv = kb * RD_THREADS + threadIdx.x;
        if (kv >= nvout) continue;
        const size_t o = kv / ivec;
        const size_t iv = kv - o * ivec;
        size_t lo = sp * split_len, hi = lo + split_len;
        if (hi > red) hi = red;
        const int4* p = reinterpret_cast<const int4*>(x + inner * (o * red)) + iv;   // + r * ivec per step in r
        A acc[VPT];
#pragma unroll
        for (int k = 0; k < VPT; ++k) acc[k] = R::identity();
        size_t r = lo;
        for (; r + UNROLL <= hi; r += UNROLL) {
            int4 v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = ld_stream(p + (r + u) * ivec);
            typename R::W m[UNROLL][VPT];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                Pack<T> pk = as_pack<T>(v[u]);
#pragma unroll
                for (int k = 0; k < VPT; ++k) m[u][k] = R::pre(map(pk.v[k]));
            }
#pragma unroll
            for (int k = 0; k < VPT; ++k) {
                auto t = R::tile(R::tile(m[0][k], m[1][k]), R::tile(m[2][k], m[3][k]));
                acc[k] = R::comb(acc[k], R::lift(t));
            }
        }
        for (; r < hi; ++r) {
            Pack<T> pk = as_pack<T>(ld_stream(p + r * ivec));
#pragma unroll
            for (int k = 0; k < VPT; ++k) acc[k] = R::comb(acc[k], R::lift(R::pre(map(pk.v[k]))));
        }
        const size_t k0 = kv * VPT;
#pragma unroll
        for (int k = 0; k < VPT; ++k) {
            if (nsplit == 1) {
                A a = acc[k];
                if (accumulate) a = R::comb((A)out[k0 + k], a);
                out[k0 + k] = narrow<A, Out>(a);
            } else {
                partials[sp * nout + k0 + k] = acc[k];
            }
        }
    }
}

// ---- ordered fold of the split partials: thread per output -----------------------------------------------------------------
template <typename R, typename Out>
__global__ void __launch_bounds__(RD_THREADS) rdim_finish_kernel(const typename R::A* __restrict__ partials, size_t nout, int nsplit,
                                                                  size_t stride_out, size_t stride_split, Out* __restrict__ out,
                                                                  int accumulate) {
    using A = typename R::A;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < nout; k += stride) {
        A acc = accumulate ? (A)out[k] : R::identity();
        for (int s = 0; s < nsplit; ++s) acc = R::comb(acc, partials[k * stride_out + (size_t)s * stride_split]);
        out[k] = (Out)acc;
    }
}

template <typename T, typename Map, typename R, typename Out>
int32_t launch_rdim(dab_ctx* ctx, const T* x, size_t inner, size_t red, size_t outer, Map map, Out* out, int accumulate) {
    using A = typename R::A;
    const size_t target_ctas = (size_t)ctx->sm_count * 8;
    if (inner == 1) {
        if (red < 4096 && outer >= (size_t)ctx->sm_count * 8) {
            // lanes per run: as many as the run has 16-byte vectors (power of two, <= 32)
            constexpr int VPT = 16 / sizeof(T);
            size_t units = red / VPT;
            if (units >= 32) return launch_group<T, Map, R, Out, 32>(ctx, x, red, outer, map, out, accumulate);
            if (units >= 16) return launch_group<T, Map, R, Out, 16>(ctx, x, red, outer, map, out, accumulate);
            if (units >= 8) return launch_group<T, Map, R, Out, 8>(ctx, x, red, outer, map, out, accumulate);
            if (units >= 4) return launch_group<T, Map, R, Out, 4>(ctx, x, red, outer, map, out, accumulate);
            return launch_group<T, Map, R, Out, 2>(ctx, x, red, outer, map, out, accumulate);
        }
        // split long runs when there are too few of them; keep every split >= 16 KiB of input
        const int nsplit = dim_nsplit(outer, target_ctas, red * sizeof(T) / 16384);
        A* partials = nullptr;
        if (nsplit > 1) {
            int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, outer * (size_t)nsplit * sizeof(A), false);
            if (st != DAB_OK) return st;
            partials = (A*)ctx->dim_scratch;
        }
        int grid = dab_persistent_grid(ctx, rdim_lead_cta_kernel<T, Map, R, Out>, RD_THREADS, outer * (size_t)nsplit);
        rdim_lead_cta_kernel<T, Map, R, Out><<<grid, RD_THREADS, 0, ctx->stream>>>(x, red, outer, nsplit, map, partials, out, accumulate);
        DAB_LAUNCHED(ctx);
        if (nsplit > 1) {
            int g2 = dab_grid_for(ctx, (outer + RD_THREADS - 1) / RD_THREADS, 8);
            rdim_finish_kernel<R, Out><<<g2, RD_THREADS, 0, ctx->stream>>>(partials, outer, nsplit, (size_t)nsplit, 1, out, accumulate);
            DAB_LAUNCHED(ctx);
        }
        return DAB_OK;
    }
    // 16-byte path when whole vectors of outputs line up; needs enough vector-outputs to be worth it
    const bool vec = (inner % (16 / sizeof(T)) == 0) && (((uintptr_t)x & 15) == 0) && (inner * outer / (16 / sizeof(T)) >= 4096);
    size_t base_ctas = vec ? (inner * outer / (16 / sizeof(T)) + RD_THREADS - 1) / RD_THREADS : (inner * outer + RD_THREADS - 1) / RD_THREADS;
    // split r so that the work items fill >= 4 waves of the persistent grid (a 1.08-wave launch loses ~45 % to the tail), while
    // every split keeps >= 256 rows so that the partial buffer stays < 1 % of the input
    const int nsplit = dim_nsplit(base_ctas, 4 * target_ctas, red / 256);
    A* partials = nullptr;
    if (nsplit > 1) {
        int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, inner * outer * (size_t)nsplit * sizeof(A), false);
        if (st != DAB_OK) return st;
        partials = (A*)ctx->dim_scratch;
    }
    if (vec) {
        int grid = dab_persistent_grid(ctx, rdim_strided_vec_kernel<T, Map, R, Out>, RD_THREADS, base_ctas * (size_t)nsplit);
        rdim_strided_vec_kernel<T, Map, R, Out><<<grid, RD_THREADS, 0, ctx->stream>>>(x, inner, red, outer, nsplit, map, partials, out, accumulate);
    } else {
        int grid = dab_persistent_grid(ctx, rdim_strided_kernel<T, Map, R, Out>, RD_THREADS, base_ctas * (size_t)nsplit);
        rdim_strided_kernel<T, Map, R, Out><<<grid, RD_THREADS, 0, ctx->stream>>>(x, inner, red, outer, nsplit, map, partials, out, accumulate);
    }
    DAB_LAUNCHED(ctx);
    if (nsplit > 1) {
        size_t nout = inner * outer;
        int g2 = dab_grid_for(ctx, (nout + RD_THREADS - 1) / RD_THREADS, 8);
        rdim_finish_kernel<R, Out><<<g2, RD_THREADS, 0, ctx->stream>>>(partials, nout, nsplit, 1, nout, out, accumulate);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

// out[0] (op)= S: lands the result of the flat whole-chunk reduce kernel when the "dimensional" reduction is really a full reduction
// (inner == outer == 1).  Accumulating a float SUM / PROD combines out[0] with the un-rounded fp64 carrier S at slot bytes [8, 16) and
// rounds once, as the launch_rdim kernels do; combining with the rounded slot[0] would round twice.
__device__ __forceinline__ double slot_carrier(const void* slot) { return *reinterpret_cast<const double*>((const char*)slot + 8); }

template <typename Out>
__global__ void scalar_into_kernel(const Out* __restrict__ slot, Out* __restrict__ out, int accumulate, int op) {
    Out v = *slot;
    if (accumulate) {
        Out o = *out;
        if constexpr (std::is_same<Out, float>::value) {
            if (op == DAB_SUM || op == DAB_PROD) {
                const double s = slot_carrier(slot);
                *out = (float)(op == DAB_SUM ? jl::add((double)o, s) : jl::mul((double)o, s));
                return;
            }
        }
        switch (op) {
            case DAB_SUM: v = jl::add(o, v); break;
            case DAB_PROD: v = jl::mul(o, v); break;
            case DAB_MAX: v = jl::max(o, v); break;
            default: v = jl::min(o, v); break;
        }
    }
    *out = v;
}

// Float16 result of a full reduction in disguise (see dab_reducedim); accumulate rounds op(out, S) once to Float16: SUM / PROD in the fp64
// carrier, MAX / MIN exactly in Float32
__global__ void half_into_kernel(const Half* __restrict__ slot, Half* __restrict__ out, int accumulate, int op) {
    Half v = *slot;
    if (accumulate) {
        const float o = (float)*out, w = (float)v;
        switch (op) {
            case DAB_SUM: v = Half(jl::add((double)o, slot_carrier(slot))); break;
            case DAB_PROD: v = Half(jl::mul((double)o, slot_carrier(slot))); break;
            case DAB_MAX: v = Half(jl::max(o, w)); break;
            default: v = Half(jl::min(o, w)); break;
        }
    }
    *out = v;
}

template <typename T>
using ResultOfSum = typename std::conditional<std::is_floating_point<T>::value, T, long long>::type;

template <typename T, int FN>
int32_t rdim_map(dab_ctx* ctx, int32_t op, const T* x, size_t inner, size_t red, size_t outer, void* out, int accumulate) {
    MapF<T, FN> map{(T)0};
    switch (op) {
        case DAB_SUM:
            return launch_rdim<T, MapF<T, FN>, SumTraits<T>, ResultOfSum<T>>(ctx, x, inner, red, outer, map, (ResultOfSum<T>*)out, accumulate);
        case DAB_PROD:
            return launch_rdim<T, MapF<T, FN>, ProdTraits<T>, ResultOfSum<T>>(ctx, x, inner, red, outer, map, (ResultOfSum<T>*)out, accumulate);
        case DAB_MAX: return launch_rdim<T, MapF<T, FN>, MaxTraits<T>, T>(ctx, x, inner, red, outer, map, (T*)out, accumulate);
        case DAB_MIN: return launch_rdim<T, MapF<T, FN>, MinTraits<T>, T>(ctx, x, inner, red, outer, map, (T*)out, accumulate);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reducedim: op %d not served (no host fallback)", op);
    }
}

template <typename T>
int32_t rdim_t(dab_ctx* ctx, int32_t op, int32_t map, const T* x, size_t inner, size_t red, size_t outer, void* out, int accumulate) {
    switch (map) {
        case DAB_MAP_ID: return rdim_map<T, DAB_MAP_ID>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_ABS: return rdim_map<T, DAB_MAP_ABS>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_ABS2: return rdim_map<T, DAB_MAP_ABS2>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_NEG: return rdim_map<T, DAB_MAP_NEG>(ctx, op, x, inner, red, outer, out, accumulate);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reducedim: map %d not served (no host fallback)", map);
    }
}

// Float16 chunks: Half elements widened to Float32 by the map (HMapF), Float32 / fp64 traits as for Float32, Float16 output
template <int FN>
int32_t rdim_h_map(dab_ctx* ctx, int32_t op, const Half* x, size_t inner, size_t red, size_t outer, void* out, int accumulate) {
    using M = HMapF<FN>;
    const M map{};
    Half* o = (Half*)out;
    switch (op) {
        case DAB_SUM: return launch_rdim<Half, M, SumTraits<float>, Half>(ctx, x, inner, red, outer, map, o, accumulate);
        case DAB_PROD: return launch_rdim<Half, M, ProdTraits<float>, Half>(ctx, x, inner, red, outer, map, o, accumulate);
        case DAB_MAX: return launch_rdim<Half, M, MaxTraits<float>, Half>(ctx, x, inner, red, outer, map, o, accumulate);
        case DAB_MIN: return launch_rdim<Half, M, MinTraits<float>, Half>(ctx, x, inner, red, outer, map, o, accumulate);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reducedim: op %d not served for Float16 (no host fallback)", op);
    }
}

int32_t rdim_h(dab_ctx* ctx, int32_t op, int32_t map, const Half* x, size_t inner, size_t red, size_t outer, void* out, int accumulate) {
    switch (map) {
        case DAB_MAP_ID: return rdim_h_map<DAB_MAP_ID>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_ABS: return rdim_h_map<DAB_MAP_ABS>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_ABS2: return rdim_h_map<DAB_MAP_ABS2>(ctx, op, x, inner, red, outer, out, accumulate);
        case DAB_MAP_NEG: return rdim_h_map<DAB_MAP_NEG>(ctx, op, x, inner, red, outer, out, accumulate);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reducedim: map %d not served for Float16 (no host fallback)", map);
    }
}

}  // namespace

extern "C" {

int32_t dab_reducedim(dab_ctx* ctx, int32_t dtype, int32_t op, int32_t map, const void* x, size_t inner, size_t reduce, size_t outer,
                      void* out, int32_t accumulate) {
    if (dtype == DAB_C64 || dtype == DAB_C128) {
        // Complex{T}: Julia's + is componentwise, so a complex SUM over (inner, reduce, outer) IS the real SUM over (2 inner, reduce, outer)
        // of the interleaved components.  No other op or map is served for the complex codes.
        if (op != DAB_SUM || map != DAB_MAP_ID)
            return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_reducedim: op %d with map %d is not served for complex dtype %d (%s; SUM with MAP_ID is)",
                            op, map, dtype, dtype == DAB_C64 ? "ComplexF32" : "ComplexF64");
        return dab_reducedim(ctx, dtype == DAB_C64 ? DAB_F32 : DAB_F64, op, map, x, 2 * inner, reduce, outer, out, accumulate);
    }
    DAB_ENTER(ctx);
    const size_t nout = inner * outer;
    if (nout == 0) return DAB_OK;
    DAB_REQUIRE(ctx, out && (x || reduce == 0), DAB_ERR_ARG, "dab_reducedim: null pointer");
    if (reduce == 0) {
        // reducing over an empty dimension: SUM/PROD give the identity, MAX/MIN throw (Base semantics)
        if (accumulate) return DAB_OK;
        if (op != DAB_SUM && op != DAB_PROD) return dab_fail(ctx, DAB_ERR_EMPTY, "reducing over an empty collection is not allowed");
        int32_t rdt;
        dab_reduce_result_dtype(dtype, op, map, &rdt);
        unsigned char v[8] = {0};
        if (op == DAB_PROD) {
            if (rdt == DAB_F32) { float o = 1.f; memcpy(v, &o, 4); }
            else if (rdt == DAB_F64) { double o = 1.0; memcpy(v, &o, 8); }
            else if (rdt == DAB_F16) { const unsigned short o = 0x3c00; memcpy(v, &o, 2); }
            else { long long o = 1; memcpy(v, &o, 8); }
        }
        return dab_fill(ctx, rdt, out, nout, v);
    }
    if (inner == 1 && outer == 1 && reduce >= (1u << 16) && (map == DAB_MAP_ID || map == DAB_MAP_ABS || map == DAB_MAP_ABS2 || map == DAB_MAP_NEG) &&
        op <= DAB_MIN) {
        // a full reduction in disguise (e.g. sum(v, dims=1) of a vector, dims=(1,2) of a matrix): use the flat streaming kernel
        int32_t st = dab_reduce(ctx, dtype, op, map, nullptr, x, reduce, ctx->result_slot);
        if (st != DAB_OK) return st;
        int32_t rdt;
        dab_reduce_result_dtype(dtype, op, map, &rdt);
        switch (rdt) {
            case DAB_F32: scalar_into_kernel<float><<<1, 1, 0, ctx->stream>>>((const float*)ctx->result_slot, (float*)out, accumulate, op); break;
            case DAB_F64: scalar_into_kernel<double><<<1, 1, 0, ctx->stream>>>((const double*)ctx->result_slot, (double*)out, accumulate, op); break;
            case DAB_I32: scalar_into_kernel<int32_t><<<1, 1, 0, ctx->stream>>>((const int32_t*)ctx->result_slot, (int32_t*)out, accumulate, op); break;
            case DAB_F16: half_into_kernel<<<1, 1, 0, ctx->stream>>>((const Half*)ctx->result_slot, (Half*)out, accumulate, op); break;
            default: scalar_into_kernel<long long><<<1, 1, 0, ctx->stream>>>((const long long*)ctx->result_slot, (long long*)out, accumulate, op); break;
        }
        DAB_LAUNCHED(ctx);
        return DAB_OK;
    }
    switch (dtype) {
        case DAB_F32: return rdim_t<float>(ctx, op, map, (const float*)x, inner, reduce, outer, out, accumulate);
        case DAB_F64: return rdim_t<double>(ctx, op, map, (const double*)x, inner, reduce, outer, out, accumulate);
        case DAB_I32: return rdim_t<int32_t>(ctx, op, map, (const int32_t*)x, inner, reduce, outer, out, accumulate);
        case DAB_I64: return rdim_t<long long>(ctx, op, map, (const long long*)x, inner, reduce, outer, out, accumulate);
        case DAB_F16:
            DAB_REQUIRE(ctx, (uintptr_t)x % 2 == 0 && (uintptr_t)out % 2 == 0, DAB_ERR_ARG, "dab_reducedim: Float16 data needs 2-byte alignment");
            return rdim_h(ctx, op, map, (const Half*)x, inner, reduce, outer, out, accumulate);
        default: return dab_fail(ctx, DAB_ERR_ARG, "dab_reducedim: bad dtype %d", dtype);
    }
}

}  // extern "C"
