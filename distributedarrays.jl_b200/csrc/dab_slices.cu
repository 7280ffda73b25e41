// dab_slices.cu -- slice functions of mapslices(f, D; dims) (reference src/mapreduce.jl:191-208) that need kernels of their own:
//   dab_sort_slices      sort every fibre x[i + inner*(r + len*o)], r < len, independently (f = sort, one slice dimension)
//   dab_svdvals_batched  singular values of a batch of small dense matrices (f = svdvals, two slice dimensions)
// The per-element code (bitonic compare/exchange, round-robin pairing, Jacobi rotation) lives in dab_slices_core.cuh.
#include <map>
#include <mutex>
#include <utility>

#include "dab_common.cuh"
#include "dab_slices_core.cuh"

namespace {

// ---- segmented sort ---------------------------------------------------------------------------------------------------------------
// One CTA sorts a GROUP of B fibres in shared memory: B = SS_CAP / (P2 + 1) fibres of P2 = next power of two >= len keys.
//   inner == 1: the group is B consecutive fibres, one contiguous run of B * len elements;
//   inner  > 1: the group is B fibres with adjacent i and the same o, so every r is one contiguous row of B elements.  Rows are staged
//               transposed (fibre-major, P2 + 1 keys apart: consecutive threads hit consecutive banks).
// Keys are encoded with SortKey<T>::enc on the way in (unsigned order == isless), padded with all-ones keys, sorted by a bitonic network
// (one __syncthreads per (k, j) stage) and decoded on the way out.  Equal keys have equal bits, so the result is the unique ascending
// arrangement of the fibre's bit patterns: the same bits dab_sort writes.
constexpr int SS_THREADS = 512;
constexpr unsigned int SS_CAP = DAB_SORT_SLICES_SMEM_LEN + 64;   // keys of shared memory per CTA (fibre pads included)

template <typename T>
__global__ void __launch_bounds__(SS_THREADS) sort_slices_kernel(const typename SortKey<T>::U* in, typename SortKey<T>::U* out, size_t inner,
                                                                  unsigned int len, size_t outer, unsigned int log2p2, unsigned int B,
                                                                  size_t ngroups) {
    using K = SortKey<T>;
    using U = typename K::U;
    extern __shared__ __align__(16) unsigned char ss_smem[];
    U* s = reinterpret_cast<U*>(ss_smem);
    const unsigned int p2 = 1u << log2p2, S = p2 + 1u;
    const size_t gpo = (inner + B - 1) / B;                       // groups per o when inner > 1
    for (size_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
        size_t base;
        unsigned int nf;
        if (inner == 1) {
            const size_t o0 = g * B;
            nf = (unsigned int)(outer - o0 < B ? outer - o0 : B);
            base = o0 * len;
            for (unsigned int t = threadIdx.x; t < nf * len; t += SS_THREADS) {
                const unsigned int b = t / len, r = t - b * len;
                s[b * S + r] = K::enc(in[base + t]);
            }
        } else {
            const size_t o = g / gpo, i0 = (g - o * gpo) * B;
            nf = (unsigned int)(inner - i0 < B ? inner - i0 : B);
            base = o * inner * len + i0;
            for (unsigned int t = threadIdx.x; t < nf * len; t += SS_THREADS) {
                const unsigned int r = t / nf, b = t - r * nf;
                s[b * S + r] = K::enc(in[base + (size_t)r * inner + b]);
            }
        }
        if (len < p2)
            for (unsigned int t = threadIdx.x; t < nf * p2; t += SS_THREADS) {
                const unsigned int b = t >> log2p2, r = t & (p2 - 1u);
                if (r >= len) s[b * S + r] = slices_pad_key<U>();
            }
        __syncthreads();
        const unsigned int half = (nf * p2) >> 1;
        for (unsigned int k = 2; k <= p2; k <<= 1)
            for (unsigned int j = k >> 1; j > 0; j >>= 1) {
                for (unsigned int p = threadIdx.x; p < half; p += SS_THREADS) {
                    const unsigned int i = slices_bitonic_lo(p, j);
                    U& a = s[slices_smem_index(i, log2p2)];
                    U& c = s[slices_smem_index(i + j, log2p2)];
                    U x = a, y = c;
                    slices_cmpx(x, y, slices_bitonic_asc(i, k, p2));
                    a = x;
                    c = y;
                }
                __syncthreads();
            }
        if (inner == 1) {
            for (unsigned int t = threadIdx.x; t < nf * len; t += SS_THREADS) {
                const unsigned int b = t / len, r = t - b * len;
                out[base + t] = K::dec(s[b * S + r]);
            }
        } else {
            for (unsigned int t = threadIdx.x; t < nf * len; t += SS_THREADS) {
                const unsigned int r = t / nf, b = t - r * nf;
                out[base + (size_t)r * inner + b] = K::dec(s[b * S + r]);
            }
        }
        __syncthreads();                                          // shared memory is reused by the next group
    }
}

template <typename T>
int32_t sort_slices_smem(dab_ctx* ctx, const void* in, void* out, size_t inner, size_t len, size_t outer) {
    using U = typename SortKey<T>::U;
    const unsigned int log2p2 = slices_log2_ceil(len);
    const unsigned int B = SS_CAP / ((1u << log2p2) + 1u);
    const size_t nfib_groups = inner == 1 ? (outer + B - 1) / B : ((inner + B - 1) / B) * outer;
    auto kern = sort_slices_kernel<T>;
    constexpr size_t max_smem = (size_t)SS_CAP * sizeof(U);
    int per_sm = 0;
    {   // >48 KiB of dynamic shared memory is an opt-in attribute of the (kernel, device) pair
        static std::mutex mu;
        static std::map<std::pair<const void*, int>, int> seen;
        std::lock_guard<std::mutex> lk(mu);
        auto key = std::make_pair((const void*)kern, ctx->device);
        auto it = seen.find(key);
        if (it == seen.end()) {
            DAB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem));
            int nb = 0;
            DAB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, SS_THREADS, max_smem));
            it = seen.emplace(key, nb < 1 ? 1 : nb).first;
        }
        per_sm = it->second;
    }
    const size_t smem = (size_t)B * ((1u << log2p2) + 1u) * sizeof(U);
    const int grid = dab_grid_for(ctx, nfib_groups, per_sm * 4);
    kern<<<grid, SS_THREADS, smem, ctx->stream>>>((const U*)in, (U*)out, inner, (unsigned int)len, outer, log2p2, B, nfib_groups);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// Fibres longer than shared memory: K11 per fibre.  inner == 1: each fibre is contiguous already; inner > 1: every o-slab is transposed
// (dab_transpose_box) into a contiguous temporary, its fibres sorted in place, and transposed back.  Scratch comes from the ctx block cache.
int32_t sort_slices_k11(dab_ctx* ctx, int32_t dtype, const void* in, void* out, size_t inner, size_t len, size_t outer) {
    const size_t es = dab_dtype_size(dtype);
    void* tmp = nullptr;
    void* slab = nullptr;
    int32_t st = dab_alloc(ctx, len * es, &tmp);
    if (st == DAB_OK && inner > 1) st = dab_alloc(ctx, inner * len * es, &slab);
    for (size_t o = 0; st == DAB_OK && o < outer; ++o) {
        const char* src = (const char*)in + o * inner * len * es;
        char* dst = (char*)out + o * inner * len * es;
        if (inner == 1) {
            st = dab_sort(ctx, dtype, src, dst, tmp, len);
            continue;
        }
        st = dab_transpose_box(ctx, (int32_t)es, slab, len, src, inner, inner, len);   // slab[r + len*i] = src[i + inner*r]
        for (size_t i = 0; st == DAB_OK && i < inner; ++i) {
            char* f = (char*)slab + i * len * es;
            st = dab_sort(ctx, dtype, f, f, tmp, len);
        }
        if (st == DAB_OK) st = dab_transpose_box(ctx, (int32_t)es, dst, inner, slab, len, len, inner);
    }
    char keep[512];
    memcpy(keep, ctx->err, sizeof keep);                          // the frees must not overwrite the text of a failure
    if (slab) dab_free(ctx, slab);
    if (tmp) dab_free(ctx, tmp);
    memcpy(ctx->err, keep, sizeof keep);
    return st;
}

// ---- batched singular values ------------------------------------------------------------------------------------------------------
// One CTA per matrix (grid-stride over the batch), the matrix in shared memory as fp64, in the orientation with nc = min(m, n) <= 32
// columns (A itself, or A^T when n > m).  A sweep is np - 1 rounds of round-robin pairs; warp k rotates pair k of the round (lanes over
// rows, shuffle-reduced dot products).  Sweeps stop when no pair needed a rotation, or after DAB_SVD_MAX_SWEEPS.  The singular values are
// the column norms, ranked descending in the kernel.  A NaN or Inf found while loading sets *status and yields NaNs for that matrix.
// The matrix is scaled by a power of two to max |a| in [0.5, 1) before the sweeps (slices_scale_exp), the norms scaled back after.
constexpr int SVD_MAX_ELEMS = 4096;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <typename T>
__global__ void __launch_bounds__(512) svdvals_kernel(const T* __restrict__ A, int m, int n, size_t batch, T* __restrict__ S,
                                                      int32_t* __restrict__ status) {
    __shared__ double W[SVD_MAX_ELEMS];
    __shared__ double nrm[32];
    __shared__ double s_wmax[16];
    __shared__ int s_bad, s_rot;
    const bool tr = n > m;
    const int M = tr ? n : m, nc = tr ? m : n, np = nc + (nc & 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int mn = m * n;
    const double tol = slices_jacobi_tol(M);
    for (size_t b = blockIdx.x; b < batch; b += gridDim.x) {
        const T* a = A + b * (size_t)mn;
        if (threadIdx.x == 0) s_bad = 0;
        __syncthreads();
        int bad = 0;
        double amax = 0.0;
        for (int t = threadIdx.x; t < mn; t += blockDim.x) {
            const double v = (double)a[t];
            if (!isfinite(v)) bad = 1;
            amax = fmax(amax, fabs(v));
            const int row = t % m, col = t / m;
            W[tr ? col + M * row : t] = v;                      // W(r, c), column-major with M rows
        }
        if (bad) s_bad = 1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0) s_wmax[warp] = amax;
        __syncthreads();
        if (s_bad) {
            if (threadIdx.x < nc) S[b * nc + threadIdx.x] = (T)NAN;
            if (threadIdx.x == 0) *status = 1;
            __syncthreads();
            continue;
        }
        amax = 0.0;
        for (int w = 0; w < nwarps; ++w) amax = fmax(amax, s_wmax[w]);
        const int e = slices_scale_exp(amax);
        for (int t = threadIdx.x; t < mn; t += blockDim.x) W[t] = ldexp(W[t], -e);
        __syncthreads();
        for (int sweep = 0; sweep < DAB_SVD_MAX_SWEEPS; ++sweep) {
            if (threadIdx.x == 0) s_rot = 0;
            __syncthreads();
            for (int r = 0; r < np - 1; ++r) {
                for (int k = warp; k < np / 2; k += nwarps) {
                    int p, q;
                    slices_rr_pair(np, r, k, &p, &q);
                    if (p >= nc || q >= nc) continue;
                    double al = 0.0, be = 0.0, ga = 0.0;
                    for (int i = lane; i < M; i += 32) {
                        const double x = W[i + M * p], y = W[i + M * q];
                        al += x * x;
                        be += y * y;
                        ga += x * y;
                    }
                    al = warp_sum(al);
                    be = warp_sum(be);
                    ga = warp_sum(ga);
                    double c, s;
                    if (slices_jacobi_rotation(al, be, ga, tol, &c, &s)) {
                        if (lane == 0) s_rot = 1;
                        for (int i = lane; i < M; i += 32) slices_jacobi_apply(&W[i + M * p], &W[i + M * q], c, s);
                    }
                }
                __syncthreads();
            }
            const int rot = s_rot;
            __syncthreads();                                      // everybody has read s_rot before it is cleared again
            if (!rot) break;
        }
        for (int c = warp; c < nc; c += nwarps) {
            double ss = 0.0;
            for (int i = lane; i < M; i += 32) ss += W[i + M * c] * W[i + M * c];
            ss = warp_sum(ss);
            if (lane == 0) nrm[c] = ldexp(sqrt(ss), e);
        }
        __syncthreads();
        if (threadIdx.x < nc) {
            const double v = nrm[threadIdx.x];
            int rank = 0;
            for (int j = 0; j < nc; ++j) rank += nrm[j] > v || (nrm[j] == v && j < (int)threadIdx.x);
            S[b * nc + rank] = (T)v;
        }
        __syncthreads();
    }
}

template <typename T>
int32_t svdvals_t(dab_ctx* ctx, const void* A, size_t m, size_t n, size_t batch, void* S, int32_t* status) {
    const int nc = (int)(m < n ? m : n), np = nc + (nc & 1);
    const int threads = 32 * (np / 2 > 1 ? (np / 2 < 16 ? np / 2 : 16) : 1);
    const int grid = dab_grid_for(ctx, batch, 2048 / threads < 8 ? 2048 / threads : 8);
    svdvals_kernel<T><<<grid, threads, 0, ctx->stream>>>((const T*)A, (int)m, (int)n, batch, (T*)S, status);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_sort_slices(dab_ctx* ctx, int32_t dtype, const void* in, void* out, size_t inner, size_t len, size_t outer) {
    DAB_ENTER(ctx);
    if (inner == 0 || len == 0 || outer == 0) return DAB_OK;
    DAB_REQUIRE(ctx, in && out, DAB_ERR_ARG, "dab_sort_slices: null pointer");
    if (len > DAB_SORT_SLICES_SMEM_LEN) {
        switch (dtype) {
            case DAB_F32: case DAB_F64: case DAB_I32: case DAB_I64: return sort_slices_k11(ctx, dtype, in, out, inner, len, outer);
            default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_sort_slices: dtype %d", dtype);
        }
    }
    switch (dtype) {
        case DAB_F32: return sort_slices_smem<float>(ctx, in, out, inner, len, outer);
        case DAB_F64: return sort_slices_smem<double>(ctx, in, out, inner, len, outer);
        case DAB_I32: return sort_slices_smem<int32_t>(ctx, in, out, inner, len, outer);
        case DAB_I64: return sort_slices_smem<int64_t>(ctx, in, out, inner, len, outer);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_sort_slices: dtype %d", dtype);
    }
}

int32_t dab_svdvals_batched(dab_ctx* ctx, int32_t dtype, const void* A, size_t m, size_t n, size_t batch, void* S, int32_t* status) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64, DAB_ERR_UNSUPPORTED, "dab_svdvals_batched: dtype %d (served: Float32 Float64)", dtype);
    const size_t k = m < n ? m : n;
    DAB_REQUIRE(ctx, k <= DAB_SVDVALS_MAX_K && m * n <= DAB_SVDVALS_MAX_ELEMS, DAB_ERR_UNSUPPORTED,
                "dab_svdvals_batched: serves min(m,n) <= %d and m*n <= %d, got %zux%zu", DAB_SVDVALS_MAX_K, DAB_SVDVALS_MAX_ELEMS, m, n);
    DAB_REQUIRE(ctx, status != nullptr, DAB_ERR_ARG, "dab_svdvals_batched: null status");
    DAB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t), ctx->stream));
    if (batch == 0 || k == 0) return DAB_OK;
    DAB_REQUIRE(ctx, A && S, DAB_ERR_ARG, "dab_svdvals_batched: null pointer");
    return dtype == DAB_F32 ? svdvals_t<float>(ctx, A, m, n, batch, S, status) : svdvals_t<double>(ctx, A, m, n, batch, S, status);
}

}  // extern "C"
