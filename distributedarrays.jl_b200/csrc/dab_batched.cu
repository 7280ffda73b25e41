// dab_batched.cu -- the two slice functions of ppeval(f, D...; dim) (reference src/mapreduce.jl:210-323) that need kernels of their own:
//   dab_matmul_batched       C_b = A_b * B_b for a batch of dense column-major slices (f = *, a matrix times a vector or a matrix)
//   dab_eigvals_sym_batched  eigenvalues of a batch of small real symmetric matrices, ascending (f = eigvals)
// The per-element code of the eigenvalue kernel (round-robin pairing, rotation, convergence test, ranking) is in dab_slices_core.cuh.
//
// Batched product, three kernels chosen by slice size (every one of them k-ordered per output element):
//   bmm_small_kernel  (m*k + k*n) elements of A_b and B_b fit BMM_SMALL_BYTES (and n > 1 or m < 32): a CTA stages G whole slices in
//                     shared memory with coalesced loads and runs a thread per output element (a 10x10 Float64 matrix x vector packs 27 slices);
//   bmv_kernel        n == 1 otherwise: a thread per output row reading A_b straight from global memory, consecutive threads on
//                     consecutive rows (one coalesced read of A, the stream of K9);
//   bmm_tile_kernel   otherwise: a 64 x 64 output tile per (slice, tile) work item, k-loop through shared memory in steps of 16, 4 x 4
//                     outputs per thread.
// Numerics as K9 / K12's SIMT path: Float32 products are exact in fp64 and accumulate there, rounded once at the end; Float64 uses one
// DFMA per k, in k order; Int32 / Int64 wrap (unsigned arithmetic of the same width).
#include <type_traits>

#include "dab_common.cuh"
#include "dab_slices_core.cuh"

namespace {

template <typename T> struct BmmAcc { using type = double; };
template <> struct BmmAcc<int32_t> { using type = uint32_t; };
template <> struct BmmAcc<int64_t> { using type = unsigned long long; };

template <typename T>
__device__ __forceinline__ typename BmmAcc<T>::type bmm_madd(T a, T b, typename BmmAcc<T>::type acc) {
    using Acc = typename BmmAcc<T>::type;
    if constexpr (std::is_floating_point<T>::value) return __fma_rn((double)a, (double)b, acc);
    else return acc + (Acc)a * (Acc)b;
}

// ---- whole slices in shared memory ----------------------------------------------------------------------------------------------------
constexpr int BMM_THREADS = 256;
constexpr size_t BMM_SMALL_BYTES = 24576;    // A_b and B_b of one slice at most; G slices per CTA fill up to this much
constexpr size_t BMM_SMALL_OUTS = 2048;      // outputs per CTA at most (8 per thread)

template <typename T>
__global__ void __launch_bounds__(BMM_THREADS) bmm_small_kernel(const T* __restrict__ A, size_t sa, const T* __restrict__ B, size_t sb,
                                                                T* __restrict__ Cm, int m, int n, int k, size_t batch, int G) {
    extern __shared__ __align__(16) unsigned char bmm_smem[];
    T* As = reinterpret_cast<T*>(bmm_smem);
    const size_t mk = (size_t)m * k, kn = (size_t)k * n, mn = (size_t)m * n;
    const size_t na = sa ? (size_t)G * mk : mk;                    // a broadcast operand (stride 0) is staged once
    T* Bs = As + na;
    const size_t ngroups = (batch + G - 1) / G;
    for (size_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
        const size_t b0 = g * G;
        const int nb = (int)(batch - b0 < (size_t)G ? batch - b0 : (size_t)G);
        // slice b's A is mk contiguous elements at b * sa: with sa == mk the group is one contiguous run
        const size_t la = sa ? (size_t)nb * mk : mk, lb = sb ? (size_t)nb * kn : kn;
        for (size_t t = threadIdx.x; t < la; t += BMM_THREADS) {
            const size_t s = t / mk;
            As[t] = A[(b0 + s) * sa + (t - s * mk)];
        }
        for (size_t t = threadIdx.x; t < lb; t += BMM_THREADS) {
            const size_t s = t / kn;
            Bs[t] = B[(b0 + s) * sb + (t - s * kn)];
        }
        __syncthreads();
        const size_t nout = (size_t)nb * mn;
        for (size_t o = threadIdx.x; o < nout; o += BMM_THREADS) {
            const size_t s = o / mn, r = o - s * mn;
            const int j = (int)(r / m), i = (int)(r - (size_t)j * m);
            const T* a = As + (sa ? s * mk : 0) + i;
            const T* bcol = Bs + (sb ? s * kn : 0) + (size_t)j * k;
            typename BmmAcc<T>::type acc = 0;
            for (int kk = 0; kk < k; ++kk) acc = bmm_madd<T>(a[(size_t)kk * m], bcol[kk], acc);
            Cm[b0 * mn + o] = (T)acc;
        }
        __syncthreads();                                          // shared memory is reused by the next group
    }
}

// ---- matrix x vector, slices too large for the staged kernel ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(BMM_THREADS) bmv_kernel(const T* __restrict__ A, size_t sa, const T* __restrict__ x, size_t sx,
                                                          T* __restrict__ y, size_t m, size_t k, size_t batch) {
    const size_t rows = m * batch;
    for (size_t o = (size_t)blockIdx.x * BMM_THREADS + threadIdx.x; o < rows; o += (size_t)gridDim.x * BMM_THREADS) {
        const size_t b = o / m, i = o - b * m;
        const T* a = A + b * sa + i;
        const T* xb = x + b * sx;
        typename BmmAcc<T>::type acc = 0;
#pragma unroll 4
        for (size_t kk = 0; kk < k; ++kk) acc = bmm_madd<T>(a[kk * m], __ldg(xb + kk), acc);
        y[o] = (T)acc;
    }
}

// ---- 64 x 64 output tiles ------------------------------------------------------------------------------------------------------------
constexpr int BT_M = 64, BT_N = 64, BT_K = 16;

template <typename T>
__global__ void __launch_bounds__(BMM_THREADS) bmm_tile_kernel(const T* __restrict__ A, size_t sa, const T* __restrict__ B, size_t sb,
                                                               T* __restrict__ Cm, int m, int n, int k, size_t batch) {
    using Acc = typename BmmAcc<T>::type;
    __shared__ T As[BT_K][BT_M + 1];
    __shared__ T Bs[BT_K][BT_N + 1];
    const int tm = (m + BT_M - 1) / BT_M, tn = (n + BT_N - 1) / BT_N;
    const size_t tiles = (size_t)tm * tn, items = tiles * batch;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    for (size_t w = blockIdx.x; w < items; w += gridDim.x) {
        const size_t b = w / tiles;
        const int t = (int)(w - b * tiles), m0 = (t % tm) * BT_M, n0 = (t / tm) * BT_N;
        const T* a = A + b * sa;
        const T* bb = B + b * sb;
        Acc acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = 0;
        for (int k0 = 0; k0 < k; k0 += BT_K) {
#pragma unroll
            for (int q = 0; q < (BT_M * BT_K) / BMM_THREADS; ++q) {
                const int idx = tid + q * BMM_THREADS, i = idx % BT_M, kk = idx / BT_M;
                const int gi = m0 + i, gk = k0 + kk;
                As[kk][i] = (gi < m && gk < k) ? a[gi + (size_t)gk * m] : T(0);
            }
#pragma unroll
            for (int q = 0; q < (BT_N * BT_K) / BMM_THREADS; ++q) {
                const int idx = tid + q * BMM_THREADS, kk = idx % BT_K, j = idx / BT_K;
                const int gj = n0 + j, gk = k0 + kk;
                Bs[kk][j] = (gj < n && gk < k) ? bb[gk + (size_t)gj * k] : T(0);
            }
            __syncthreads();
            const int kend = k - k0 < BT_K ? k - k0 : BT_K;       // the k that exist, in order
            for (int kk = 0; kk < kend; ++kk) {
                T av[4], bv[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) av[r] = As[kk][tx + 16 * r];
#pragma unroll
                for (int c = 0; c < 4; ++c) bv[c] = Bs[kk][ty + 16 * c];
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[r][c] = bmm_madd<T>(av[r], bv[c], acc[r][c]);
            }
            __syncthreads();
        }
        T* cb = Cm + b * (size_t)m * n;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int gj = n0 + ty + 16 * c;
            if (gj >= n) continue;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int gi = m0 + tx + 16 * r;
                if (gi < m) cb[gi + (size_t)gj * m] = (T)acc[r][c];
            }
        }
    }
}

template <typename T>
int32_t matmul_batched_t(dab_ctx* ctx, size_t m, size_t n, size_t k, const T* A, size_t sa, const T* B, size_t sb, T* Cm, size_t batch) {
    const size_t slice_bytes = (m * k + k * n) * sizeof(T);
    if (slice_bytes <= BMM_SMALL_BYTES && (n > 1 || m < 32)) {   // a matrix x vector of >= 32 rows streams better straight from HBM
        const size_t per = slice_bytes ? BMM_SMALL_BYTES / slice_bytes : batch;
        size_t G = per < BMM_SMALL_OUTS / (m * n) ? per : BMM_SMALL_OUTS / (m * n);
        if (G < 1) G = 1;
        if (G > batch) G = batch;
        const size_t smem = ((sa ? G : 1) * m * k + (sb ? G : 1) * k * n) * sizeof(T);
        auto kern = bmm_small_kernel<T>;
        const int grid = dab_grid_for(ctx, (batch + G - 1) / G, 8);
        kern<<<grid, BMM_THREADS, smem, ctx->stream>>>(A, sa, B, sb, Cm, (int)m, (int)n, (int)k, batch, (int)G);
    } else if (n == 1) {
        const int grid = dab_grid_for(ctx, (m * batch + BMM_THREADS - 1) / BMM_THREADS, 8);
        bmv_kernel<T><<<grid, BMM_THREADS, 0, ctx->stream>>>(A, sa, B, sb, Cm, m, k, batch);
    } else {
        const size_t items = ((m + BT_M - 1) / BT_M) * ((n + BT_N - 1) / BT_N) * batch;
        const int grid = dab_grid_for(ctx, items, 4);
        bmm_tile_kernel<T><<<grid, BMM_THREADS, 0, ctx->stream>>>(A, sa, B, sb, Cm, (int)m, (int)n, (int)k, batch);
    }
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// ---- batched symmetric eigenvalues --------------------------------------------------------------------------------------------------
// One CTA per matrix (grid-stride over the batch), the matrix in dynamic shared memory as fp64 (n * n * 8 bytes, 32 KiB at n = 64).
// Loading flags a NaN / Inf (status bit 1) and, for a finite matrix, an entry with A[i,j] != A[j,i] (bit 2); such a matrix yields NaNs.
// The matrix is scaled by 2^-e, max |a| * 2^-e in [0.5, 1), before the sweeps (slices_scale_exp) and the eigenvalues by 2^e after them.
// A round: threads k < np/2 compute the rotation of pair k from the current pivots; all rows are rotated; all columns are rotated; the
// rotated a_pq, a_qp are set to 0 (what the rotation makes them, less its rounding).  The diagonal is ranked ascending at the end.
constexpr int EIG_MAX_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(EIG_MAX_THREADS) eigvals_sym_kernel(const T* __restrict__ A, int n, size_t batch, T* __restrict__ W,
                                                                     int32_t* __restrict__ status) {
    extern __shared__ __align__(16) double eig_smem[];
    double* M = eig_smem;                                         // n * n, column-major
    double* cs = M + n * n;                                       // c of pair k, 32
    double* sn = cs + 32;                                         // s of pair k (0: no rotation), 32
    double* d = sn + 32;                                          // the diagonal, 64
    __shared__ double s_wmax[EIG_MAX_THREADS / 32];
    __shared__ int s_flags, s_rot;
    const int np = n + (n & 1), npairs = np / 2, nn = n * n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (size_t b = blockIdx.x; b < batch; b += gridDim.x) {
        const T* a = A + b * (size_t)nn;
        if (threadIdx.x == 0) s_flags = 0;
        __syncthreads();
        int bad = 0;
        double amax = 0.0;
        for (int t = threadIdx.x; t < nn; t += blockDim.x) {
            const double v = (double)a[t];
            if (!isfinite(v)) bad = 1;
            amax = fmax(amax, fabs(v));
            M[t] = v;
        }
        if (bad) atomicOr(&s_flags, 1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0) s_wmax[warp] = amax;
        __syncthreads();
        if (s_flags == 0) {
            int asym = 0;
            for (int t = threadIdx.x; t < nn; t += blockDim.x) {
                const int i = t % n, j = t / n;
                if (i < j && M[t] != M[j + n * i]) asym = 1;      // == semantics: -0.0 equals 0.0
            }
            if (asym) atomicOr(&s_flags, 2);
        }
        __syncthreads();
        const int flags = s_flags;
        if (flags) {
            for (int t = threadIdx.x; t < n; t += blockDim.x) W[b * n + t] = (T)NAN;
            if (threadIdx.x == 0) atomicOr(status, flags);
            __syncthreads();                                      // s_flags is reset for the next matrix only after everybody read it
            continue;
        }
        amax = 0.0;
        for (int w = 0; w < nwarps; ++w) amax = fmax(amax, s_wmax[w]);
        const int e = slices_scale_exp(amax);
        for (int t = threadIdx.x; t < nn; t += blockDim.x) M[t] = ldexp(M[t], -e);
        __syncthreads();
        for (int sweep = 0; sweep < DAB_EIG_MAX_SWEEPS; ++sweep) {
            if (threadIdx.x == 0) s_rot = 0;
            __syncthreads();
            for (int r = 0; r < np - 1; ++r) {
                if (threadIdx.x < npairs) {
                    int p, q;
                    slices_rr_pair(np, r, threadIdx.x, &p, &q);
                    double c = 1.0, s = 0.0;
                    if (p < n && q < n && slices_sym_rotation(M[p + n * p], M[q + n * q], M[p + n * q], &c, &s)) s_rot = 1;
                    cs[threadIdx.x] = c;
                    sn[threadIdx.x] = s;
                }
                __syncthreads();
                for (int w = threadIdx.x; w < npairs * n; w += blockDim.x) {          // rows p, q of J^T A
                    const int k = w / n, j = w - k * n;
                    const double s = sn[k];
                    if (s == 0.0) continue;
                    int p, q;
                    slices_rr_pair(np, r, k, &p, &q);
                    slices_jacobi_apply(&M[p + n * j], &M[q + n * j], cs[k], s);
                }
                __syncthreads();
                for (int w = threadIdx.x; w < npairs * n; w += blockDim.x) {          // columns p, q of (J^T A) J
                    const int k = w / n, i = w - k * n;
                    const double s = sn[k];
                    if (s == 0.0) continue;
                    int p, q;
                    slices_rr_pair(np, r, k, &p, &q);
                    slices_jacobi_apply(&M[i + n * p], &M[i + n * q], cs[k], s);
                }
                __syncthreads();
                // a pair meets once per sweep, so the next round's pivots never include these two entries: no barrier is needed before it
                if (threadIdx.x < npairs && sn[threadIdx.x] != 0.0) {
                    int p, q;
                    slices_rr_pair(np, r, threadIdx.x, &p, &q);
                    M[p + n * q] = 0.0;
                    M[q + n * p] = 0.0;
                }
            }
            __syncthreads();
            const int rot = s_rot;
            __syncthreads();                                      // everybody has read s_rot before it is cleared again
            if (!rot) break;
        }
        for (int t = threadIdx.x; t < n; t += blockDim.x) d[t] = M[t + n * t];
        __syncthreads();
        for (int t = threadIdx.x; t < n; t += blockDim.x) W[b * n + slices_rank_asc(d, n, t)] = (T)ldexp(d[t], e);
        __syncthreads();
    }
}

template <typename T>
int32_t eigvals_sym_t(dab_ctx* ctx, const void* A, size_t n, size_t batch, void* W, int32_t* status) {
    const int np = (int)(n + (n & 1));
    int threads = ((np / 2) * (int)n + 31) / 32 * 32;
    if (threads < 32) threads = 32;
    if (threads > EIG_MAX_THREADS) threads = EIG_MAX_THREADS;
    const size_t smem = (n * n + 128) * sizeof(double);
    const int grid = dab_grid_for(ctx, batch, 2048 / threads < 32 ? 2048 / threads : 32);
    eigvals_sym_kernel<T><<<grid, threads, smem, ctx->stream>>>((const T*)A, (int)n, batch, (T*)W, status);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_matmul_batched(dab_ctx* ctx, int32_t dtype, size_t m, size_t n, size_t k, const void* A, size_t strideA, const void* B,
                           size_t strideB, void* C, size_t batch) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64 || dtype == DAB_I32 || dtype == DAB_I64, DAB_ERR_UNSUPPORTED,
                "dab_matmul_batched: dtype %d (served: Float32 Float64 Int32 Int64)", dtype);
    DAB_REQUIRE(ctx, m < (1ull << 31) && n < (1ull << 31) && k < (1ull << 31), DAB_ERR_UNSUPPORTED,
                "dab_matmul_batched: slice dimensions must be below 2^31, got %zu x %zu x %zu", m, n, k);
    if (batch == 0 || m == 0 || n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, C != nullptr && (k == 0 || (A != nullptr && B != nullptr)), DAB_ERR_ARG, "dab_matmul_batched: null pointer");
    switch (dtype) {
        case DAB_F32: return matmul_batched_t<float>(ctx, m, n, k, (const float*)A, strideA, (const float*)B, strideB, (float*)C, batch);
        case DAB_F64: return matmul_batched_t<double>(ctx, m, n, k, (const double*)A, strideA, (const double*)B, strideB, (double*)C, batch);
        case DAB_I32: return matmul_batched_t<int32_t>(ctx, m, n, k, (const int32_t*)A, strideA, (const int32_t*)B, strideB, (int32_t*)C, batch);
        default: return matmul_batched_t<int64_t>(ctx, m, n, k, (const int64_t*)A, strideA, (const int64_t*)B, strideB, (int64_t*)C, batch);
    }
}

int32_t dab_eigvals_sym_batched(dab_ctx* ctx, int32_t dtype, const void* A, size_t n, size_t batch, void* W, int32_t* status) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64, DAB_ERR_UNSUPPORTED, "dab_eigvals_sym_batched: dtype %d (served: Float32 Float64)",
                dtype);
    DAB_REQUIRE(ctx, n <= DAB_EIGVALS_SYM_MAX_N, DAB_ERR_UNSUPPORTED, "dab_eigvals_sym_batched: serves n <= %d, got %zu x %zu",
                DAB_EIGVALS_SYM_MAX_N, n, n);
    DAB_REQUIRE(ctx, status != nullptr, DAB_ERR_ARG, "dab_eigvals_sym_batched: null status");
    DAB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t), ctx->stream));
    if (batch == 0 || n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, A && W, DAB_ERR_ARG, "dab_eigvals_sym_batched: null pointer");
    return dtype == DAB_F32 ? eigvals_sym_t<float>(ctx, A, n, batch, W, status) : eigvals_sym_t<double>(ctx, A, n, batch, W, status);
}

}  // extern "C"
