// dab_lu_batched.cu -- K27: the linear-algebra slice functions of ppeval / mapslices built on an LU factorization:
//   dab_ldiv_batched  X_b = A_b \ B_b for a batch of small square slices (f = \, Julia's dispatch: diagonal, triangular or LU)
//   dab_det_batched   D_b = det(A_b)                                      (f = det: triangular product or LU)
// The per-element code (structure tests, pivot choice, elimination, substitutions, det accumulation, status word) is in dab_lu_core.cuh.
// Every slice is factored in fp64 whatever T is, and rounded to T once.
//
// Two kernels, chosen by n:
//   lu_group_kernel  n <= 32: a group of NB = 4 / 8 / 16 / 32 lanes per matrix (32 / NB matrices per warp), lane r holding row r of its
//                    matrix in registers (NB doubles, indexed only by unrolled constants; <= 128 registers, 4 CTAs per SM).  Rows are never moved: every lane keeps the
//                    position `pos` its row has in P*A, the pivot search is a shuffle reduction over the group, and the pivot row reaches
//                    the other lanes through a 32-double shared-memory buffer per warp.  RHS columns stream through the substitutions
//                    one at a time, a ballot naming the lane at each position.
//   lu_block_kernel  32 < n <= 64: one CTA of 256 threads per matrix (grid-stride over the batch), the matrix in shared memory as fp64,
//                    rows swapped in place; the substitutions run 4 RHS columns at a time.
// Every control-flow decision that guards a shuffle, ballot or barrier is uniform over the warp (group kernel) or the CTA (block kernel).
#include "dab_common.cuh"
#include "dab_lu_core.cuh"

namespace {

constexpr unsigned int LU_FULL = 0xffffffffu;
constexpr int LU_THREADS = 128;

template <int NB>
__device__ __forceinline__ unsigned int lu_group_mask(int sub) {
    return NB == 32 ? LU_FULL : (((1u << NB) - 1u) << (sub * NB));
}

// ---- n <= 32: one group of NB lanes per matrix -------------------------------------------------------------------------------------------
template <typename T, int NB, bool DET>
__global__ void __launch_bounds__(LU_THREADS, 4) lu_group_kernel(const T* __restrict__ A, size_t sa, const T* __restrict__ B, size_t sb,
                                                                 T* __restrict__ X, int n, int nrhs, size_t batch,
                                                                 unsigned long long* __restrict__ status) {
    constexpr int G = 32 / NB;                                     // matrices per warp
    __shared__ __align__(16) double buf[LU_THREADS / 32][32];     // per warp: NB doubles per group
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, sub = lane / NB, r = lane - sub * NB, base = sub * NB;
    double* gbuf = &buf[wib][base];
    const unsigned int gmask = lu_group_mask<NB>(sub);
    const size_t nwarps = (size_t)gridDim.x * (LU_THREADS / 32);
    for (size_t b0 = ((size_t)blockIdx.x * (LU_THREADS / 32) + wib) * G; b0 < batch; b0 += nwarps * G) {
        const size_t b = b0 + sub;
        const bool here = b < batch, live = here && r < n;
        const T* a_in = A + (here ? b : 0) * sa;
        double a[NB];
        bool nl = false, nu = false, nf = false;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            a[j] = (live && j < n) ? (double)a_in[r + (size_t)n * j] : 0.0;
            nl |= lu_breaks_lower(r, j, a[j]);
            nu |= lu_breaks_upper(r, j, a[j]);
            nf |= !isfinite(a[j]);
        }
        const bool not_lower = (__ballot_sync(LU_FULL, nl) & gmask) != 0u;
        const bool not_upper = (__ballot_sync(LU_FULL, nu) & gmask) != 0u;
        const bool nonfinite = (__ballot_sync(LU_FULL, nf) & gmask) != 0u;
        const int path = DET ? (lu_det_triangular(not_lower, not_upper) ? LU_PATH_DIAG : LU_PATH_LU) : lu_ldiv_path(not_lower, not_upper);
        const bool do_lu = path == LU_PATH_LU;
        int pos = r, swaps = 0;
        if (__any_sync(LU_FULL, do_lu)) {
#pragma unroll
            for (int k = 0; k < NB; ++k) {
                if (k >= n) break;
                // pivot: the best (key, position) of the candidates pos >= k; ties can only be equal keys at distinct positions
                double key = (live && pos >= k) ? lu_pivot_key(a[k], pos, k) : -2.0;
                int kpl = (pos << 8) | r;
#pragma unroll
                for (int o = NB / 2; o > 0; o >>= 1) {
                    const double ok = __shfl_xor_sync(LU_FULL, key, o);
                    const int op = __shfl_xor_sync(LU_FULL, kpl, o);
                    if (lu_pivot_wins(ok, op >> 8, key, kpl >> 8)) {
                        key = ok;
                        kpl = op;
                    }
                }
                const int kp = kpl >> 8, kl = kpl & 0xff;
                const double piv = __shfl_sync(LU_FULL, a[k], base + kl);
                if (do_lu) {                                       // swap positions k and kp
                    swaps += kp != k;
                    if (pos == k) pos = kp;
                    if (r == kl) pos = k;
                }
                __syncwarp();                                      // the previous step's readers are done with the buffer
                if (r == kl) {
#pragma unroll
                    for (int q = (k + 1) / 2; q < NB / 2; ++q) reinterpret_cast<double2*>(gbuf)[q] = make_double2(a[2 * q], a[2 * q + 1]);
                }
                __syncwarp();
                if (do_lu && live && pos > k && piv != 0.0) {     // a zero pivot leaves the column as it is (dgetrf2 only sets info)
                    const double l = lu_multiplier(a[k], piv, 1.0 / piv, lu_use_reciprocal(piv));
                    a[k] = l;
#pragma unroll
                    for (int q = (k + 1) / 2; q < NB / 2; ++q) {
                        const double2 u = reinterpret_cast<const double2*>(gbuf)[q];
                        if (2 * q > k) a[2 * q] = lu_update(a[2 * q], l, u.x);
                        a[2 * q + 1] = lu_update(a[2 * q + 1], l, u.y);
                    }
                }
            }
        }
        // the diagonal entry of U (of A on the triangular paths) at every position, in position order
        double dself = 0.0;
#pragma unroll
        for (int j = 0; j < NB; ++j)
            if (j == pos) dself = a[j];
        __syncwarp();
        if (live) gbuf[pos] = dself;
        __syncwarp();
        if (DET) {
            if (r == 0 && here) {
                double p = 1.0;
                int info = 0;
                for (int j = 0; j < n; ++j) {
                    const double d = gbuf[j];
                    p = lu_det_step(p, d);
                    if (d == 0.0 && info == 0) info = j + 1;
                }
                X[b] = (T)(do_lu ? lu_det_finish(p, swaps, info) : p);
            }
            __syncwarp();                                          // the buffer is rewritten by the next matrix
            continue;
        }
        if (r == 0 && here) {
            int info = 0;
            for (int j = 0; j < n && info == 0; ++j)
                if (gbuf[j] == 0.0) info = j + 1;
            const bool bad_nf = do_lu && nonfinite;                // getrf!'s chkfinite runs on the LU path only
            if (bad_nf || (info != 0 && (path != LU_PATH_DIAG || nrhs > 0))) atomicMin(status, lu_status_key(b, info, bad_nf));
        }
        __syncwarp();
        const bool fwd = path == LU_PATH_LU || path == LU_PATH_LOWER, unit = do_lu;
        const bool bwd = path == LU_PATH_LU || path == LU_PATH_UPPER, diag = path == LU_PATH_DIAG;
        const T* b_in = B + (here ? b : 0) * sb;
        T* x_out = X + (here ? b : 0) * (size_t)n * (size_t)nrhs;
        const bool any_fwd = __any_sync(LU_FULL, fwd), any_bwd = __any_sync(LU_FULL, bwd);
        for (int c = 0; c < nrhs; ++c) {
            double y = live ? (double)b_in[r + (size_t)n * c] : 0.0;   // lane r holds b_r, which P*b puts at position pos
            if (diag) y = lu_divide(y, dself);
            if (any_fwd) {
#pragma unroll
                for (int s = 0; s < NB; ++s) {
                    if (s >= n) break;
                    if (fwd && !unit && pos == s) y = lu_divide(y, dself);
                    const unsigned int who = __ballot_sync(LU_FULL, pos == s) & gmask;
                    const double ys = __shfl_sync(LU_FULL, y, __ffs(who) - 1);
                    if (fwd && pos > s) y = lu_subst(y, a[s], ys);
                }
            }
            if (any_bwd) {
#pragma unroll
                for (int s = NB - 1; s >= 0; --s) {
                    if (s >= n) continue;
                    if (bwd && pos == s) y = lu_divide(y, dself);
                    const unsigned int who = __ballot_sync(LU_FULL, pos == s) & gmask;
                    const double ys = __shfl_sync(LU_FULL, y, __ffs(who) - 1);
                    if (bwd && pos < s) y = lu_subst(y, a[s], ys);
                }
            }
            if (live) x_out[pos + (size_t)n * c] = (T)y;
        }
    }
}

// ---- 32 < n <= 64: one CTA per matrix --------------------------------------------------------------------------------------------------
constexpr int LUB_THREADS = 256, LUB_LD = DAB_LU_MAX_N + 1, LUB_CW = LUB_THREADS / DAB_LU_MAX_N;

template <typename T, bool DET>
__global__ void __launch_bounds__(LUB_THREADS) lu_block_kernel(const T* __restrict__ A, size_t sa, const T* __restrict__ B, size_t sb,
                                                               T* __restrict__ X, int n, int nrhs, size_t batch,
                                                               unsigned long long* __restrict__ status) {
    __shared__ double M[DAB_LU_MAX_N * LUB_LD];                   // column-major, leading dimension 65
    __shared__ double Y[LUB_CW * DAB_LU_MAX_N];                   // x_s of the column being solved, per RHS column of the chunk
    __shared__ int perm[DAB_LU_MAX_N];                            // row of A at each position of P*A
    __shared__ int s_flags, s_p;
    __shared__ double s_piv;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, ri = t & (DAB_LU_MAX_N - 1), cj = t / DAB_LU_MAX_N;
    for (size_t b = blockIdx.x; b < batch; b += gridDim.x) {
        const T* a_in = A + b * sa;
        if (t == 0) s_flags = 0;
        __syncthreads();
        int fl = 0;
        for (int e = t; e < n * n; e += LUB_THREADS) {
            const int i = e % n, j = e / n;
            const double v = (double)a_in[e];
            M[i + LUB_LD * j] = v;
            fl |= (lu_breaks_lower(i, j, v) ? 1 : 0) | (lu_breaks_upper(i, j, v) ? 2 : 0) | (isfinite(v) ? 0 : 4);
        }
        if (t < n) perm[t] = t;
        fl = __reduce_or_sync(LU_FULL, fl);
        if (lane == 0 && fl) atomicOr(&s_flags, fl);
        __syncthreads();
        const int flags = s_flags;
        const bool not_lower = flags & 1, not_upper = flags & 2, nonfinite = flags & 4;
        const int path = DET ? (lu_det_triangular(not_lower, not_upper) ? LU_PATH_DIAG : LU_PATH_LU) : lu_ldiv_path(not_lower, not_upper);
        const bool do_lu = path == LU_PATH_LU;
        int swaps = 0, info = 0;
        if (do_lu) {
            for (int k = 0; k < n; ++k) {
                if (warp == 0) {
                    double key = -2.0;
                    int kp = DAB_LU_MAX_N;
                    for (int i = k + lane; i < n; i += 32) {
                        const double ki = lu_pivot_key(M[i + LUB_LD * k], i, k);
                        if (lu_pivot_wins(ki, i, key, kp)) {
                            key = ki;
                            kp = i;
                        }
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const double ok = __shfl_xor_sync(LU_FULL, key, o);
                        const int op = __shfl_xor_sync(LU_FULL, kp, o);
                        if (lu_pivot_wins(ok, op, key, kp)) {
                            key = ok;
                            kp = op;
                        }
                    }
                    if (lane == 0) {
                        s_p = kp;
                        s_piv = M[kp + LUB_LD * k];
                    }
                }
                __syncthreads();
                const int p = s_p;
                const double piv = s_piv;
                if (p != k) {
                    ++swaps;
                    for (int j = t; j < n; j += LUB_THREADS) {
                        const double u = M[k + LUB_LD * j];
                        M[k + LUB_LD * j] = M[p + LUB_LD * j];
                        M[p + LUB_LD * j] = u;
                    }
                    if (t == 0) {
                        const int q = perm[k];
                        perm[k] = perm[p];
                        perm[p] = q;
                    }
                }
                if (piv == 0.0 && info == 0) info = k + 1;
                __syncthreads();
                if (piv != 0.0) {
                    const bool recip = lu_use_reciprocal(piv);
                    const double rpiv = 1.0 / piv;
                    for (int i = k + 1 + t; i < n; i += LUB_THREADS) M[i + LUB_LD * k] = lu_multiplier(M[i + LUB_LD * k], piv, rpiv, recip);
                    __syncthreads();
                    const int i = k + 1 + ri;
                    if (i < n) {
                        const double l = M[i + LUB_LD * k];
                        for (int j = k + 1 + cj; j < n; j += LUB_CW) M[i + LUB_LD * j] = lu_update(M[i + LUB_LD * j], l, M[k + LUB_LD * j]);
                    }
                }
                __syncthreads();
            }
        }
        if (DET) {
            if (t == 0) {
                double p = 1.0;
                for (int j = 0; j < n; ++j) p = lu_det_step(p, M[j + LUB_LD * j]);
                X[b] = (T)(do_lu ? lu_det_finish(p, swaps, info) : p);
            }
            __syncthreads();
            continue;
        }
        if (t == 0) {
            int first = 0;
            for (int j = 0; j < n && first == 0; ++j)
                if (M[j + LUB_LD * j] == 0.0) first = j + 1;
            const bool bad_nf = do_lu && nonfinite;
            if (bad_nf || (first != 0 && (path != LU_PATH_DIAG || nrhs > 0))) atomicMin(status, lu_status_key(b, first, bad_nf));
        }
        const bool fwd = path == LU_PATH_LU || path == LU_PATH_LOWER, unit = do_lu;
        const bool bwd = path == LU_PATH_LU || path == LU_PATH_UPPER;
        const T* b_in = B + b * sb;
        T* x_out = X + b * (size_t)n * (size_t)nrhs;
        const int i = ri;
        for (int c0 = 0; c0 < nrhs; c0 += LUB_CW) {
            const int c = c0 + cj;
            const bool act = i < n && c < nrhs;
            double* y = Y + cj * DAB_LU_MAX_N;
            double yi = act ? (double)b_in[perm[i] + (size_t)n * c] : 0.0;
            if (path == LU_PATH_DIAG && act) yi = lu_divide(yi, M[i + LUB_LD * i]);
            if (fwd) {
                for (int s = 0; s < n; ++s) {
                    if (i == s) {
                        if (!unit && act) yi = lu_divide(yi, M[s + LUB_LD * s]);
                        y[s] = yi;
                    }
                    __syncthreads();
                    if (act && i > s) yi = lu_subst(yi, M[i + LUB_LD * s], y[s]);
                }
            }
            if (bwd) {
                for (int s = n - 1; s >= 0; --s) {
                    if (i == s) {
                        if (act) yi = lu_divide(yi, M[s + LUB_LD * s]);
                        y[s] = yi;
                    }
                    __syncthreads();
                    if (act && i < s) yi = lu_subst(yi, M[i + LUB_LD * s], y[s]);
                }
            }
            if (act) x_out[i + (size_t)n * c] = (T)yi;
            __syncthreads();                                       // Y is rewritten by the next chunk of columns
        }
        __syncthreads();                                          // M is rewritten by the next matrix
    }
}

template <typename T, bool DET>
int32_t lu_batched_t(dab_ctx* ctx, size_t n, size_t nrhs, const void* A, size_t sa, const void* B, size_t sb, void* X, size_t batch,
                     unsigned long long* status) {
    const T* a = (const T*)A;
    const T* bb = (const T*)B;
    T* x = (T*)X;
    if (n > 32) {
        auto kern = lu_block_kernel<T, DET>;
        kern<<<dab_persistent_grid(ctx, kern, LUB_THREADS, batch), LUB_THREADS, 0, ctx->stream>>>(a, sa, bb, sb, x, (int)n, (int)nrhs, batch,
                                                                                                 status);
    } else {
        const int nb = n <= 4 ? 4 : n <= 8 ? 8 : n <= 16 ? 16 : 32;
        const size_t per_block = (size_t)(LU_THREADS / 32) * (size_t)(32 / nb);
        const size_t blocks = (batch + per_block - 1) / per_block;
        auto kern = nb == 4 ? lu_group_kernel<T, 4, DET> : nb == 8 ? lu_group_kernel<T, 8, DET> : nb == 16 ? lu_group_kernel<T, 16, DET>
                                                                                                         : lu_group_kernel<T, 32, DET>;
        kern<<<dab_persistent_grid(ctx, kern, LU_THREADS, blocks), LU_THREADS, 0, ctx->stream>>>(a, sa, bb, sb, x, (int)n, (int)nrhs, batch,
                                                                                                status);
    }
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_ldiv_batched(dab_ctx* ctx, int32_t dtype, size_t n, size_t nrhs, const void* A, size_t strideA, const void* B, size_t strideB,
                         void* X, size_t batch, void* status) {
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64, DAB_ERR_UNSUPPORTED, "dab_ldiv_batched: dtype %d (served: Float32 Float64)", dtype);
    DAB_REQUIRE(ctx, n <= DAB_LU_MAX_N, DAB_ERR_UNSUPPORTED, "dab_ldiv_batched: serves n <= %d, got %zu x %zu", DAB_LU_MAX_N, n, n);
    DAB_REQUIRE(ctx, nrhs < (1ull << 31), DAB_ERR_UNSUPPORTED, "dab_ldiv_batched: nrhs must be below 2^31, got %zu", nrhs);
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, status != nullptr, DAB_ERR_ARG, "dab_ldiv_batched: null status");
    DAB_CUDA(ctx, cudaMemsetAsync(status, 0xFF, sizeof(unsigned long long), ctx->stream));
    if (batch == 0 || n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, A != nullptr && (nrhs == 0 || (B != nullptr && X != nullptr)), DAB_ERR_ARG, "dab_ldiv_batched: null pointer");
    unsigned long long* st = (unsigned long long*)status;
    return dtype == DAB_F32 ? lu_batched_t<float, false>(ctx, n, nrhs, A, strideA, B, strideB, X, batch, st)
                            : lu_batched_t<double, false>(ctx, n, nrhs, A, strideA, B, strideB, X, batch, st);
}

int32_t dab_det_batched(dab_ctx* ctx, int32_t dtype, size_t n, const void* A, size_t strideA, void* D, size_t batch) {
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64, DAB_ERR_UNSUPPORTED, "dab_det_batched: dtype %d (served: Float32 Float64)", dtype);
    DAB_REQUIRE(ctx, n <= DAB_LU_MAX_N, DAB_ERR_UNSUPPORTED, "dab_det_batched: serves n <= %d, got %zu x %zu", DAB_LU_MAX_N, n, n);
    DAB_ENTER(ctx);
    if (batch == 0) return DAB_OK;
    DAB_REQUIRE(ctx, D != nullptr && (n == 0 || A != nullptr), DAB_ERR_ARG, "dab_det_batched: null pointer");
    return dtype == DAB_F32 ? lu_batched_t<float, true>(ctx, n, 0, A, strideA, nullptr, 0, D, batch, nullptr)
                            : lu_batched_t<double, true>(ctx, n, 0, A, strideA, nullptr, 0, D, batch, nullptr);
}

}  // extern "C"
