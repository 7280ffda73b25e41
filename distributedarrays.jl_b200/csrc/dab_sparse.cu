// dab_sparse.cu -- K18 / K19: the tile product of mul!(y::DVector, A::DMatrix, x) when the chunks of A are SparseMatrixCSC (reference
// src/linalg.jl:95-97, 141: localpart(A)*xj and localpart(A)'*xj dispatch to SparseArrays), on one CSC chunk in HBM.
//
// K18 dab_spmv: out[r] = fold(+, v[p] * x[idx[p]] for p in ptr[r] : ptr[r+1]-1), started from zero(T), in storage order.
//   That is SparseArrays' own loop for both products of a real T: A'*x (_At_or_Ac_mul_B!) folds each column of the CSC arrays from
//   zero, and A*x (_spmatmul!) adds nzv[j]*x[col] into C[row] column after column, i.e. each row in ascending column order -- the fold
//   over that row of the row-major copy K19 makes.  Arithmetic is in T with every product and every add rounded on its own (__fmul_rn /
//   __fadd_rn, and the library is built with -fmad=false); Int32 / Int64 wrap, computed in unsigned arithmetic.
//
//   A group of G lanes (G in 1, 2, ..., 32, chosen per launch from nnz / rows) owns one row.  Each round the group loads G consecutive
//   (idx, v) pairs coalesced, gathers x through the read-only path and forms the G products in parallel; every lane then takes the G
//   products from the group in lane order (warp shuffles) and adds them to its running sum, so the sum is the sequential fold.  The next
//   round's loads are issued before the current round is folded.  The cost of the order: one row takes at least as many dependent adds
//   as it has entries.  The round count is the warp's maximum, so the shuffles stay warp-uniform.
//
// K19 dab_csc_to_csr: the row-major copy of a chunk, stable in column order.  word[k] = row[k] << 32 | k is sorted by K11 (dab_sort on
//   Int64; the row is below 2^31, so the words are non-negative and signed order is the order of (row, k)); k ascends with the column in
//   a CSC chunk, so the sorted words list rows ascending and, within a row, columns ascending.  The column of entry k is found by a
//   binary search of colptr, the value is gathered from nzval, and rowptr[r] is the number of words below r << 32.
#include <type_traits>

#include "dab_common.cuh"

namespace {

constexpr int SP_THREADS = 256;
constexpr unsigned FULL = 0xFFFFFFFFu;

template <typename T> struct SpAcc { using type = T; };
template <> struct SpAcc<int32_t> { using type = uint32_t; };   // wrap-around without signed-overflow UB
template <> struct SpAcc<int64_t> { using type = uint64_t; };

__device__ __forceinline__ float sp_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float sp_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double sp_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double sp_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ uint32_t sp_mul(uint32_t a, uint32_t b) { return a * b; }
__device__ __forceinline__ uint32_t sp_add(uint32_t a, uint32_t b) { return a + b; }
__device__ __forceinline__ uint64_t sp_mul(uint64_t a, uint64_t b) { return a * b; }
__device__ __forceinline__ uint64_t sp_add(uint64_t a, uint64_t b) { return a + b; }

// product of entry p, or zero for a lane past the end of its row (never added: the fold only takes the first `cnt` lanes)
template <typename T>
__device__ __forceinline__ typename SpAcc<T>::type sp_term(const int32_t* __restrict__ idx, const T* __restrict__ val,
                                                           const T* __restrict__ x, long long p, long long end) {
    using A = typename SpAcc<T>::type;
    if (p >= end) return A(0);
    const int32_t i = __ldcs(idx + p);
    const T v = __ldcs(val + p);
    return sp_mul((A)v, (A)__ldg(x + i));
}

template <typename T, int G>
__global__ void __launch_bounds__(SP_THREADS) spmv_kernel(size_t nrows, const long long* __restrict__ ptr, const int32_t* __restrict__ idx,
                                                          const T* __restrict__ val, const T* __restrict__ x, T* __restrict__ out) {
    using A = typename SpAcc<T>::type;
    constexpr int RPW = 32 / G;                                   // rows per warp
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const size_t warp = ((size_t)blockIdx.x * SP_THREADS + threadIdx.x) >> 5;
    const size_t nwarps = ((size_t)gridDim.x * SP_THREADS) >> 5;
    for (size_t base = warp * RPW; base < nrows; base += nwarps * RPW) {   // warp-uniform trip count
        const size_t row = base + (size_t)(lane / G);
        long long start = 0, end = 0;
        if (row < nrows) {
            start = __ldg(ptr + row);
            end = __ldg(ptr + row + 1);
        }
        const unsigned len = (unsigned)(end - start);             // < 2^32 entries per chunk
        const unsigned rounds = __reduce_max_sync(FULL, (len + (G - 1)) / G);
        A acc = A(0);
        A cur = sp_term<T>(idx, val, x, start + sub, end);
        for (unsigned r = 0; r < rounds; ++r) {
            const long long pn = start + (long long)(r + 1) * G + sub;
            const A nxt = (r + 1 < rounds) ? sp_term<T>(idx, val, x, pn, end) : A(0);
            const unsigned done = r * G;
            const unsigned cnt = len > done ? (len - done < (unsigned)G ? len - done : (unsigned)G) : 0u;
            if constexpr (G == 1) {
                if (cnt) acc = sp_add(acc, cur);
            } else {
#pragma unroll
                for (int k = 0; k < G; ++k) {
                    const A q = __shfl_sync(FULL, cur, k, G);
                    if ((unsigned)k < cnt) acc = sp_add(acc, q);
                }
            }
            cur = nxt;
        }
        if (row < nrows && sub == 0) out[row] = (T)acc;
    }
}

template <typename T, int G>
int32_t launch_spmv(dab_ctx* ctx, size_t nrows, const long long* ptr, const int32_t* idx, const void* val, const void* x, void* out) {
    constexpr int RPW = 32 / G;
    const size_t warps = (nrows + RPW - 1) / RPW;
    const size_t blocks = (warps + SP_THREADS / 32 - 1) / (SP_THREADS / 32);
    auto kern = spmv_kernel<T, G>;
    const int grid = dab_persistent_grid(ctx, kern, SP_THREADS, blocks);
    kern<<<grid, SP_THREADS, 0, ctx->stream>>>(nrows, ptr, idx, (const T*)val, (const T*)x, (T*)out);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// G: the smallest power of two >= the mean row length, 1..32
int spmv_group(size_t nrows, size_t nnz) {
    const size_t mean = nrows ? (nnz + nrows - 1) / nrows : 0;
    int g = 1;
    while (g < 32 && (size_t)g < mean) g <<= 1;
    return g;
}

template <typename T>
int32_t spmv_t(dab_ctx* ctx, size_t nrows, size_t nnz, const long long* ptr, const int32_t* idx, const void* val, const void* x, void* out) {
    switch (spmv_group(nrows, nnz)) {
        case 1: return launch_spmv<T, 1>(ctx, nrows, ptr, idx, val, x, out);
        case 2: return launch_spmv<T, 2>(ctx, nrows, ptr, idx, val, x, out);
        case 4: return launch_spmv<T, 4>(ctx, nrows, ptr, idx, val, x, out);
        case 8: return launch_spmv<T, 8>(ctx, nrows, ptr, idx, val, x, out);
        case 16: return launch_spmv<T, 16>(ctx, nrows, ptr, idx, val, x, out);
        default: return launch_spmv<T, 32>(ctx, nrows, ptr, idx, val, x, out);
    }
}

// ---- K19 ---------------------------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(SP_THREADS) csr_pack_kernel(const int32_t* __restrict__ rowval, unsigned long long* __restrict__ words, size_t nnz) {
    const size_t stride = (size_t)gridDim.x * SP_THREADS;
    for (size_t k = (size_t)blockIdx.x * SP_THREADS + threadIdx.x; k < nnz; k += stride)
        words[k] = ((unsigned long long)(uint32_t)__ldcs(rowval + k) << 32) | (unsigned long long)k;
}

// colidx[j] = the column holding storage position k = lo32(sorted[j]) (largest c with colptr[c] <= k), val[j] = nzval[k]
template <typename V>
__global__ void __launch_bounds__(SP_THREADS) csr_unpack_kernel(const unsigned long long* __restrict__ sorted, const long long* __restrict__ colptr,
                                                                size_t ncols, const V* __restrict__ nzval, int32_t* __restrict__ colidx,
                                                                V* __restrict__ val, size_t nnz) {
    const size_t stride = (size_t)gridDim.x * SP_THREADS;
    for (size_t j = (size_t)blockIdx.x * SP_THREADS + threadIdx.x; j < nnz; j += stride) {
        const long long k = (long long)(sorted[j] & 0xFFFFFFFFull);
        size_t lo = 0, hi = ncols;                                // invariant: colptr[lo] <= k < colptr[hi]
        while (hi - lo > 1) {
            const size_t mid = lo + ((hi - lo) >> 1);
            if (__ldg(colptr + mid) <= k) lo = mid;
            else hi = mid;
        }
        colidx[j] = (int32_t)lo;
        val[j] = __ldg(nzval + k);
    }
}

// rowptr[r] = number of sorted words below r << 32, r = 0..nrows
__global__ void __launch_bounds__(SP_THREADS) csr_rowptr_kernel(const unsigned long long* __restrict__ sorted, size_t nnz, long long* __restrict__ rowptr,
                                                                size_t nrows) {
    const size_t stride = (size_t)gridDim.x * SP_THREADS;
    for (size_t r = (size_t)blockIdx.x * SP_THREADS + threadIdx.x; r <= nrows; r += stride) {
        const unsigned long long key = (unsigned long long)r << 32;
        size_t lo = 0, hi = nnz;
        while (lo < hi) {
            const size_t mid = lo + ((hi - lo) >> 1);
            if (__ldg(sorted + mid) < key) lo = mid + 1;
            else hi = mid;
        }
        rowptr[r] = (long long)lo;
    }
}

template <typename V>
int32_t csc_to_csr_t(dab_ctx* ctx, size_t m, size_t n, size_t nnz, const long long* colptr, const int32_t* rowval, const void* nzval,
                     long long* rowptr, int32_t* colidx, void* val) {
    unsigned long long* words = nullptr;
    unsigned long long* tmp = nullptr;
    if (nnz) {
        DAB_CUDA(ctx, cudaMallocAsync((void**)&words, nnz * 8, ctx->stream));
        DAB_CUDA(ctx, cudaMallocAsync((void**)&tmp, nnz * 8, ctx->stream));
        const int g = dab_grid_for(ctx, (nnz + SP_THREADS - 1) / SP_THREADS, 8);
        csr_pack_kernel<<<g, SP_THREADS, 0, ctx->stream>>>(rowval, words, nnz);
        DAB_LAUNCHED(ctx);
        int32_t st = dab_sort(ctx, DAB_I64, words, words, tmp, nnz);
        if (st != DAB_OK) return st;
        csr_unpack_kernel<V><<<g, SP_THREADS, 0, ctx->stream>>>(words, colptr, n, (const V*)nzval, colidx, (V*)val, nnz);
        DAB_LAUNCHED(ctx);
    }
    const int gr = dab_grid_for(ctx, (m + 1 + SP_THREADS - 1) / SP_THREADS, 8);
    csr_rowptr_kernel<<<gr, SP_THREADS, 0, ctx->stream>>>(words, nnz, rowptr, m);
    DAB_LAUNCHED(ctx);
    if (nnz) {
        DAB_CUDA(ctx, cudaFreeAsync(tmp, ctx->stream));
        DAB_CUDA(ctx, cudaFreeAsync(words, ctx->stream));
    }
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_spmv(dab_ctx* ctx, int32_t dtype, size_t nrows, size_t nnz, const void* ptr, const void* idx, const void* val, const void* x,
                 void* out) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64 || dtype == DAB_I32 || dtype == DAB_I64, DAB_ERR_UNSUPPORTED,
                "dab_spmv: dtype %d (served: F32 F64 I32 I64)", dtype);
    DAB_REQUIRE(ctx, nnz <= 0xFFFFFFFFull, DAB_ERR_UNSUPPORTED, "dab_spmv: chunks of 2^32 or more stored entries are not served");
    DAB_REQUIRE(ctx, nrows == 0 || (ptr && out), DAB_ERR_ARG, "dab_spmv: null pointer");
    DAB_REQUIRE(ctx, nnz == 0 || (idx && val && x), DAB_ERR_ARG, "dab_spmv: null pointer");
    if (nrows == 0) return DAB_OK;
    const long long* p = (const long long*)ptr;
    const int32_t* i = (const int32_t*)idx;
    switch (dtype) {
        case DAB_F32: return spmv_t<float>(ctx, nrows, nnz, p, i, val, x, out);
        case DAB_F64: return spmv_t<double>(ctx, nrows, nnz, p, i, val, x, out);
        case DAB_I32: return spmv_t<int32_t>(ctx, nrows, nnz, p, i, val, x, out);
        default: return spmv_t<int64_t>(ctx, nrows, nnz, p, i, val, x, out);
    }
}

int32_t dab_csc_to_csr(dab_ctx* ctx, int32_t dtype, size_t m, size_t n, size_t nnz, const void* colptr, const void* rowval, const void* nzval,
                       void* rowptr, void* colidx, void* val) {
    DAB_ENTER(ctx);
    const size_t es = dab_dtype_size(dtype);
    DAB_REQUIRE(ctx, dtype == DAB_F32 || dtype == DAB_F64 || dtype == DAB_I32 || dtype == DAB_I64, DAB_ERR_UNSUPPORTED,
                "dab_csc_to_csr: dtype %d (served: F32 F64 I32 I64)", dtype);
    DAB_REQUIRE(ctx, m <= 0x7FFFFFFFull && n <= 0x7FFFFFFFull, DAB_ERR_UNSUPPORTED,
                "dab_csc_to_csr: chunks of more than 2^31-1 rows or columns are not served");
    DAB_REQUIRE(ctx, nnz < 0xFFFFF000ull, DAB_ERR_UNSUPPORTED, "dab_csc_to_csr: chunks of 2^32 - 4096 or more stored entries are not served");
    DAB_REQUIRE(ctx, rowptr != nullptr, DAB_ERR_ARG, "dab_csc_to_csr: null pointer");
    DAB_REQUIRE(ctx, nnz == 0 || (colptr && rowval && nzval && colidx && val), DAB_ERR_ARG, "dab_csc_to_csr: null pointer");
    DAB_REQUIRE(ctx, nnz == 0 || n > 0, DAB_ERR_ARG, "dab_csc_to_csr: stored entries in a chunk without columns");
    const long long* cp = (const long long*)colptr;
    const int32_t* rv = (const int32_t*)rowval;
    if (es == 4) return csc_to_csr_t<uint32_t>(ctx, m, n, nnz, cp, rv, nzval, (long long*)rowptr, (int32_t*)colidx, val);
    return csc_to_csr_t<uint64_t>(ctx, m, n, nnz, cp, rv, nzval, (long long*)rowptr, (int32_t*)colidx, val);
}

}  // extern "C"
