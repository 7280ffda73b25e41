// dab_sortperm_slices.cu -- K26, sortperm(A; dims) of one chunk in which the sorted dimension is whole: for every fibre of the chunk collapsed
// to (inner, len, outer), the 1-based global linear indices of its elements in the stable isless order of their keys (and, optionally, the
// values moved to the same places).  The index arithmetic, the pair packing and the compare live in dab_sortperm_slices_core.cuh.
//   len <= DAB_SORTPERM_SLICES_SMEM_LEN  sortperm_slices_kernel: dab_sort_slices' structure, one CTA sorts a group of fibres in shared
//                                        memory with a bitonic network over (radix key, position) pairs
//   longer fibres                        two chunk-wide stable K21 passes (dab_sort_pairs), by key and then by fibre id, and two small
//                                        kernels around them: the launch count does not depend on the number of fibres
#include <map>
#include <mutex>
#include <utility>

#include "dab_common.cuh"
#include "dab_sortperm_slices_core.cuh"

namespace {

// ---- short fibres -------------------------------------------------------------------------------------------------------------------
// Shared memory per CTA: the fibre bases of the group (SPS_MAX_FIBRES Int64), then SPS_CAP 8-byte slot words (fibre pads included), then
// for 64-bit keys SPS_CAP 4-byte positions.  Fibres are P2 + 1 slots apart, as in dab_sort_slices (conflict-free transposed staging).
constexpr int SPS_THREADS = 512;
constexpr unsigned int SPS_CAP = DAB_SORTPERM_SLICES_SMEM_LEN + 64;
constexpr unsigned int SPS_MAX_FIBRES = 1024;                     // fibres per group (only fibres of <= 4 elements reach it)
constexpr size_t SPS_BASE_BYTES = SPS_MAX_FIBRES * sizeof(long long);

__device__ __forceinline__ void sps_copy_val(int val_bytes, const void* vals, size_t src, void* vals_out, size_t dst) {
    if (val_bytes == 4) static_cast<uint32_t*>(vals_out)[dst] = static_cast<const uint32_t*>(vals)[src];
    else static_cast<unsigned long long*>(vals_out)[dst] = static_cast<const unsigned long long*>(vals)[src];
}

template <typename T>
__global__ void __launch_bounds__(SPS_THREADS) sortperm_slices_kernel(const typename SortKey<T>::U* __restrict__ keys, const SpsMap m,
                                                                      size_t inner, unsigned int len, size_t outer, unsigned int log2p2,
                                                                      unsigned int B, size_t ngroups, int64_t* __restrict__ perm, int val_bytes,
                                                                      const void* __restrict__ vals, void* __restrict__ vals_out) {
    using U = typename SortKey<T>::U;
    using SL = SpsSlot<U>;
    extern __shared__ __align__(16) unsigned char sps_smem[];
    long long* fb = reinterpret_cast<long long*>(sps_smem);
    const unsigned int p2 = 1u << log2p2, S = p2 + 1u;
    unsigned long long* w = reinterpret_cast<unsigned long long*>(sps_smem + SPS_BASE_BYTES);
    unsigned int* ps = reinterpret_cast<unsigned int*>(w + (size_t)B * S);
    for (size_t g = blockIdx.x; g < ngroups; g += gridDim.x) {
        const SpsGroup G = sps_group(g, inner, len, outer, B);
        const unsigned int nf = G.nf;
        for (unsigned int t = threadIdx.x; t < nf; t += SPS_THREADS)
            fb[t] = inner == 1 ? sps_fibre_base(m, 0, G.o0 + t) : sps_fibre_base(m, G.i0 + t, G.o0);
        for (unsigned int t = threadIdx.x; t < nf * len; t += SPS_THREADS) {
            unsigned int b, r;
            const size_t off = sps_group_elem(inner, len, nf, t, &b, &r);
            w[b * S + r] = SL::word(sortby_radix_key<T>(keys[G.base + off]), r);
            if constexpr (SL::SPLIT) ps[b * S + r] = r;
        }
        if (len < p2)
            for (unsigned int t = threadIdx.x; t < nf * p2; t += SPS_THREADS) {
                const unsigned int b = t >> log2p2, r = t & (p2 - 1u);
                if (r >= len) {
                    w[b * S + r] = SL::pad();
                    if constexpr (SL::SPLIT) ps[b * S + r] = ~0u;
                }
            }
        __syncthreads();
        const unsigned int half = (nf * p2) >> 1;
        for (unsigned int k = 2; k <= p2; k <<= 1)
            for (unsigned int j = k >> 1; j > 0; j >>= 1) {
                for (unsigned int p = threadIdx.x; p < half; p += SPS_THREADS) {
                    const unsigned int i = slices_bitonic_lo(p, j);
                    const unsigned int ia = slices_smem_index(i, log2p2), ic = slices_smem_index(i + j, log2p2);
                    unsigned long long x = w[ia], y = w[ic];
                    unsigned int px = 0, py = 0;
                    if constexpr (SL::SPLIT) {
                        px = ps[ia];
                        py = ps[ic];
                    }
                    sps_cmpx<SL::SPLIT>(x, y, px, py, slices_bitonic_asc(i, k, p2));
                    w[ia] = x;
                    w[ic] = y;
                    if constexpr (SL::SPLIT) {
                        ps[ia] = px;
                        ps[ic] = py;
                    }
                }
                __syncthreads();
            }
        for (unsigned int t = threadIdx.x; t < nf * len; t += SPS_THREADS) {
            unsigned int b, r;
            const size_t off = sps_group_elem(inner, len, nf, t, &b, &r);
            const unsigned int s = SL::pos(w[b * S + r], SL::SPLIT ? ps[b * S + r] : 0u);
            perm[G.base + off] = fb[b] + (long long)s * (long long)m.gdim;
            if (vals_out) sps_copy_val(val_bytes, vals, G.base + sps_group_offset(inner, len, b, s), vals_out, G.base + off);
        }
        __syncthreads();                                          // shared memory is reused by the next group
    }
}

template <typename T>
int32_t sortperm_slices_smem(dab_ctx* ctx, const void* keys, const SpsMap& m, size_t inner, size_t len, size_t outer, int64_t* perm,
                             int32_t val_bytes, const void* vals, void* vals_out) {
    using U = typename SortKey<T>::U;
    constexpr size_t slot_bytes = sizeof(unsigned long long) + (SpsSlot<U>::SPLIT ? sizeof(unsigned int) : 0);
    constexpr size_t max_smem = SPS_BASE_BYTES + (size_t)SPS_CAP * slot_bytes;
    const unsigned int log2p2 = slices_log2_ceil(len);
    unsigned int B = SPS_CAP / ((1u << log2p2) + 1u);
    if (B > SPS_MAX_FIBRES) B = SPS_MAX_FIBRES;
    const size_t ngroups = sps_ngroups(inner, outer, B);
    auto kern = sortperm_slices_kernel<T>;
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
            DAB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, SPS_THREADS, max_smem));
            it = seen.emplace(key, nb < 1 ? 1 : nb).first;
        }
        per_sm = it->second;
    }
    const size_t smem = SPS_BASE_BYTES + (size_t)B * ((1u << log2p2) + 1u) * slot_bytes;
    const int grid = dab_grid_for(ctx, ngroups, per_sm * 4);
    kern<<<grid, SPS_THREADS, smem, ctx->stream>>>((const U*)keys, m, inner, (unsigned int)len, outer, log2p2, B, ngroups, perm, val_bytes,
                                                   vals, vals_out);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// ---- long fibres --------------------------------------------------------------------------------------------------------------------
constexpr int SPS_FLAT_THREADS = 256;

// fid[j] = fibre id of the chunk position pos1[j]; the element at position 0 of each fibre also writes the fibre's base index
__global__ void __launch_bounds__(SPS_FLAT_THREADS) sortperm_fibre_id_kernel(const int64_t* __restrict__ pos1, size_t n, unsigned long long inner,
                                                                             unsigned long long len, const SpsMap m, int32_t* __restrict__ fid,
                                                                             long long* __restrict__ fbase) {
    for (size_t j = (size_t)blockIdx.x * SPS_FLAT_THREADS + threadIdx.x; j < n; j += (size_t)gridDim.x * SPS_FLAT_THREADS) {
        unsigned int s;
        const unsigned int f = sps_fibre_id((unsigned long long)pos1[j], inner, len, &s);
        fid[j] = (int32_t)f;
        if (s == 0) {
            unsigned long long i;
            const unsigned long long o = sps_divmod(f, inner, &i);
            fbase[f] = sps_fibre_base(m, i, o);
        }
    }
}

// entry k of the fibre-major order (chunk position pos2[k]) is rank k mod len of its fibre: its global index and value go to their place
__global__ void __launch_bounds__(SPS_FLAT_THREADS) sortperm_finish_kernel(const int64_t* __restrict__ pos2, size_t n, unsigned long long inner,
                                                                           unsigned long long len, const long long* __restrict__ fbase,
                                                                           unsigned long long gdim, int64_t* __restrict__ perm, int val_bytes,
                                                                           const void* __restrict__ vals, void* __restrict__ vals_out) {
    for (size_t k = (size_t)blockIdx.x * SPS_FLAT_THREADS + threadIdx.x; k < n; k += (size_t)gridDim.x * SPS_FLAT_THREADS) {
        const unsigned long long q = (unsigned long long)pos2[k];
        unsigned int s;
        const unsigned int f = sps_fibre_id(q, inner, len, &s);
        const size_t dst = sps_out_index(k, inner, len);
        perm[dst] = fbase[f] + (long long)s * (long long)gdim;
        if (vals_out) sps_copy_val(val_bytes, vals, q, vals_out, dst);
    }
}

inline size_t sps_stride(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

int32_t sortperm_slices_long(dab_ctx* ctx, int32_t key_dtype, int key_bytes, const void* keys, const SpsMap& m, size_t inner, size_t len,
                             size_t outer, int64_t* perm, int32_t val_bytes, const void* vals, void* vals_out) {
    const size_t n = inner * len * outer, nfib = inner * outer;
    size_t s1 = 0, s2 = 0;
    int32_t st = dab_sort_pairs_scratch_bytes(key_dtype, n, &s1);
    if (st == DAB_OK) st = dab_sort_pairs_scratch_bytes(DAB_I32, n, &s2);
    if (st != DAB_OK) return dab_fail(ctx, st, "dab_sortperm_slices: key dtype %d", key_dtype);
    const size_t sk = sps_stride(n * key_bytes), sf = sps_stride(n * 4), sp = sps_stride(n * 8), sb = sps_stride(nfib * 8);
    const size_t ss = sps_stride(s1 > s2 ? s1 : s2);
    char* blk = nullptr;
    st = dab_alloc(ctx, sk + 2 * sf + 2 * sp + sb + ss, (void**)&blk);
    if (st != DAB_OK) return st;
    void* keys_out = blk;                                         // pass 1's sorted keys (not used)
    int32_t* fid = (int32_t*)(blk + sk);
    int32_t* fid_out = (int32_t*)(blk + sk + sf);                 // pass 2's sorted fibre ids (not used)
    int64_t* pos1 = (int64_t*)(blk + sk + 2 * sf);
    int64_t* pos2 = (int64_t*)(blk + sk + 2 * sf + sp);
    long long* fbase = (long long*)(blk + sk + 2 * sf + 2 * sp);
    void* scratch = blk + sk + 2 * sf + 2 * sp + sb;
    const int grid = dab_grid_for(ctx, (n + SPS_FLAT_THREADS - 1) / SPS_FLAT_THREADS, 8);
    st = dab_sort_pairs(ctx, key_dtype, keys, keys_out, nullptr, 0, pos1, scratch, ss, n);
    if (st == DAB_OK) {
        sortperm_fibre_id_kernel<<<grid, SPS_FLAT_THREADS, 0, ctx->stream>>>(pos1, n, inner, len, m, fid, fbase);
        ctx->launches++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) st = dab_fail_cuda(ctx, e, "sortperm_fibre_id_kernel", __FILE__, __LINE__);
    }
    if (st == DAB_OK) st = dab_sort_pairs(ctx, DAB_I32, fid, fid_out, pos1, 0, pos2, scratch, ss, n);
    if (st == DAB_OK) {
        sortperm_finish_kernel<<<grid, SPS_FLAT_THREADS, 0, ctx->stream>>>(pos2, n, inner, len, fbase, m.gdim, perm, val_bytes, vals, vals_out);
        ctx->launches++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) st = dab_fail_cuda(ctx, e, "sortperm_finish_kernel", __FILE__, __LINE__);
    }
    char keep[512];
    memcpy(keep, ctx->err, sizeof keep);                          // the free must not overwrite the text of a failure
    dab_free(ctx, blk);
    memcpy(ctx->err, keep, sizeof keep);
    return st;
}

}  // namespace

extern "C" {

int32_t dab_sortperm_slices(dab_ctx* ctx, int32_t key_dtype, const void* keys, int32_t ndim, const size_t* chunk_dims, const size_t* chunk_lo,
                            const size_t* global_dims, int32_t dim, int64_t* perm, int32_t val_bytes, const void* vals, void* vals_out) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, chunk_dims && chunk_lo && global_dims, DAB_ERR_ARG, "dab_sortperm_slices: null dims");
    DAB_REQUIRE(ctx, ndim <= DAB_SPS_MAX_DIMS, DAB_ERR_UNSUPPORTED, "dab_sortperm_slices: %d dims (served: up to %d)", ndim, DAB_SPS_MAX_DIMS);
    DAB_REQUIRE(ctx, ndim >= 1 && dim >= 1 && dim <= ndim, DAB_ERR_ARG, "dab_sortperm_slices: dim %d of a %d-dimensional chunk", dim, ndim);
    SpsMap m;
    DAB_REQUIRE(ctx, sps_make_map(ndim, chunk_dims, chunk_lo, global_dims, dim, &m), DAB_ERR_ARG,
                "dab_sortperm_slices: dimension %d is not whole in the chunk, or the chunk lies outside the array", dim);
    int key_bytes = 0;
    switch (key_dtype) {
        case DAB_F32: case DAB_I32: key_bytes = 4; break;
        case DAB_F64: case DAB_I64: key_bytes = 8; break;
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_sortperm_slices: key dtype %d (served: Float32 Float64 Int32 Int64)", key_dtype);
    }
    DAB_REQUIRE(ctx, (vals == nullptr) == (vals_out == nullptr), DAB_ERR_ARG, "dab_sortperm_slices: vals and vals_out go together");
    DAB_REQUIRE(ctx, vals == nullptr || val_bytes == 4 || val_bytes == 8, DAB_ERR_ARG, "dab_sortperm_slices: val_bytes %d (4 or 8)", val_bytes);
    size_t inner = 1, outer = 1;
    for (int k = 0; k < dim - 1; ++k) inner *= chunk_dims[k];
    for (int k = dim; k < ndim; ++k) outer *= chunk_dims[k];
    const size_t len = chunk_dims[dim - 1], n = inner * len * outer;
    if (n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, keys && perm, DAB_ERR_ARG, "dab_sortperm_slices: null pointer");
    if (len > DAB_SORTPERM_SLICES_SMEM_LEN) {
        DAB_REQUIRE(ctx, n < 0xFFFFF000ull, DAB_ERR_UNSUPPORTED,
                    "dab_sortperm_slices: chunks of 2^32 - 4096 or more elements with fibres longer than %d are not served",
                    DAB_SORTPERM_SLICES_SMEM_LEN);
        return sortperm_slices_long(ctx, key_dtype, key_bytes, keys, m, inner, len, outer, perm, val_bytes, vals, vals_out);
    }
    switch (key_dtype) {
        case DAB_F32: return sortperm_slices_smem<float>(ctx, keys, m, inner, len, outer, perm, val_bytes, vals, vals_out);
        case DAB_F64: return sortperm_slices_smem<double>(ctx, keys, m, inner, len, outer, perm, val_bytes, vals, vals_out);
        case DAB_I32: return sortperm_slices_smem<int32_t>(ctx, keys, m, inner, len, outer, perm, val_bytes, vals, vals_out);
        default: return sortperm_slices_smem<int64_t>(ctx, keys, m, inner, len, outer, perm, val_bytes, vals, vals_out);
    }
}

}  // extern "C"
