// tools/sweep_sort.cu -- design sweep for K11 (the LSD radix sort of one chunk, distributedarrays.jl_b200/csrc/dab_sort.cu).
// Not part of the product: it tells us which scatter kernel libdab200.so should ship next.  Self-checking (every variant's output
// is compared with cub::DeviceRadixSort, which is also timed as the library yardstick).
//
// Why: round 1's scatter kernel runs at 0.85 TB/s (57 Gkeys/s per pass) and is 87 % of the sort.  The ncu capture + SASS show the
// key loads sunk into the ranking loop (one LDG per 32-key step = KPT serialised DRAM round trips per tile).  Variants here:
//   V0  round-1 structure: keys loaded into registers (predicated), ballots + per-warp counters, direct scatter
//   V1  keys staged global->shared with cp.async (all copies in flight by construction), ranking / scatter read shared memory
//   V2  V1 + the tile is reordered by digit in shared memory, then written in runs (consecutive threads -> consecutive addresses)
// each at KPT = 8 and 16 keys per thread, for 64-bit and 32-bit keys.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -o sweep_sort sweep_sort.cu ; run: ./sweep_sort [log2n]
#include <cuda_pipeline.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cub/device/device_radix_sort.cuh>
#include <vector>

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e = (x);                                                           \
        if (e != cudaSuccess) {                                                        \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
            exit(1);                                                                   \
        }                                                                              \
    } while (0)

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

struct Bases { uint32_t b[256]; };

__device__ __forceinline__ unsigned int match_digit(unsigned int dg) {
    unsigned int m = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 9; ++b) {
        const bool bit = (dg >> b) & 1u;
        const unsigned int bal = __ballot_sync(0xffffffffu, bit);
        m &= bit ? bal : ~bal;
    }
    return m;
}

template <typename U>
__global__ void gen_kernel(U* x, size_t n, uint64_t seed) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t z = i + (seed + 1ull) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    x[i] = (U)z;
}

// ---- all-digit histogram and per-tile counts (as in the product) ---------------------------------------------------------------
template <typename U, int KPT>
__global__ void __launch_bounds__(THREADS) hist_kernel(const U* __restrict__ in, size_t n, unsigned long long* __restrict__ ghist) {
    constexpr int DIGITS = sizeof(U);
    constexpr int TILE = THREADS * KPT;
    __shared__ unsigned int sh[DIGITS][256];
    for (int i = threadIdx.x; i < DIGITS * 256; i += THREADS) (&sh[0][0])[i] = 0;
    __syncthreads();
    for (size_t base = (size_t)blockIdx.x * TILE; base < n; base += (size_t)gridDim.x * TILE)
        for (int k = 0; k < KPT; ++k) {
            const size_t i = base + (size_t)k * THREADS + threadIdx.x;
            if (i < n) {
                const U key = in[i];
#pragma unroll
                for (int d = 0; d < DIGITS; ++d) atomicAdd(&sh[d][(unsigned)(key >> (8 * d)) & 255u], 1u);
            }
        }
    __syncthreads();
    for (int i = threadIdx.x; i < DIGITS * 256; i += THREADS) {
        const unsigned int c = (&sh[0][0])[i];
        if (c) atomicAdd(ghist + i, (unsigned long long)c);
    }
}

template <typename U, int KPT>
__global__ void __launch_bounds__(THREADS) count_kernel(const U* __restrict__ in, size_t n, int shift, unsigned int nblocks,
                                                        unsigned int* __restrict__ counts) {
    constexpr int TILE = THREADS * KPT;
    __shared__ unsigned int sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const size_t base = (size_t)blockIdx.x * TILE;
#pragma unroll 4
    for (int k = 0; k < KPT; ++k) {
        const size_t i = base + (size_t)k * THREADS + threadIdx.x;
        if (i < n) atomicAdd(&sh[(unsigned)(in[i] >> shift) & 255u], 1u);
    }
    __syncthreads();
    counts[(size_t)threadIdx.x * nblocks + blockIdx.x] = sh[threadIdx.x];
}

__global__ void __launch_bounds__(1024) scan_kernel(unsigned int* __restrict__ counts, unsigned int nblocks) {
    __shared__ unsigned int wsum[32];
    __shared__ unsigned int carry_s;
    unsigned int* row = counts + (size_t)blockIdx.x * nblocks;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (unsigned int base = 0; base < nblocks; base += 1024) {
        const unsigned int i = base + threadIdx.x;
        const unsigned int v = i < nblocks ? row[i] : 0;
        unsigned int inc = v;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const unsigned int t = __shfl_up_sync(0xffffffffu, inc, s);
            if (lane >= s) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            unsigned int w = wsum[lane];
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, w, s);
                if (lane >= s) w += t;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        const unsigned int carry = carry_s;
        const unsigned int excl = carry + (warp ? wsum[warp - 1] : 0) + inc - v;
        if (i < nblocks) row[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + wsum[31];
        __syncthreads();
    }
}

// ---- scatter variants ----------------------------------------------------------------------------------------------------------------
// V0: the round-1 kernel
template <typename U, int KPT>
__global__ void __launch_bounds__(THREADS) scatter_v0(const U* __restrict__ in, U* __restrict__ out, size_t n, int shift, unsigned int nblocks,
                                                      const unsigned int* __restrict__ offsets, Bases bases) {
    constexpr int TILE = THREADS * KPT;
    __shared__ unsigned int wc[WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < WARPS * 256; i += THREADS) (&wc[0][0])[i] = 0;
    __syncthreads();
    const size_t wbase = (size_t)blockIdx.x * TILE + (size_t)warp * (KPT * 32);
    const unsigned int lt = (1u << lane) - 1u;
    U key[KPT];
    unsigned short rank[KPT];
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const size_t i = wbase + (size_t)k * 32 + lane;
        key[k] = i < n ? __ldcs(in + i) : U(0);
    }
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const size_t i = wbase + (size_t)k * 32 + lane;
        const bool valid = i < n;
        const unsigned int dg = valid ? ((unsigned)(key[k] >> shift) & 255u) : 256u;
        const unsigned int grp = match_digit(dg);
        const unsigned int before = __popc(grp & lt);
        const int leader = __ffs(grp) - 1;
        unsigned int old = 0;
        if (valid && before == 0) old = atomicAdd(&wc[warp][dg], (unsigned int)__popc(grp));
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[k] = (unsigned short)(old + before);
    }
    __syncthreads();
    {
        const int d = threadIdx.x;
        unsigned int run = bases.b[d] + offsets[(size_t)d * nblocks + blockIdx.x];
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            const unsigned int c = wc[w][d];
            wc[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const size_t i = wbase + (size_t)k * 32 + lane;
        if (i < n) out[wc[warp][(unsigned)(key[k] >> shift) & 255u] + rank[k]] = key[k];
    }
}

// V1 / V2: keys staged in shared memory with cp.async; REORDER = write the tile in digit order (runs) instead of key by key
template <typename U, int KPT, bool REORDER>
__global__ void __launch_bounds__(THREADS) scatter_v12(const U* __restrict__ in, U* __restrict__ out, size_t n, int shift, unsigned int nblocks,
                                                       const unsigned int* __restrict__ offsets, Bases bases) {
    constexpr int TILE = THREADS * KPT;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    U* skey = reinterpret_cast<U*>(smem_raw);                                   // [TILE] keys in input order (warp-striped runs)
    U* sout = skey + (REORDER ? TILE : 0);                                      // [TILE] keys in digit order (V2 only)
    unsigned int* wc = reinterpret_cast<unsigned int*>(sout + TILE);            // [WARPS][256]
    unsigned int* dstart = wc + WARPS * 256;                                    // [256] first tile-local slot of each digit (V2)
    unsigned int* gbase = dstart + 256;                                         // [256] global address of that slot (V2)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t tbase = (size_t)blockIdx.x * TILE;
    const int wofs = warp * (KPT * 32);
    // stage: every copy of the warp's run is issued before anything waits
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const int t = wofs + k * 32 + lane;
        if (tbase + t < n) __pipeline_memcpy_async(skey + t, in + tbase + t, sizeof(U));
    }
    __pipeline_commit();
    for (int i = threadIdx.x; i < WARPS * 256; i += THREADS) wc[i] = 0;
    __pipeline_wait_prior(0);
    __syncthreads();
    const unsigned int lt = (1u << lane) - 1u;
    unsigned short rank[KPT];
#pragma unroll
    for (int k = 0; k < KPT; ++k) {
        const int t = wofs + k * 32 + lane;
        const bool valid = tbase + t < n;
        const unsigned int dg = valid ? ((unsigned)(skey[t] >> shift) & 255u) : 256u;
        const unsigned int grp = match_digit(dg);
        const unsigned int before = __popc(grp & lt);
        const int leader = __ffs(grp) - 1;
        unsigned int old = 0;
        if (valid && before == 0) old = atomicAdd(&wc[warp * 256 + dg], (unsigned int)__popc(grp));
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[k] = (unsigned short)(old + before);
    }
    __syncthreads();
    if (!REORDER) {
        {
            const int d = threadIdx.x;
            unsigned int run = bases.b[d] + offsets[(size_t)d * nblocks + blockIdx.x];
#pragma unroll
            for (int w = 0; w < WARPS; ++w) {
                const unsigned int c = wc[w * 256 + d];
                wc[w * 256 + d] = run;
                run += c;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < KPT; ++k) {
            const int t = wofs + k * 32 + lane;
            if (tbase + t < n) {
                const U key = skey[t];
                out[wc[warp * 256 + ((unsigned)(key >> shift) & 255u)] + rank[k]] = key;
            }
        }
    } else {
        // tile-local digit order: exclusive scan of the tile's digit totals (256 threads = 256 digits), then per-warp bases
        __shared__ unsigned int wsum[WARPS];
        const int d = threadIdx.x;
        unsigned int tot = 0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) tot += wc[w * 256 + d];
        unsigned int inc = tot;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const unsigned int v = __shfl_up_sync(0xffffffffu, inc, s);
            if (lane >= s) inc += v;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        unsigned int wpre = 0;
        for (int w = 0; w < warp; ++w) wpre += wsum[w];
        const unsigned int start = wpre + inc - tot;                                     // first tile-local slot of digit d
        dstart[d] = start;
        gbase[d] = bases.b[d] + offsets[(size_t)d * nblocks + blockIdx.x];
        unsigned int run = start;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            const unsigned int c = wc[w * 256 + d];
            wc[w * 256 + d] = run;
            run += c;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < KPT; ++k) {
            const int t = wofs + k * 32 + lane;
            if (tbase + t < n) {
                const U key = skey[t];
                sout[wc[warp * 256 + ((unsigned)(key >> shift) & 255u)] + rank[k]] = key;
            }
        }
        __syncthreads();
        const unsigned int cnt = (tbase + TILE <= n) ? TILE : (unsigned int)(n - tbase);
#pragma unroll
        for (int k = 0; k < KPT; ++k) {
            const unsigned int t = k * THREADS + threadIdx.x;                            // consecutive threads -> consecutive slots
            if (t < cnt) {
                const U key = sout[t];
                const unsigned int dg = (unsigned)(key >> shift) & 255u;
                out[gbase[dg] + (t - dstart[dg])] = key;
            }
        }
    }
}

// ---- driver -----------------------------------------------------------------------------------------------------------------------------
template <typename U, int KPT, int VARIANT>
float run_sort(const U* in, U* bufA, U* bufB, size_t n, unsigned long long* ghist, unsigned int* counts, int sm_count, int reps, U** result) {
    constexpr int DIGITS = sizeof(U);
    constexpr int TILE = THREADS * KPT;
    const unsigned int nblocks = (unsigned int)((n + TILE - 1) / TILE);
    std::vector<unsigned long long> hh(DIGITS * 256);
    size_t smem = 0;
    if (VARIANT == 1) smem = (size_t)TILE * sizeof(U) + WARPS * 256 * 4 + 2 * 256 * 4;
    if (VARIANT == 2) smem = (size_t)2 * TILE * sizeof(U) + WARPS * 256 * 4 + 2 * 256 * 4;
    if (VARIANT == 1) CK(cudaFuncSetAttribute(scatter_v12<U, KPT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (VARIANT == 2) CK(cudaFuncSetAttribute(scatter_v12<U, KPT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int r = 0; r < reps + 1; ++r) {
        CK(cudaEventRecord(e0));
        CK(cudaMemsetAsync(ghist, 0, DIGITS * 256 * 8));
        unsigned int hgrid = nblocks < (unsigned)sm_count * 4u ? nblocks : (unsigned)sm_count * 4u;
        hist_kernel<U, KPT><<<hgrid, THREADS>>>(in, n, ghist);
        CK(cudaMemcpy(hh.data(), ghist, DIGITS * 256 * 8, cudaMemcpyDeviceToHost));
        const U* src = in;
        for (int d = 0; d < DIGITS; ++d) {
            U* dst = ((DIGITS - 1 - d) % 2 == 0) ? bufA : bufB;                          // last pass lands in bufA
            Bases bases;
            unsigned long long run = 0;
            for (int b = 0; b < 256; ++b) {
                bases.b[b] = (uint32_t)run;
                run += hh[d * 256 + b];
            }
            count_kernel<U, KPT><<<nblocks, THREADS>>>(src, n, 8 * d, nblocks, counts);
            scan_kernel<<<256, 1024>>>(counts, nblocks);
            if (VARIANT == 0) scatter_v0<U, KPT><<<nblocks, THREADS>>>(src, dst, n, 8 * d, nblocks, counts, bases);
            if (VARIANT == 1) scatter_v12<U, KPT, false><<<nblocks, THREADS, smem>>>(src, dst, n, 8 * d, nblocks, counts, bases);
            if (VARIANT == 2) scatter_v12<U, KPT, true><<<nblocks, THREADS, smem>>>(src, dst, n, 8 * d, nblocks, counts, bases);
            src = dst;
        }
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r > 0 && ms < best) best = ms;                                               // r == 0 is the warm-up
    }
    *result = bufA;
    return best;
}

template <typename U>
bool same(const U* a, const U* b, size_t n) {
    std::vector<U> ha(n), hb(n);
    CK(cudaMemcpy(ha.data(), a, n * sizeof(U), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hb.data(), b, n * sizeof(U), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i)
        if (ha[i] != hb[i]) {
            printf("    MISMATCH at %zu\n", i);
            return false;
        }
    return true;
}

template <typename U>
void sweep(const char* name, size_t n, int sm_count) {
    U *in, *a, *b, *ref;
    CK(cudaMalloc(&in, n * sizeof(U)));
    CK(cudaMalloc(&a, n * sizeof(U)));
    CK(cudaMalloc(&b, n * sizeof(U)));
    CK(cudaMalloc(&ref, n * sizeof(U)));
    gen_kernel<U><<<(unsigned)((n + 255) / 256), 256>>>(in, n, 42);
    unsigned long long* ghist;
    unsigned int* counts;
    CK(cudaMalloc(&ghist, 8 * 256 * 8));
    CK(cudaMalloc(&counts, (size_t)256 * ((n + 2047) / 2048) * 4));
    // library yardstick + reference result
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, in, ref, n);
    CK(cudaMalloc(&tmp, tmp_bytes));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    float cub_ms = 1e30f;
    for (int r = 0; r < 4; ++r) {
        CK(cudaEventRecord(e0));
        cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, in, ref, n);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r > 0 && ms < cub_ms) cub_ms = ms;
    }
    printf("%s n=%zu: cub::DeviceRadixSort (library yardstick) %8.3f ms %7.2f Gkeys/s\n", name, n, cub_ms, n / cub_ms / 1e6);
    U* res;
    float ms;
#define RUN(K, V, label)                                                                                             \
    ms = run_sort<U, K, V>(in, a, b, n, ghist, counts, sm_count, 3, &res);                                           \
    printf("  %-44s KPT=%2d %8.3f ms %7.2f Gkeys/s  %s\n", label, K, ms, n / ms / 1e6, same(res, ref, n) ? "ok" : "WRONG"); \
    fflush(stdout);
    RUN(8, 0, "V0 register keys, direct scatter (round 1)")
    RUN(16, 0, "V0 register keys, direct scatter (round 1)")
    RUN(8, 1, "V1 cp.async staged keys, direct scatter")
    RUN(16, 1, "V1 cp.async staged keys, direct scatter")
    RUN(8, 2, "V2 staged + reorder in shared, run writes")
    RUN(16, 2, "V2 staged + reorder in shared, run writes")
#undef RUN
    CK(cudaFree(in));
    CK(cudaFree(a));
    CK(cudaFree(b));
    CK(cudaFree(ref));
    CK(cudaFree(ghist));
    CK(cudaFree(counts));
    CK(cudaFree(tmp));
}

int main(int argc, char** argv) {
    const int lg = argc > 1 ? atoi(argv[1]) : 27;
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    printf("%s, %d SMs; unsigned keys (the product adds an order-preserving bijection on the first read / last write)\n", p.name,
           p.multiProcessorCount);
    sweep<uint64_t>("u64", (size_t)1 << lg, p.multiProcessorCount);
    sweep<uint32_t>("u32", (size_t)1 << (lg + 1), p.multiProcessorCount);
    return 0;
}
