// tools/sweep_stream.cu -- design-space sweep for the two streaming kernels of the hot path on a real GPU:
//   (1) y = a*x + b   (read 4 B + write 4 B per element)   and   (2) sum(x)   (read 4 B per element),
// over: vector loads in flight per thread (UNROLL), resident CTAs per SM, CTA size, tile interleaving vs contiguous per-CTA
// ranges, cache policy of the loads/stores, and a TMA (cp.async.bulk + mbarrier ring, in-place in shared memory) variant.
// Not part of the product: it only tells us which variant libdab200.so should ship.  Build: nvcc -O3 -gencode
// arch=compute_90a,code=sm_90a -fmad=false -o sweep_stream sweep_stream.cu ; run: ./sweep_stream [log2n]
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                          \
    do {                                                                               \
        cudaError_t e = (x);                                                           \
        if (e != cudaSuccess) {                                                        \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
            exit(1);                                                                   \
        }                                                                              \
    } while (0)

// ------------------------------------------------------------------ cache-policy flavoured 16-byte accesses
template <int POL>
__device__ __forceinline__ float4 ld16(const float4* p) {
    float4 r;
    if (POL == 0) r = *p;                                            // default ld.global
    else if (POL == 1) r = __ldcs(p);                               // ld.global.cs (evict-first)
    else if (POL == 2) r = __ldg(p);                                // ld.global.nc
    else if (POL == 3)
        asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    else
        asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
template <int POL>
__device__ __forceinline__ void st16(float4* p, float4 v) {
    if (POL == 0) *p = v;
    else if (POL == 1) __stcs(p, v);                                // st.global.cs
    else if (POL == 2) __stwt(p, v);                                // st.global.wt
    else if (POL == 3) __stcg(p, v);                                // st.global.cg
    else asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
}
__device__ __forceinline__ float4 aff(float4 v, float a, float b) {
    v.x = __fadd_rn(__fmul_rn(a, v.x), b);
    v.y = __fadd_rn(__fmul_rn(a, v.y), b);
    v.z = __fadd_rn(__fmul_rn(a, v.z), b);
    v.w = __fadd_rn(__fmul_rn(a, v.w), b);
    return v;
}

// ------------------------------------------------------------------ 32-byte (256-bit) accesses: ld/st .v8.b32 from sm_100 on,
// two 16-byte accesses before (sm_90 has no 256-bit global access)
struct __align__(32) f8 { float v[8]; };
template <int POL>
__device__ __forceinline__ f8 ld32(const f8* p) {
    f8 r;
#if __CUDA_ARCH__ < 1000
    reinterpret_cast<float4*>(r.v)[0] = ld16<POL == 0 ? 0 : POL == 1 ? 1 : 3>(reinterpret_cast<const float4*>(p));
    reinterpret_cast<float4*>(r.v)[1] = ld16<POL == 0 ? 0 : POL == 1 ? 1 : 3>(reinterpret_cast<const float4*>(p) + 1);
#else
    unsigned* u = reinterpret_cast<unsigned*>(r.v);
    if (POL == 0)
        asm volatile("ld.global.v8.b32 {%0,%1,%2,%3,%4,%5,%6,%7}, [%8];" : "=r"(u[0]), "=r"(u[1]), "=r"(u[2]), "=r"(u[3]), "=r"(u[4]), "=r"(u[5]), "=r"(u[6]), "=r"(u[7]) : "l"(p));
    else if (POL == 1)
        asm volatile("ld.global.L1::no_allocate.L2::evict_first.v8.b32 {%0,%1,%2,%3,%4,%5,%6,%7}, [%8];" : "=r"(u[0]), "=r"(u[1]), "=r"(u[2]), "=r"(u[3]), "=r"(u[4]), "=r"(u[5]), "=r"(u[6]), "=r"(u[7]) : "l"(p));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v8.b32 {%0,%1,%2,%3,%4,%5,%6,%7}, [%8];" : "=r"(u[0]), "=r"(u[1]), "=r"(u[2]), "=r"(u[3]), "=r"(u[4]), "=r"(u[5]), "=r"(u[6]), "=r"(u[7]) : "l"(p));
#endif
    return r;
}
template <int POL>
__device__ __forceinline__ void st32(f8* p, const f8& r) {
#if __CUDA_ARCH__ < 1000
    st16<POL == 0 ? 0 : 1>(reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(r.v)[0]);
    st16<POL == 0 ? 0 : 1>(reinterpret_cast<float4*>(p) + 1, reinterpret_cast<const float4*>(r.v)[1]);
#else
    const unsigned* u = reinterpret_cast<const unsigned*>(r.v);
    if (POL == 0)
        asm volatile("st.global.v8.b32 [%0], {%1,%2,%3,%4,%5,%6,%7,%8};" ::"l"(p), "r"(u[0]), "r"(u[1]), "r"(u[2]), "r"(u[3]), "r"(u[4]), "r"(u[5]), "r"(u[6]), "r"(u[7]));
    else
        asm volatile("st.global.L1::no_allocate.L2::evict_first.v8.b32 [%0], {%1,%2,%3,%4,%5,%6,%7,%8};" ::"l"(p), "r"(u[0]), "r"(u[1]), "r"(u[2]), "r"(u[3]), "r"(u[4]), "r"(u[5]), "r"(u[6]), "r"(u[7]));
#endif
}
template <int THREADS, int UNROLL, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_tiles32(f8* __restrict__ y, const f8* __restrict__ x, size_t nvec, float a, float b) {
    const size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const size_t base = t * TILE + threadIdx.x;
        f8 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld32<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
#pragma unroll
            for (int k = 0; k < 8; ++k) r[u].v[k] = __fadd_rn(__fmul_rn(a, r[u].v[k]), b);
            st32<SP>(y + base + (size_t)u * THREADS, r[u]);
        }
    }
}
template <int THREADS, int UNROLL, int LP>
__global__ void __launch_bounds__(THREADS) sum_tiles32(const f8* __restrict__ x, size_t nvec, double* __restrict__ out) {
    const size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    double acc = 0.0;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const size_t base = t * TILE + threadIdx.x;
        f8 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld32<LP>(x + base + (size_t)u * THREADS);
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) s += ((r[u].v[0] + r[u].v[1]) + (r[u].v[2] + r[u].v[3])) + ((r[u].v[4] + r[u].v[5]) + (r[u].v[6] + r[u].v[7]));
        acc += (double)s;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    __shared__ double sm[32];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < THREADS / 32; ++i) t += sm[i];
        out[blockIdx.x] = t;
    }
}

// ------------------------------------------------------------------ (1a) interleaved tiles, persistent grid
template <int THREADS, int UNROLL, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_tiles(float4* __restrict__ y, const float4* __restrict__ x, size_t nvec, float a, float b) {
    const size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const size_t base = t * TILE + threadIdx.x;
        float4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) st16<SP>(y + base + (size_t)u * THREADS, aff(r[u], a, b));
    }
}
// ------------------------------------------------------------------ (1b) one contiguous range per CTA
template <int THREADS, int UNROLL, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_ranges(float4* __restrict__ y, const float4* __restrict__ x, size_t nvec, float a, float b) {
    const size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    const size_t per = (ntiles + gridDim.x - 1) / gridDim.x;
    const size_t t0 = per * blockIdx.x, t1 = (t0 + per < ntiles) ? t0 + per : ntiles;
    for (size_t t = t0; t < t1; ++t) {
        const size_t base = t * TILE + threadIdx.x;
        float4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) st16<SP>(y + base + (size_t)u * THREADS, aff(r[u], a, b));
    }
}
// ------------------------------------------------------------------ (1c) non-persistent: one tile per CTA
template <int THREADS, int UNROLL, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_flat(float4* __restrict__ y, const float4* __restrict__ x, size_t nvec, float a, float b) {
    const size_t base = (size_t)blockIdx.x * THREADS * UNROLL + threadIdx.x;
    float4 r[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) st16<SP>(y + base + (size_t)u * THREADS, aff(r[u], a, b));
}

// ------------------------------------------------------------------ (1c') flat grid, K consecutive tiles per CTA
template <int THREADS, int UNROLL, int K, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_flatk(float4* __restrict__ y, const float4* __restrict__ x, size_t nvec, float a, float b) {
    size_t base = (size_t)blockIdx.x * THREADS * UNROLL * K + threadIdx.x;
#pragma unroll 1
    for (int k = 0; k < K; ++k, base += (size_t)THREADS * UNROLL) {
        float4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) st16<SP>(y + base + (size_t)u * THREADS, aff(r[u], a, b));
    }
}
template <int THREADS, int UNROLL, int LP, int SP>
__global__ void __launch_bounds__(THREADS) affine_flat32(f8* __restrict__ y, const f8* __restrict__ x, size_t nvec, float a, float b) {
    const size_t base = (size_t)blockIdx.x * THREADS * UNROLL + threadIdx.x;
    f8 r[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) r[u] = ld32<LP>(x + base + (size_t)u * THREADS);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
#pragma unroll
        for (int k = 0; k < 8; ++k) r[u].v[k] = __fadd_rn(__fmul_rn(a, r[u].v[k]), b);
        st32<SP>(y + base + (size_t)u * THREADS, r[u]);
    }
}
// flat sum: K consecutive tiles per CTA, one partial per CTA
template <int THREADS, int UNROLL, int K, int LP>
__global__ void __launch_bounds__(THREADS) sum_flatk(const float4* __restrict__ x, size_t nvec, double* __restrict__ out) {
    size_t base = (size_t)blockIdx.x * THREADS * UNROLL * K + threadIdx.x;
    double acc = 0.0;
#pragma unroll 1
    for (int k = 0; k < K; ++k, base += (size_t)THREADS * UNROLL) {
        float4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) s += (r[u].x + r[u].y) + (r[u].z + r[u].w);
        acc += (double)s;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    __shared__ double sm[32];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < THREADS / 32; ++i) t += sm[i];
        out[blockIdx.x] = t;
    }
}

// ------------------------------------------------------------------ (1d) TMA bulk copy ring, compute in place in shared memory
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int THREADS, int TILE_BYTES, int STAGES>
__global__ void __launch_bounds__(THREADS) affine_tma(float* __restrict__ y, const float* __restrict__ x, size_t n, float a, float b) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4* buf = reinterpret_cast<float4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    constexpr int TILE_F4 = TILE_BYTES / 16;
    constexpr size_t TILE_ELEMS = TILE_BYTES / 4;
    const size_t ntiles = n / TILE_ELEMS;
    // this CTA's tiles: blockIdx.x, blockIdx.x + gridDim.x, ...
    const size_t mine = (ntiles > blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES - 1 && (size_t)s < mine; ++s) {
            const size_t tile = blockIdx.x + (size_t)s * gridDim.x;
            mbar_expect_tx(&full[s], TILE_BYTES);
            bulk_load(buf + (size_t)s * TILE_F4, x + tile * TILE_ELEMS, TILE_BYTES, &full[s]);
        }
    }
    for (size_t it = 0; it < mine; ++it) {
        const int s = (int)(it % STAGES);
        const uint32_t parity = (uint32_t)((it / STAGES) & 1);
        mbar_wait(&full[s], parity);
        float4* p = buf + (size_t)s * TILE_F4;
#pragma unroll 4
        for (int i = threadIdx.x; i < TILE_F4; i += THREADS) p[i] = aff(p[i], a, b);
        fence_async();
        __syncthreads();
        if (threadIdx.x == 0) {
            const size_t tile = blockIdx.x + it * gridDim.x;
            bulk_store(y + tile * TILE_ELEMS, p, TILE_BYTES);
            bulk_commit();
            const size_t nxt = it + STAGES - 1;
            if (nxt < mine) {
                const int sn = (int)(nxt % STAGES);
                bulk_wait_read<1>();  // the store that last read stage sn (committed one iteration ago) is done with smem
                const size_t tn = blockIdx.x + nxt * gridDim.x;
                mbar_expect_tx(&full[sn], TILE_BYTES);
                bulk_load(buf + (size_t)sn * TILE_F4, x + tn * TILE_ELEMS, TILE_BYTES, &full[sn]);
            }
        }
    }
    if (threadIdx.x == 0) bulk_wait_read<0>();
}

// ------------------------------------------------------------------ (2) sum: read-only stream
template <int THREADS, int UNROLL, int LP>
__global__ void __launch_bounds__(THREADS) sum_tiles(const float4* __restrict__ x, size_t nvec, double* __restrict__ out) {
    const size_t TILE = (size_t)THREADS * UNROLL;
    const size_t ntiles = nvec / TILE;
    double acc = 0.0;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const size_t base = t * TILE + threadIdx.x;
        float4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) r[u] = ld16<LP>(x + base + (size_t)u * THREADS);
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) s += (r[u].x + r[u].y) + (r[u].z + r[u].w);
        acc += (double)s;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    __shared__ double sm[32];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < THREADS / 32; ++i) t += sm[i];
        out[blockIdx.x] = t;
    }
}

// ------------------------------------------------------------------ driver
struct Timer {
    cudaEvent_t e0, e1;
    Timer() {
        CK(cudaEventCreate(&e0));
        CK(cudaEventCreate(&e1));
    }
    template <typename F>
    float run(F f, int warm = 2, int iters = 8) {
        for (int i = 0; i < warm; ++i) f();
        CK(cudaEventRecord(e0));
        for (int i = 0; i < iters; ++i) f();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        CK(cudaGetLastError());
        return ms / iters;
    }
};

static float *gx, *gy;
static double* gout;
static size_t gn;
static int gsms;
static Timer* T;

template <int THREADS, int UNROLL, int LP, int SP>
void run_tiles(const char* shape, int per_sm) {
    size_t nvec = gn / 4;
    int grid = gsms * per_sm;
    float ms;
    if (shape[0] == 't') ms = T->run([&] { affine_tiles<THREADS, UNROLL, LP, SP><<<grid, THREADS>>>((float4*)gy, (const float4*)gx, nvec, 1.5f, 0.25f); });
    else if (shape[0] == 'r') ms = T->run([&] { affine_ranges<THREADS, UNROLL, LP, SP><<<grid, THREADS>>>((float4*)gy, (const float4*)gx, nvec, 1.5f, 0.25f); });
    else {
        grid = (int)(nvec / ((size_t)THREADS * UNROLL));
        ms = T->run([&] { affine_flat<THREADS, UNROLL, LP, SP><<<grid, THREADS>>>((float4*)gy, (const float4*)gx, nvec, 1.5f, 0.25f); });
    }
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, affine_tiles<THREADS, UNROLL, LP, SP>, THREADS, 0);
    printf("affine %-6s thr=%4d unroll=%d ld=%d st=%d ctas/sm=%2d (occ %2d) : %7.3f ms  %7.1f GB/s\n", shape, THREADS, UNROLL, LP, SP, per_sm, occ, ms,
           8.0 * gn / ms / 1e6);
    fflush(stdout);
}

template <int THREADS, int UNROLL, int LP, int SP>
void run_tiles32(int per_sm) {
    size_t nvec = gn / 8;
    int grid = gsms * per_sm;
    float ms = T->run([&] { affine_tiles32<THREADS, UNROLL, LP, SP><<<grid, THREADS>>>((f8*)gy, (const f8*)gx, nvec, 1.5f, 0.25f); });
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, affine_tiles32<THREADS, UNROLL, LP, SP>, THREADS, 0);
    printf("affine tile32 thr=%4d unroll=%d ld=%d st=%d ctas/sm=%2d (occ %2d) : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, LP, SP, per_sm, occ, ms, 8.0 * gn / ms / 1e6);
    fflush(stdout);
}
template <int THREADS, int UNROLL, int LP>
void run_sum32(int per_sm) {
    size_t nvec = gn / 8;
    int grid = gsms * per_sm;
    float ms = T->run([&] { sum_tiles32<THREADS, UNROLL, LP><<<grid, THREADS>>>((const f8*)gx, nvec, gout); });
    printf("sum    tile32 thr=%4d unroll=%d ld=%d      ctas/sm=%2d          : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, LP, per_sm, ms, 4.0 * gn / ms / 1e6);
    fflush(stdout);
}

template <int THREADS, int UNROLL, int K, int LP, int SP>
void run_flatk() {
    size_t nvec = gn / 4;
    int grid = (int)(nvec / ((size_t)THREADS * UNROLL * K));
    float ms = T->run([&] { affine_flatk<THREADS, UNROLL, K, LP, SP><<<grid, THREADS>>>((float4*)gy, (const float4*)gx, nvec, 1.5f, 0.25f); });
    printf("affine flatk  thr=%4d unroll=%d K=%2d ld=%d st=%d grid=%8d          : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, K, LP, SP, grid, ms, 8.0 * gn / ms / 1e6);
    fflush(stdout);
}
template <int THREADS, int UNROLL, int LP, int SP>
void run_flat32() {
    size_t nvec = gn / 8;
    int grid = (int)(nvec / ((size_t)THREADS * UNROLL));
    float ms = T->run([&] { affine_flat32<THREADS, UNROLL, LP, SP><<<grid, THREADS>>>((f8*)gy, (const f8*)gx, nvec, 1.5f, 0.25f); });
    printf("affine flat32 thr=%4d unroll=%d      ld=%d st=%d grid=%8d          : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, LP, SP, grid, ms, 8.0 * gn / ms / 1e6);
    fflush(stdout);
}
template <int THREADS, int UNROLL, int K, int LP>
void run_sumflatk() {
    size_t nvec = gn / 4;
    int grid = (int)(nvec / ((size_t)THREADS * UNROLL * K));
    if ((size_t)grid * 8 > (64u << 20)) { printf("skip\n"); return; }
    float ms = T->run([&] { sum_flatk<THREADS, UNROLL, K, LP><<<grid, THREADS>>>((const float4*)gx, nvec, gout); });
    printf("sum    flatk  thr=%4d unroll=%d K=%2d ld=%d      grid=%8d          : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, K, LP, grid, ms, 4.0 * gn / ms / 1e6);
    fflush(stdout);
}

template <int THREADS, int TILE_BYTES, int STAGES>
void run_tma(int per_sm) {
    size_t smem = (size_t)STAGES * TILE_BYTES + 8 * STAGES;
    CK(cudaFuncSetAttribute(affine_tma<THREADS, TILE_BYTES, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, affine_tma<THREADS, TILE_BYTES, STAGES>, THREADS, smem);
    if (per_sm > occ) return;
    int grid = gsms * per_sm;
    float ms = T->run([&] { affine_tma<THREADS, TILE_BYTES, STAGES><<<grid, THREADS, smem>>>(gy, gx, gn, 1.5f, 0.25f); });
    printf("affine tma    thr=%4d tile=%5d stages=%d ctas/sm=%2d (occ %2d) : %7.3f ms  %7.1f GB/s\n", THREADS, TILE_BYTES, STAGES, per_sm, occ, ms,
           8.0 * gn / ms / 1e6);
    fflush(stdout);
}

template <int THREADS, int UNROLL, int LP>
void run_sum(int per_sm) {
    size_t nvec = gn / 4;
    int grid = gsms * per_sm;
    float ms = T->run([&] { sum_tiles<THREADS, UNROLL, LP><<<grid, THREADS>>>((const float4*)gx, nvec, gout); });
    printf("sum    tiles  thr=%4d unroll=%d ld=%d      ctas/sm=%2d          : %7.3f ms  %7.1f GB/s\n", THREADS, UNROLL, LP, per_sm, ms, 4.0 * gn / ms / 1e6);
    fflush(stdout);
}

__global__ void fill_kernel(float* x, size_t n) {
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) x[i] = (float)(i & 1023) * 0.001f;
}

int main(int argc, char** argv) {
    int lg = argc > 1 ? atoi(argv[1]) : 30;
    gn = (size_t)1 << lg;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    gsms = prop.multiProcessorCount;
    printf("device %s, %d SMs, n = 2^%d floats\n", prop.name, gsms, lg);
    CK(cudaMalloc(&gx, gn * 4));
    CK(cudaMalloc(&gy, gn * 4));
    CK(cudaMalloc(&gout, 64 << 20));
    fill_kernel<<<gsms * 8, 256>>>(gx, gn);
    CK(cudaDeviceSynchronize());
    T = new Timer();
    // reference points: plain device-to-device memcpy (what a STREAM-style "copy" peak looks like)
    float ms = T->run([&] { CK(cudaMemcpyAsync(gy, gx, gn * 4, cudaMemcpyDeviceToDevice)); });
    printf("cudaMemcpy D2D                                                  : %7.3f ms  %7.1f GB/s\n", ms, 8.0 * gn / ms / 1e6);

    // ---- interleaved tiles: unroll x ctas/sm (evict-first loads and stores)
    run_tiles<256, 1, 1, 1>("tiles", 8);
    run_tiles<256, 2, 1, 1>("tiles", 8);
    run_tiles<256, 4, 1, 1>("tiles", 8);
    run_tiles<256, 4, 1, 1>("tiles", 4);
    run_tiles<256, 4, 1, 1>("tiles", 2);
    run_tiles<256, 8, 1, 1>("tiles", 4);
    run_tiles<256, 8, 1, 1>("tiles", 2);
    run_tiles<256, 2, 1, 1>("tiles", 4);
    run_tiles<512, 2, 1, 1>("tiles", 4);
    run_tiles<512, 4, 1, 1>("tiles", 2);
    run_tiles<1024, 2, 1, 1>("tiles", 2);
    run_tiles<1024, 1, 1, 1>("tiles", 2);
    run_tiles<128, 4, 1, 1>("tiles", 16);
    run_tiles<128, 8, 1, 1>("tiles", 8);
    // ---- contiguous per-CTA ranges and flat grids
    run_tiles<256, 4, 1, 1>("ranges", 8);
    run_tiles<256, 2, 1, 1>("ranges", 8);
    run_tiles<256, 4, 1, 1>("ranges", 4);
    run_tiles<256, 4, 1, 1>("flat", 0);
    run_tiles<256, 2, 1, 1>("flat", 0);
    run_tiles<256, 1, 1, 1>("flat", 0);
    run_tiles<512, 1, 1, 1>("flat", 0);
    run_tiles<1024, 1, 1, 1>("flat", 0);
    // ---- cache policies at the best-looking middle point
    run_tiles<256, 4, 0, 0>("tiles", 8);
    run_tiles<256, 4, 2, 0>("tiles", 8);
    run_tiles<256, 4, 3, 4>("tiles", 8);
    run_tiles<256, 4, 4, 1>("tiles", 8);
    run_tiles<256, 4, 1, 0>("tiles", 8);
    run_tiles<256, 4, 1, 2>("tiles", 8);
    run_tiles<256, 4, 1, 3>("tiles", 8);
    run_tiles<256, 2, 0, 0>("tiles", 8);
    run_tiles<256, 2, 3, 4>("tiles", 8);
    // ---- flat grids in depth
    run_flatk<256, 1, 1, 1, 1>();
    run_flatk<256, 2, 1, 1, 1>();
    run_flatk<256, 4, 1, 1, 1>();
    run_flatk<128, 2, 1, 1, 1>();
    run_flatk<128, 4, 1, 1, 1>();
    run_flatk<512, 2, 1, 1, 1>();
    run_flatk<256, 2, 1, 0, 0>();
    run_flatk<256, 2, 1, 3, 4>();
    run_flatk<256, 2, 1, 2, 1>();
    run_flatk<256, 2, 2, 1, 1>();
    run_flatk<256, 2, 4, 1, 1>();
    run_flatk<256, 2, 8, 1, 1>();
    run_flatk<256, 4, 2, 1, 1>();
    run_flatk<256, 4, 4, 1, 1>();
    run_flatk<256, 1, 4, 1, 1>();
    run_flatk<256, 1, 8, 1, 1>();
    run_flat32<256, 1, 1, 1>();
    run_flat32<256, 2, 1, 1>();
    run_flat32<128, 1, 1, 1>();
    run_flat32<128, 2, 1, 1>();
    run_flat32<256, 1, 0, 0>();
    run_sumflatk<256, 4, 1, 1>();
    run_sumflatk<256, 4, 2, 1>();
    run_sumflatk<256, 4, 4, 1>();
    run_sumflatk<256, 4, 8, 1>();
    run_sumflatk<256, 4, 16, 1>();
    run_sumflatk<256, 4, 32, 1>();
    run_sumflatk<256, 2, 4, 1>();
    run_sumflatk<256, 2, 8, 1>();
    run_sumflatk<256, 2, 16, 1>();
    run_sumflatk<256, 8, 4, 1>();
    run_sumflatk<256, 8, 8, 1>();
    run_sumflatk<512, 4, 4, 1>();
    run_sumflatk<128, 4, 8, 1>();
    run_sumflatk<256, 4, 8, 3>();
    // ---- 256-bit accesses
    run_tiles32<256, 1, 0, 0>(8);
    run_tiles32<256, 2, 0, 0>(8);
    run_tiles32<256, 2, 0, 0>(4);
    run_tiles32<256, 4, 0, 0>(4);
    run_tiles32<256, 1, 1, 1>(8);
    run_tiles32<256, 2, 1, 1>(8);
    run_tiles32<256, 2, 1, 1>(4);
    run_tiles32<256, 4, 1, 1>(4);
    run_tiles32<256, 2, 2, 1>(8);
    run_tiles32<512, 1, 1, 1>(4);
    run_tiles32<128, 2, 1, 1>(16);
    // ---- TMA ring
    run_tma<128, 8192, 4>(4);
    run_tma<128, 8192, 4>(6);
    run_tma<256, 16384, 3>(2);
    run_tma<256, 16384, 4>(2);
    run_tma<256, 16384, 4>(3);
    run_tma<256, 16384, 6>(2);
    run_tma<256, 32768, 3>(1);
    run_tma<256, 32768, 3>(2);
    run_tma<256, 32768, 4>(1);
    run_tma<512, 32768, 6>(1);
    run_tma<512, 65536, 3>(1);
    run_tma<128, 4096, 6>(8);
    run_tma<256, 8192, 6>(4);
    // ---- sum
    run_sum<256, 1, 1>(8);
    run_sum<256, 2, 1>(8);
    run_sum<256, 4, 1>(8);
    run_sum<256, 4, 1>(6);
    run_sum<256, 4, 1>(4);
    run_sum<256, 8, 1>(4);
    run_sum<256, 8, 1>(2);
    run_sum<512, 4, 1>(4);
    run_sum<512, 2, 1>(4);
    run_sum<1024, 2, 1>(2);
    run_sum<256, 4, 0>(8);
    run_sum<256, 4, 3>(8);
    run_sum<256, 8, 3>(4);
    run_sum32<256, 1, 1>(8);
    run_sum32<256, 2, 1>(8);
    run_sum32<256, 2, 1>(4);
    run_sum32<256, 4, 1>(4);
    run_sum32<256, 2, 0>(8);
    run_sum32<256, 2, 2>(8);
    run_sum32<512, 2, 1>(4);
    return 0;
}
