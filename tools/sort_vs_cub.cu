// tools/sort_vs_cub.cu -- K11 (dab_sort, through the C ABI of libdab200.so) against cub::DeviceRadixSort::SortKeys, the library
// yardstick.  Self-checking: every dab_sort result is compared element by element with CUB's on the device.  Not part of the product.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I include -o tools/sort_vs_cub tools/sort_vs_cub.cu \
//        -L distributedarrays.jl_b200/csrc -ldab200 -Xlinker -rpath -Xlinker '$ORIGIN/../distributedarrays.jl_b200/csrc'
//   tools/sort_vs_cub [log2n_64bit=27] [log2n_32bit=28] [reps=5] [variants=3] [test mask=0xff]
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cub/device/device_radix_sort.cuh>

#include "dab200.h"

#define CK(x)                                                                              \
    do {                                                                                   \
        cudaError_t e = (x);                                                               \
        if (e != cudaSuccess) {                                                            \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
            exit(1);                                                                       \
        }                                                                                  \
    } while (0)
#define DK(ctx, x)                                                                  \
    do {                                                                            \
        int32_t s = (x);                                                            \
        if (s != 0) {                                                               \
            printf("dab error %d: %s at line %d\n", s, dab_last_error(ctx), __LINE__); \
            exit(1);                                                                \
        }                                                                           \
    } while (0)

template <typename U>
__global__ void gen_kernel(U* x, size_t n, uint64_t seed, int mode) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t z = i + (seed + 1ull) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    if (mode == 1) z = z % 1000001ull;           // Int in 0:10^6 (the reference's own sort test data, test/darray.jl:1015-1025)
    x[i] = (U)z;
}
// uniform floats in [0,1) (what rand(Float32/Float64) gives): a realistic float key distribution, few exponent values
template <typename F>
__global__ void genf_kernel(F* x, size_t n, uint64_t seed) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t z = i + (seed + 1ull) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    x[i] = (F)((double)(z >> 11) * (1.0 / 9007199254740992.0)) - (F)0.5;
}
template <typename U>
__global__ void diff_kernel(const U* a, const U* b, size_t n, unsigned long long* bad) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && a[i] != b[i]) atomicAdd(bad, 1ull);
}

template <typename T, typename U>
void run(dab_ctx* ctx, const char* name, int32_t dtype, size_t n, int mode, int reps, int nvariants) {
    U *in, *out, *tmp, *ref;
    CK(cudaMalloc(&in, n * sizeof(U)));
    CK(cudaMalloc(&out, n * sizeof(U)));
    CK(cudaMalloc(&tmp, n * sizeof(U)));
    CK(cudaMalloc(&ref, n * sizeof(U)));
    unsigned long long* bad;
    CK(cudaMalloc(&bad, 8));
    void* stream_v;
    DK(ctx, dab_stream(ctx, &stream_v));
    cudaStream_t st = (cudaStream_t)stream_v;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    if (mode == 2) genf_kernel<T><<<blocks, 256, 0, st>>>((T*)in, n, 7);
    else gen_kernel<U><<<blocks, 256, 0, st>>>(in, n, 7, mode);
    CK(cudaStreamSynchronize(st));
    // ---- CUB yardstick (keys-only, out of place, full key width); sorts T so the order is the same as ours
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const T*)in, (T*)ref, n, 0, (int)(8 * sizeof(T)), st);
    void* cub_tmp;
    CK(cudaMalloc(&cub_tmp, cub_bytes));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    float best_cub = 1e30f;
    for (int r = 0; r < reps + 1; ++r) {
        CK(cudaEventRecord(e0, st));
        cub::DeviceRadixSort::SortKeys(cub_tmp, cub_bytes, (const T*)in, (T*)ref, n, 0, (int)(8 * sizeof(T)), st);
        CK(cudaEventRecord(e1, st));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r > 0 && ms < best_cub) best_cub = ms;
    }
    const double bytes_1pass = (double)n * sizeof(U);
    printf("%-28s n=%zu  CUB %.3f ms = %.2f Gkeys/s\n", name, n, best_cub, n / best_cub / 1e6);
    for (int v = 0; v < nvariants; ++v) {
        if (v > 0) break;   // the tile-shape sweep of round 2 (dab_set_option "sort_variant") has been folded into the shipped default
        float best = 1e30f;
        for (int r = 0; r < reps + 1; ++r) {
            CK(cudaEventRecord(e0, st));
            DK(ctx, dab_sort(ctx, dtype, in, out, tmp, n));
            CK(cudaEventRecord(e1, st));
            CK(cudaEventSynchronize(e1));
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (r > 0 && ms < best) best = ms;
        }
        CK(cudaMemsetAsync(bad, 0, 8, st));
        diff_kernel<U><<<blocks, 256, 0, st>>>(out, ref, n, bad);
        unsigned long long hbad = 0;
        CK(cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        // algorithmic bytes of a full-width sort: 1 histogram read + (read + write) per digit pass
        const int passes = (int)sizeof(U);
        const double algo = bytes_1pass * (1 + 2 * passes);
        printf("    dab_sort variant %d: %.3f ms = %.2f Gkeys/s  (%.2fx CUB)  full-width algorithmic traffic %.0f GB/s  mismatches vs CUB: %llu%s\n", v,
               best, n / best / 1e6, best_cub / best, algo / best / 1e6, hbad, hbad ? "  *** WRONG ***" : "");
    }
    // in-place call (in == out) must give the same result
    CK(cudaMemcpyAsync(out, in, n * sizeof(U), cudaMemcpyDeviceToDevice, st));
    DK(ctx, dab_sort(ctx, dtype, out, out, tmp, n));
    CK(cudaMemsetAsync(bad, 0, 8, st));
    diff_kernel<U><<<blocks, 256, 0, st>>>(out, ref, n, bad);
    unsigned long long hbad = 0;
    CK(cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    printf("    in-place: mismatches vs CUB: %llu%s\n", hbad, hbad ? "  *** WRONG ***" : "");
    CK(cudaFree(in));
    CK(cudaFree(out));
    CK(cudaFree(tmp));
    CK(cudaFree(ref));
    CK(cudaFree(cub_tmp));
    CK(cudaFree(bad));
}

int main(int argc, char** argv) {
    const int l64 = argc > 1 ? atoi(argv[1]) : 27, l32 = argc > 2 ? atoi(argv[2]) : 28, reps = argc > 3 ? atoi(argv[3]) : 5;
    const int nv = argc > 4 ? atoi(argv[4]) : 3;
    const int mask = argc > 5 ? atoi(argv[5]) : 0xff;   // bit k selects test k
    dab_ctx* ctx;
    DK(nullptr, dab_init(0, &ctx));
    if (mask & 1) run<int64_t, uint64_t>(ctx, "Int64 full range", DAB_I64, (size_t)1 << l64, 0, reps, nv);
    if (mask & 2) run<int64_t, uint64_t>(ctx, "Int64 in 0:10^6", DAB_I64, (size_t)1 << l64, 1, reps, nv);
    if (mask & 4) run<double, uint64_t>(ctx, "Float64 uniform [-.5,.5)", DAB_F64, (size_t)1 << l64, 2, reps, nv);
    if (mask & 8) run<int32_t, uint32_t>(ctx, "Int32 full range", DAB_I32, (size_t)1 << l32, 0, reps, nv);
    if (mask & 16) run<float, uint32_t>(ctx, "Float32 uniform [-.5,.5)", DAB_F32, (size_t)1 << l32, 2, reps, nv);
    if (mask & 32) run<int64_t, uint64_t>(ctx, "Int64 full range, ragged", DAB_I64, ((size_t)1 << 20) + 12345, 0, reps, nv);
    if (mask & 64) run<float, uint32_t>(ctx, "Float32, ragged small", DAB_F32, 5000, 2, reps, nv);
    dab_shutdown(ctx);
    return 0;
}
