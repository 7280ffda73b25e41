// sweep_gemv.cu -- which property of a column-major Float32 chunk whose leading dimension is not a multiple of 16 bytes makes A*x
// (K9) slow?  Drives the PRODUCT kernels (dab_gemv.cu is included, the rest comes from libdab200.so) with explicit grids:
//   * gemv_n_kernel<float,4,4,1> (aligned, consecutive columns) on m = 2^15, 32800 (multiple of 128 B), 32772 (multiple of 16 B only)
//   * gemv_n_phase_kernel<float,4,4> (4 phase classes, column stride 4) on the same aligned m's and on odd / even misaligned m's
// each over the number of column splits (CTAs in flight) and the CTAs resident per SM (limited through dynamic shared memory).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false --expt-relaxed-constexpr -o tools/sweep_gemv \
//        tools/sweep_gemv.cu -Ldistributedarrays.jl_b200/csrc -ldab200 -Xlinker -rpath='$ORIGIN/../distributedarrays.jl_b200/csrc'
#include "../distributedarrays.jl_b200/csrc/dab_gemv.cu"

#include <cstdlib>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

int main() {
    int sm = 0;
    CK(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0));
    const size_t cap = (size_t)32800 * 16400 + 64;
    float *A, *x, *y;
    double* part;
    CK(cudaMalloc(&A, cap * 4));
    CK(cudaMalloc(&x, 20000 * 4));
    CK(cudaMalloc(&y, 40000 * 4));
    CK(cudaMalloc(&part, (size_t)160 * 33000 * 8));
    CK(cudaMemset(A, 0, cap * 4));
    CK(cudaMemset(x, 0, 20000 * 4));
    auto kA = gemv_n_kernel<float, 4, 4, 1>;
    auto kP = gemv_n_phase_kernel<float, 4, 4>;
    CK(cudaFuncSetAttribute(kA, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CK(cudaFuncSetAttribute(kP, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    struct Case { size_t m, n; int phase; const char* what; };
    const Case cases[] = {
        {32768, 16384, 0, "aligned kernel, m = 2^15"},
        {32800, 16384, 0, "aligned kernel, m = 32800 (x128 B)"},
        {32772, 16384, 0, "aligned kernel, m = 32772 (x16 B only)"},
        {32768, 16384, 1, "phase kernel,   m = 2^15 (all phases 0)"},
        {32800, 16384, 1, "phase kernel,   m = 32800 (all phases 0)"},
        {32772, 16384, 1, "phase kernel,   m = 32772 (all phases 0)"},
        {32767, 16385, 1, "phase kernel,   m = 32767 (odd)"},
        {32769, 16384, 1, "phase kernel,   m = 32769 (odd)"},
        {32770, 16384, 1, "phase kernel,   m = 32770 (even)"},
    };
    for (const Case& c : cases) {
        const int VEC = 4, lrt = 8;
        const size_t rvecs = c.phase ? (c.m + 2 * (VEC - 1)) / VEC : (c.m + VEC - 1) / VEC;
        const size_t gx = (rvecs + 255) / 256;
        const int cmul = c.phase ? VEC : 1;
        for (int resident : {3, 4, 6})
            for (int frac8 : {4, 8, 16, 32}) {   // CTAs launched = frac8/8 of the resident slots
                size_t dyn = (size_t)(227 * 1024 / resident - 10 * 1024) / 1024 * 1024;
                if (dyn > 100 * 1024) dyn = 100 * 1024;
                int occ = 0;
                CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, c.phase ? (const void*)kP : (const void*)kA, 256, dyn));
                const size_t slots = (size_t)sm * occ * frac8 / 8;
                size_t nsplit = slots / (gx * cmul);
                if (nsplit < 1) nsplit = 1;
                const size_t nk = (c.n + cmul - 1) / cmul;
                size_t cps = (nk + nsplit - 1) / nsplit;
                nsplit = (nk + cps - 1) / cps;
                const size_t ny = nsplit * cmul;
                if (ny > 160) continue;
                dim3 grid((unsigned)gx, (unsigned)ny);
                auto launch = [&]() {
                    if (c.phase) kP<<<grid, 256, dyn>>>(A, c.m, c.n, x, lrt, cps, 0, part);
                    else kA<<<grid, 256, dyn>>>(A, c.m, c.n, x, lrt, cps, part, y);
                };
                for (int w = 0; w < 3; ++w) launch();
                CK(cudaDeviceSynchronize());
                CK(cudaEventRecord(e0));
                for (int r = 0; r < 10; ++r) launch();
                CK(cudaEventRecord(e1));
                CK(cudaDeviceSynchronize());
                float ms = 0;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                ms /= 10;
                printf("%-42s resident %d/SM, grid %3zu x %3zu = %5zu CTAs (%4.2f of slots): %.4f ms %7.1f GB/s\n", c.what, occ, gx, ny, gx * ny,
                       (double)(gx * ny) / ((double)sm * occ), ms, (double)c.m * c.n * 4 / ms / 1e6);
            }
    }
    return 0;
}
