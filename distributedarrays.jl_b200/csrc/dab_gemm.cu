// dab_gemm.cu -- K12: the tile product of the matrix-matrix mul! (widening row f4, the one contraction on the scope list).
//
// Replaces   localpart(A) * convert(localtype(B), Bjk)   /   transpose(localpart(A)) * ...   inside
// _matmatmul!(C::DMatrix, A::DMatrix, B::AbstractMatrix, alpha, beta, tA)  (reference src/linalg.jl:189-257, the remotecall at
// :218-226).  Column-major (Julia) operands:  R[m x n] = op(A) * B,  op(A) = A (m x k) or A^T (A stored k x m),  B is k x n.
// The caller combines the tile results exactly as the reference does (scale C by beta, add!(localpart(C), R, alpha) per tile).
//
// Float32 -> gemm_tf32x3_kernel, hand-written for sm_90a (Hopper):
//   * operands arrive by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B tensor maps) into a 6-stage shared-memory ring, completion on
//     mbarriers; out-of-range rows / columns / k are zero-filled by the TMA unit, so ragged edges need no special code.  One producer warp.
//   * "3xTF32": per 8-deep k-step the three products a_lo*b_hi + a_hi*b_lo + a_hi*b_hi (the dropped a_lo*b_lo term is 2^-22 relative).
//     The B tile (K-major in shared memory, as wgmma needs for tf32) is split into tf32 "hi" (round-to-nearest, in place) and "lo" (the
//     rounded remainder) by the consumer threads.  A goes to the tensor core from REGISTERS: an untransposed column-major A is MN-major,
//     which wgmma does not accept for tf32 from shared memory, so every thread loads its fragment from the swizzled tile and splits it there.
//   * two consumer warpgroups issue wgmma.mma_async m64n128k8 (a_hi x [b_hi | b_lo]) and m64n64k8 (a_lo x b_hi); CTA tile 128 x 64
//   * two-level accumulation, because the tensor core does not round its fp32 accumulator to nearest (the error grows with the number of
//     accumulating instructions): the register accumulators only sum TG_KC = 64 consecutive k, then each finished partial tile is
//     added to fp32 registers with round-to-nearest
// Everything else (Float64, Int32, Int64; Float32 operands whose base / leading dimension are not 16-byte aligned, which TMA cannot
// address) -> gemm_simt_kernel: shared-memory tiled FMA kernel, fp64 with DFMA, integers wrap like Julia's.
#include <cuda.h>

#include <map>
#include <mutex>
#include <utility>

#include "dab_common.cuh"

namespace {

// ======================================================================= generic SIMT tile kernel =====================================
constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;

template <typename T> __device__ __forceinline__ T gemm_fma(T a, T b, T c);
template <> __device__ __forceinline__ float gemm_fma<float>(float a, float b, float c) { return __fmaf_rn(a, b, c); }
template <> __device__ __forceinline__ double gemm_fma<double>(double a, double b, double c) { return __fma_rn(a, b, c); }
template <> __device__ __forceinline__ int32_t gemm_fma<int32_t>(int32_t a, int32_t b, int32_t c) {
    return (int32_t)((uint32_t)a * (uint32_t)b + (uint32_t)c);
}
template <> __device__ __forceinline__ long long gemm_fma<long long>(long long a, long long b, long long c) {
    return (long long)((unsigned long long)a * (unsigned long long)b + (unsigned long long)c);
}

template <typename T, bool TA>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const T* __restrict__ A, size_t lda, const T* __restrict__ B, size_t ldb, T* __restrict__ C,
                                                        size_t ldc, size_t m, size_t n, size_t k) {
    __shared__ T As[SG_BK][SG_BM + 1];
    __shared__ T Bs[SG_BK][SG_BN + 1];
    const size_t m0 = (size_t)blockIdx.x * SG_BM, n0 = (size_t)blockIdx.y * SG_BN;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    T acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = T(0);
    for (size_t k0 = 0; k0 < k; k0 += SG_BK) {
#pragma unroll
        for (int q = 0; q < (SG_BM * SG_BK) / 256; ++q) {
            const int idx = tid + q * 256;
            int i, kk;
            if (TA) { kk = idx % SG_BK; i = idx / SG_BK; } else { i = idx % SG_BM; kk = idx / SG_BM; }
            const size_t gi = m0 + i, gk = k0 + kk;
            T v = T(0);
            if (gi < m && gk < k) v = TA ? A[gk + gi * lda] : A[gi + gk * lda];
            As[kk][i] = v;
        }
#pragma unroll
        for (int q = 0; q < (SG_BN * SG_BK) / 256; ++q) {
            const int idx = tid + q * 256;
            const int kk = idx % SG_BK, j = idx / SG_BK;
            const size_t gj = n0 + j, gk = k0 + kk;
            Bs[kk][j] = (gj < n && gk < k) ? B[gk + gj * ldb] : T(0);
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < SG_BK; ++kk) {
            T a[4], b[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = As[kk][tx + 16 * r];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = Bs[kk][ty + 16 * c];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = gemm_fma<T>(a[r], b[c], acc[r][c]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const size_t gj = n0 + ty + 16 * c;
        if (gj >= n) continue;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const size_t gi = m0 + tx + 16 * r;
            if (gi < m) C[gi + gj * ldc] = acc[r][c];
        }
    }
}

template <typename T>
int32_t launch_simt(dab_ctx* ctx, int transA, size_t m, size_t n, size_t k, const T* A, size_t lda, const T* B, size_t ldb, T* C, size_t ldc) {
    const size_t gx = (m + SG_BM - 1) / SG_BM, gy = (n + SG_BN - 1) / SG_BN;
    if (gx > 0x7fffffffull || gy > 65535ull) return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_gemm: tile grid %zu x %zu too large", gx, gy);
    dim3 grid((unsigned)gx, (unsigned)gy);
    if (transA) gemm_simt_kernel<T, true><<<grid, 256, 0, ctx->stream>>>(A, lda, B, ldb, C, ldc, m, n, k);
    else gemm_simt_kernel<T, false><<<grid, 256, 0, ctx->stream>>>(A, lda, B, ldb, C, ldc, m, n, k);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// ======================================================================= wgmma 3xTF32 kernel ==========================================
constexpr int TG_M = 128, TG_N = 64, TG_K = 32, TG_STAGES = 6;
constexpr int TG_KC = 64;                                        // k extent of one register partial (a multiple of TG_K)
constexpr int TG_A_BYTES = TG_M * TG_K * 4;                      // 16 KiB: one A tile (128 x 32 fp32)
constexpr int TG_B_BYTES = TG_N * TG_K * 4;                      // 8 KiB: one B tile (32 x 64 fp32), K-major rows of 128 bytes
constexpr int TG_STAGE_BYTES = TG_A_BYTES + 2 * TG_B_BYTES;      // A, B_hi, B_lo (B_lo right behind B_hi: [B_hi | B_lo] is one N = 128 operand)
constexpr int TG_CONSUMERS = 256;                                // two warpgroups, 64 rows of the tile each
constexpr int TG_THREADS = TG_CONSUMERS + 32;                    // + one TMA producer warp
constexpr int TG_BAR_OFFSET = TG_STAGES * TG_STAGE_BYTES;
constexpr int TG_SMEM_BYTES = TG_BAR_OFFSET + 128 + 1024;        // + barriers + slack for the 1024-byte alignment of the swizzle atoms
static_assert(TG_SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(c0), "r"(c1)
                 : "memory");
}
// wgmma shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle (the layout TMA's SWIZZLE_128B writes): start
// address, leading byte offset (unused by swizzled K-major operands), stride byte offset = 1024 (8-row atoms of 128-byte rows), layout 1
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// D (64 x N fp32, registers) (+)= A (64 x 8 tf32, registers: rows g / g+8, k t / t+4 of the warp's 16-row slice) x B (8 x N tf32, shared)
__device__ __forceinline__ void wgmma_n128(float* d, const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n64(float* d, const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit_wait() {
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// keeps the compiler from moving reads / writes of an accumulator register across the asynchronous wgmma that owns it
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// fp32 -> (tf32 hi, tf32 lo) with INTEGER arithmetic: round-to-nearest (ties away, the semantics of cvt.rna.tf32.f32) is "add half an ulp of
// the 13 dropped bits, clear them"; IADD / LOP3 / FSUB run at full rate, cvt.rna.tf32.f32 does not.  Both halves have their low 13 bits
// cleared, so the products do not depend on how the tensor core treats the bits a tf32 operand drops.
__device__ __forceinline__ float tf32_rn(float v) { return __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u); }
__device__ __forceinline__ float4 split_tf32(float4& v) {   // v <- hi (tf32, round to nearest), returns lo = tf32_rn(v - hi)
    float4 lo;
    const float hx = tf32_rn(v.x), hy = tf32_rn(v.y), hz = tf32_rn(v.z), hw = tf32_rn(v.w);
    lo.x = tf32_rn(__fsub_rn(v.x, hx));
    lo.y = tf32_rn(__fsub_rn(v.y, hy));
    lo.z = tf32_rn(__fsub_rn(v.z, hz));
    lo.w = tf32_rn(__fsub_rn(v.w, hw));
    v = make_float4(hx, hy, hz, hw);
    return lo;
}

template <bool TA>
__global__ void __launch_bounds__(TG_THREADS, 1) gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                                                                    float* __restrict__ C, size_t ldc, uint32_t m, uint32_t n, uint32_t k, uint32_t kc_blocks) {
    extern __shared__ unsigned char tg_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tg_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar0 = sbase + TG_BAR_OFFSET;   // full[s] = bar0 + 8 s, empty[s] = bar0 + 8 (TG_STAGES + s)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t m0 = blockIdx.x * TG_M, n0 = blockIdx.y * TG_N;
    const uint32_t nkb = (k + TG_K - 1) / TG_K;
    if (threadIdx.x == 0) {
        for (int s = 0; s < TG_STAGES; ++s) {
            mbar_init(bar0 + 8 * s, 1);
            mbar_init(bar0 + 8 * (TG_STAGES + s), 2);   // one arrival per consumer warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == TG_CONSUMERS / 32) {
        // ===== TMA producer =====
        if (lane == 0) {
            for (uint32_t kb = 0; kb < nkb; ++kb) {
                const uint32_t s = kb % TG_STAGES, ph = (kb / TG_STAGES) & 1u;
                mbar_wait(bar0 + 8 * (TG_STAGES + s), ph ^ 1u);
                const uint32_t full = bar0 + 8 * s;
                mbar_expect_tx(full, TG_A_BYTES + TG_B_BYTES);
                const uint32_t a_dst = sbase + s * TG_STAGE_BYTES, b_dst = a_dst + TG_A_BYTES;
                const int32_t k0 = (int32_t)(kb * TG_K);
                if (TA) {
                    tma_load_2d(a_dst, &mapA, full, k0, (int32_t)m0);                       // box {32 k, 128 m}: K-major rows of 128 bytes
                } else {
#pragma unroll
                    for (int a = 0; a < 4; ++a)                                             // box {32 m, 32 k}: four M-blocks of 32 k-rows x 128 bytes
                        tma_load_2d(a_dst + a * 4096, &mapA, full, (int32_t)(m0 + 32 * a), k0);
                }
                tma_load_2d(b_dst, &mapB, full, k0, (int32_t)n0);                           // box {32 k, 64 n}
            }
        }
        return;
    }

    // ===== two consumer warpgroups: warpgroup wg owns tile rows 64 wg .. 64 wg + 63 =====
    const int tid = threadIdx.x, wg = warp >> 2, g = lane >> 2, t = lane & 3;
    const uint32_t r0 = 64u * wg + 16u * (warp & 3) + g;   // the thread's tile rows: r0 and r0 + 8
    // acc[0, 32): partial hi*hi product of the current k chunk; acc[32, 64) and acc2: the correction products a_hi*b_lo and a_lo*b_hi (kept
    // apart so that the two wgmmas of a k-step do not write the same registers, which would serialize them).  The tensor
    // core does not round its fp32 accumulator to nearest, and that error grows with the number of accumulating instructions: a partial only
    // sums TG_KC consecutive k before it is added to `sum` with round-to-nearest.
    float acc[64], acc2[32], sum[32];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) sum[i] = acc2[i] = 0.0f;
    uint32_t chunks_done = 0;
    for (uint32_t kb = 0; kb < nkb; ++kb) {
        const uint32_t s = kb % TG_STAGES, ph = (kb / TG_STAGES) & 1u;
        mbar_wait(bar0 + 8 * s, ph);
        unsigned char* st = smem + s * TG_STAGE_BYTES;
        // converters: B -> (tf32 hi in place, tf32 lo behind it), elementwise, so the swizzled layout is irrelevant
        float4* bh = reinterpret_cast<float4*>(st + TG_A_BYTES);
        float4* bl = bh + TG_B_BYTES / 16;
#pragma unroll
        for (int q = 0; q < TG_B_BYTES / 16 / TG_CONSUMERS; ++q) {
            const int i = tid + q * TG_CONSUMERS;
            float4 v = bh[i];
            const float4 lo = split_tf32(v);
            bh[i] = v;
            bl[i] = lo;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");                       // generic-proxy stores -> visible to wgmma
        asm volatile("bar.sync 1, %0;" ::"n"(TG_CONSUMERS) : "memory");
        const bool chunk_start = (kb % kc_blocks) == 0;
        const uint32_t b_hi = sbase + s * TG_STAGE_BYTES + TG_A_BYTES;
        const float* As = reinterpret_cast<const float*>(st);
#pragma unroll
        for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
#pragma unroll
        for (int i = 0; i < 32; ++i) fence_operand(acc2[i]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            // A fragment of k-step j, split into hi / lo in registers
            uint32_t ah[4], al[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const uint32_t r = r0 + 8u * (e & 1), kk = 8u * j + t + 4u * (e >> 1);
                // TA: row r holds 32 k (128 B), 16-byte chunk kk/4 stored at chunk (kk/4) ^ (r%8).  Otherwise: four 4 KiB blocks of 32 rows;
                // k-row kk of block r/32 holds 32 m, 16-byte chunk (r%32)/4 stored at chunk ((r%32)/4) ^ (kk%8)
                const uint32_t off = TA ? r * 32u + ((((kk >> 2) ^ (r & 7u))) << 2) + (kk & 3u)
                                        : (r >> 5) * 1024u + kk * 32u + (((((r & 31u) >> 2) ^ (kk & 7u))) << 2) + (r & 3u);
                const float v = As[off];
                const float hi = tf32_rn(v);
                ah[e] = __float_as_uint(hi);
                al[e] = __float_as_uint(tf32_rn(__fsub_rn(v, hi)));
            }
            // a_hi x [b_hi | b_lo] as ONE N = 128 instruction (b_lo sits right behind b_hi, same 1024-byte atom stride): columns 0-63 take
            // the main product, 64-127 the correction a_hi*b_lo; then a_lo x b_hi into acc2.  k-step j starts 32 B further inside the
            // swizzled 128-byte rows.
            const uint64_t dbh = gmma_desc(b_hi + 32u * j);
            wgmma_n128(acc, ah, dbh, (chunk_start && j == 0) ? 0u : 1u);
            wgmma_n64(acc2, al, dbh, (chunk_start && j == 0) ? 0u : 1u);
        }
        wgmma_commit_wait();
#pragma unroll
        for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
#pragma unroll
        for (int i = 0; i < 32; ++i) fence_operand(acc2[i]);
        if ((warp & 3) == 0 && lane == 0) mbar_arrive(bar0 + 8 * (TG_STAGES + s));            // this warpgroup is done with the stage
        if ((kb + 1) % kc_blocks == 0 || kb + 1 == nkb) {                                      // partial tile complete
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const float p = __fadd_rn(acc[i], __fadd_rn(acc[32 + i], acc2[i]));
                sum[i] = chunks_done == 0 ? p : __fadd_rn(sum[i], p);
            }
            ++chunks_done;
        }
    }
    // epilogue: accumulator element i of the thread is row r0 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 t + i % 2
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        const uint32_t row = m0 + r0 + 8u * ((i >> 1) & 1), col = n0 + 8u * (i >> 2) + 2u * t + (i & 1);
        if (row < m && col < n) C[row + (size_t)col * ldc] = sum[i];
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
        else cudaGetLastError();
    }
    return fn;
}

// 2-D fp32 tensor map over a column-major matrix: dim 0 = the contiguous direction (extent d0), dim 1 = columns (extent d1, ld elements apart)
int32_t make_map(dab_ctx* ctx, CUtensorMap* map, const float* base, size_t d0, size_t d1, size_t ld, uint32_t box0, uint32_t box1) {
    EncodeTiledFn enc = encode_tiled();
    if (!enc) return dab_fail(ctx, DAB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)d0, (cuuint64_t)d1};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {box0, box1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return dab_fail(ctx, DAB_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d (dims %zu x %zu, ld %zu)", (int)r, d0, d1, ld);
    return DAB_OK;
}

bool tma_ok(const void* p, size_t ld) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && (ld % 4) == 0 && ld < ((size_t)1 << 38); }

int32_t launch_tf32x3(dab_ctx* ctx, int transA, size_t m, size_t n, size_t k, const float* A, size_t lda, const float* B, size_t ldb, float* C, size_t ldc) {
    CUtensorMap mapA, mapB;
    // transposed A and B are K-major tiles (rows of 32 k); an untransposed A arrives as four blocks of 32 k-rows x 32 m, which the consumer
    // threads read back into wgmma's register fragments
    int32_t st = transA ? make_map(ctx, &mapA, A, k, m, lda, 32, 128) : make_map(ctx, &mapA, A, m, k, lda, 32, 32);
    if (st != DAB_OK) return st;
    st = make_map(ctx, &mapB, B, k, n, ldb, 32, TG_N);
    if (st != DAB_OK) return st;
    const size_t gx = (m + TG_M - 1) / TG_M, gy = (n + TG_N - 1) / TG_N;
    if (gx > 0x7fffffffull || gy > 65535ull) return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_gemm: tile grid %zu x %zu too large", gx, gy);
    auto launch = [&](auto kern) -> int32_t {
        static std::mutex mu;
        static std::map<std::pair<const void*, int>, bool> done;   // the >48 KiB opt-in is per (function, device)
        {
            std::lock_guard<std::mutex> lk(mu);
            auto key = std::make_pair((const void*)kern, ctx->device);
            if (!done.count(key)) {
                DAB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM_BYTES));
                done[key] = true;
            }
        }
        dim3 grid((unsigned)gx, (unsigned)gy);
        kern<<<grid, TG_THREADS, TG_SMEM_BYTES, ctx->stream>>>(mapA, mapB, C, ldc, (uint32_t)m, (uint32_t)n, (uint32_t)k, TG_KC / TG_K);
        return DAB_OK;
    };
    const int32_t rc = transA ? launch(gemm_tf32x3_kernel<true>) : launch(gemm_tf32x3_kernel<false>);
    if (rc != DAB_OK) return rc;
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" {

int32_t dab_gemm(dab_ctx* ctx, int32_t dtype, int32_t transA, size_t m, size_t n, size_t k, const void* A, size_t lda, const void* B, size_t ldb, void* C,
                 size_t ldc) {
    DAB_ENTER(ctx);
    if (m == 0 || n == 0) return DAB_OK;
    DAB_REQUIRE(ctx, C && (k == 0 || (A && B)), DAB_ERR_ARG, "dab_gemm: null pointer");
    DAB_REQUIRE(ctx, ldc >= m && (k == 0 || (lda >= (transA ? k : m) && ldb >= k)), DAB_ERR_ARG, "dab_gemm: leading dimension smaller than the rows");
    // B with ONE column (A * b for a DMatrix b of width 1, the narrowest block of a column-split B): the product is the matrix-vector
    // product K9 already serves at the HBM roofline (one read of A, fp64 / wrap-around carriers); a 128-wide tensor-core tile would spend
    // 127/128 of its MMAs on padding and stream A at the shared-memory rate.  Needs a dense A (lda == rows), which is what a chunk is.
    if (n == 1 && k > 0 && lda == (transA ? k : m) && (dtype == DAB_F32 || dtype == DAB_F64 || dtype == DAB_I32 || dtype == DAB_I64))
        return dab_gemv(ctx, dtype, transA ? 1 : 0, A, lda, transA ? m : k, B, C);
    switch (dtype) {
        case DAB_F32: {
            const bool big = m < ((size_t)1 << 31) && n < ((size_t)1 << 31) && k < ((size_t)1 << 31);
            if (k > 0 && big && tma_ok(A, lda) && tma_ok(B, ldb))
                return launch_tf32x3(ctx, transA, m, n, k, (const float*)A, lda, (const float*)B, ldb, (float*)C, ldc);
            return launch_simt<float>(ctx, transA, m, n, k, (const float*)A, lda, (const float*)B, ldb, (float*)C, ldc);
        }
        case DAB_F64: return launch_simt<double>(ctx, transA, m, n, k, (const double*)A, lda, (const double*)B, ldb, (double*)C, ldc);
        case DAB_I32: return launch_simt<int32_t>(ctx, transA, m, n, k, (const int32_t*)A, lda, (const int32_t*)B, ldb, (int32_t*)C, ldc);
        case DAB_I64: return launch_simt<long long>(ctx, transA, m, n, k, (const long long*)A, lda, (const long long*)B, ldb, (long long*)C, ldc);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_gemm: dtype %d (served: F32 F64 I32 I64)", dtype);
    }
}

}  // extern "C"
