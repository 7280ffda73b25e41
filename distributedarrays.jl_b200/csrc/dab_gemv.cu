// dab_gemv.cu -- K9: the per-tile matrix-vector product of mul!(y::DVector, A::DMatrix, x) (reference src/linalg.jl:78-118) and of
// its adjoint/transpose form (:120-167):   R[i,j] = localpart(A) * xj   /   localpart(A)' * xj   on one column-major chunk.
//
// Roofline: HBM.  Every element of the chunk is read exactly once (elem_bytes per element); x (one column / row block of the
// vector) is re-read out of L1/L2, the result vector is negligible.  No tensor cores: 2 flop per 4 bytes.
//
// Numerics.  Float32/Float64 products are accumulated in fp64 (the f32 x f32 product is exact in fp64), each output rounded once
// at the end; Int32/Int64 wrap like Julia's machine integers (order-independent).  The reference calls BLAS gemv for floats, whose
// summation order is unspecified, so the float contract is the north-star tolerance (1e-6 rel), not bit equality.
// Determinism: the split of the reduction over CTAs depends only on (m, n, dtype); partials are combined in split order.
//
//   trans = 0 (r = A x, reduce over columns):  a thread owns VEC consecutive rows and sweeps columns; a CTA is RT row-vectors x CL
//       column lanes (RT * CL = 256); the column range is split over gridDim.y.  Column lanes are folded through shared memory in
//       lane order, splits by gemv_finish.
//   trans = 1 (r = A' x, reduce down each contiguous column):  LI lanes run down a column (16-B loads), a thread carries COLS
//       adjacent columns so x is loaded once per COLS column elements; the row range is split over gridDim.y.
//   Columns that do not start on 16-byte boundaries (leading dimension not a multiple of 16 bytes): the *_phase kernels deal the
//       columns into VEC classes of equal phase and keep the 16-byte loads; A x takes that kernel for aligned chunks as well.
#include "dab_common.cuh"

namespace {

constexpr int GV_THREADS = 256;

template <typename T> struct GvAcc { using type = T; };
template <> struct GvAcc<float> { using type = double; };
template <> struct GvAcc<int32_t> { using type = uint32_t; };   // wrap-around without signed-overflow UB
template <> struct GvAcc<int64_t> { using type = uint64_t; };

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) GvVec { T v[VEC]; };

// acc += a * b.  fp64: one DFMA (for Float32 inputs the product is exact in fp64, so fused and unfused agree bit for bit)
__device__ __forceinline__ void gv_mac(double& acc, double a, double b) { acc = __fma_rn(a, b, acc); }
__device__ __forceinline__ void gv_mac(uint32_t& acc, uint32_t a, uint32_t b) { acc += a * b; }
__device__ __forceinline__ void gv_mac(uint64_t& acc, uint64_t a, uint64_t b) { acc += a * b; }

template <typename T, int VEC>
__device__ __forceinline__ GvVec<T, VEC> gv_load_stream(const T* p) {
    GvVec<T, VEC> r;
    if constexpr (sizeof(T) * VEC == 16) {
        int4 t = __ldcs(reinterpret_cast<const int4*>(p));
        memcpy(&r, &t, 16);
    } else {
        static_assert(VEC == 1, "vector width");
        r.v[0] = __ldcs(p);
    }
    return r;
}
template <typename T, int VEC>
__device__ __forceinline__ GvVec<T, VEC> gv_load_cached(const T* p) {
    GvVec<T, VEC> r;
    if constexpr (sizeof(T) * VEC == 16) {
        int4 t = __ldg(reinterpret_cast<const int4*>(p));
        memcpy(&r, &t, 16);
    } else {
        r.v[0] = __ldg(p);
    }
    return r;
}

// ---- r = A x ----------------------------------------------------------------------------------------------------------------
// grid (row tiles, column splits); lrt = log2(RT).  A thread owns R groups of VEC consecutive rows, RT*VEC rows apart, so a CTA covers
// R*RT*VEC CONSECUTIVE rows of every column it touches.
// Loads in flight per thread: U = 4 columns x R = 1 row group, for 16-byte and unit-wise loads (leading dimension not a multiple of 16
// bytes) alike.  For the unit-wise loads (U, R) = (4, 1) gave a steady rate in the design sweep; more loads in flight -- (8, 1), (16, 1),
// (4, 2), (2, 4), (4, 4) -- swung widely with the column stride.
constexpr int GV_N_U = 4, GV_N_R = 1;
template <typename T, int VEC>
__global__ void __launch_bounds__(GV_THREADS) gemv_n_kernel(const T* __restrict__ A, size_t m, size_t n, const T* __restrict__ x, int lrt,
                                                            size_t cols_per_split, typename GvAcc<T>::type* __restrict__ part,
                                                            T* __restrict__ y) {
    using Acc = typename GvAcc<T>::type;
    constexpr int U = GV_N_U, R = GV_N_R;
    __shared__ Acc sh[GV_THREADS * VEC * R];
    const int RT = 1 << lrt, CL = GV_THREADS >> lrt;
    const int ri = threadIdx.x & (RT - 1), cl = threadIdx.x >> lrt;
    const size_t rstep = (size_t)RT * VEC;                              // rows between a thread's groups
    const size_t row0 = (size_t)blockIdx.x * R * rstep + (size_t)ri * VEC;
    const size_t jlo = (size_t)blockIdx.y * cols_per_split;
    const size_t jhi = (jlo + cols_per_split < n) ? jlo + cols_per_split : n;
    Acc acc[R][VEC];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[r][v] = Acc(0);
    if (row0 < m) {
        const T* col = A + row0;
        // all R groups of this thread inside the matrix: the common case; the last row tile takes the guarded path
        const bool full = row0 + (size_t)(R - 1) * rstep + VEC <= m;
        size_t j = jlo + cl;
        const size_t step = (size_t)CL;
        if (full) {
            for (; j + (U - 1) * step < jhi; j += U * step) {
                GvVec<T, VEC> a[U][R];
                T xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
#pragma unroll
                    for (int r = 0; r < R; ++r) a[u][r] = gv_load_stream<T, VEC>(col + (j + u * step) * m + r * rstep);
                    xv[u] = __ldg(x + j + u * step);
                }
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int v = 0; v < VEC; ++v) gv_mac(acc[r][v], (Acc)a[u][r].v[v], (Acc)xv[u]);
            }
        }
        for (; j < jhi; j += step) {
            const Acc xj = (Acc)__ldg(x + j);
#pragma unroll
            for (int r = 0; r < R; ++r)
                if (row0 + (size_t)r * rstep < m) {
                    GvVec<T, VEC> a = gv_load_stream<T, VEC>(col + j * m + r * rstep);
#pragma unroll
                    for (int v = 0; v < VEC; ++v) gv_mac(acc[r][v], (Acc)a.v[v], xj);
                }
        }
    }
    if (CL > 1) {  // fold the column lanes in lane order
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int v = 0; v < VEC; ++v) sh[(threadIdx.x * R + r) * VEC + v] = acc[r][v];
        __syncthreads();
        if (cl == 0)
            for (int c = 1; c < CL; ++c)
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) acc[r][v] += sh[((((c << lrt) + ri)) * R + r) * VEC + v];
    }
    if (cl == 0) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const size_t row = row0 + (size_t)r * rstep;
            if (row < m) {
                if (part) {
#pragma unroll
                    for (int v = 0; v < VEC; ++v) part[(size_t)blockIdx.y * m + row + v] = acc[r][v];
                } else {
#pragma unroll
                    for (int v = 0; v < VEC; ++v) y[row + v] = (T)acc[r][v];
                }
            }
        }
    }
}

// ---- r = A x, columns NOT 16-byte aligned ------------------------------------------------------------------------------------------
// The leading dimension is not a multiple of VEC (the 37/36-row splits defaultdist produces), so column j starts phase(j) =
// (a0 + j*m) mod VEC elements past a 16-byte boundary.  Columns j and j + VEC share their phase, so the columns are dealt into VEC
// classes (blockIdx.y % VEC) and a CTA sweeps one class with a column stride of VEC: inside a class every thread's 16-byte word sits at
// the same offset in every column, i.e. the thread owns rows 4t - p .. 4t - p + 3 for the class's phase p and runs the aligned kernel's
// loop unchanged.  The two threads per column whose word straddles a column boundary (rows < 0 or >= m belong to the neighbouring
// columns) mask those elements.  Aligned chunks take the same kernel (every phase is 0, no warp is masked).  Each class writes its own partial vector; gemv_finish adds the classes and the splits in index order.
template <typename T, int VEC, int U>
__global__ void __launch_bounds__(GV_THREADS, 4) gemv_n_phase_kernel(const T* __restrict__ A, size_t m, size_t n, const T* __restrict__ x, int lrt,
                                                                  size_t cols_per_split, int a0, typename GvAcc<T>::type* __restrict__ part) {
    using Acc = typename GvAcc<T>::type;
    __shared__ Acc sh[GV_THREADS * VEC];
    const int RT = 1 << lrt, CL = GV_THREADS >> lrt;
    const int ri = threadIdx.x & (RT - 1), cl = threadIdx.x >> lrt;
    const int klass = blockIdx.y % VEC;
    const size_t split = blockIdx.y / VEC;
    const int p = (int)(((size_t)a0 + (size_t)klass * (m % VEC)) % VEC);
    const size_t nk = n > (size_t)klass ? (n - klass + VEC - 1) / VEC : 0;   // columns of this class
    const size_t jlo = split * cols_per_split;
    const size_t jhi = (jlo + cols_per_split < nk) ? jlo + cols_per_split : nk;
    const long long rowbase = (long long)((size_t)blockIdx.x * RT * VEC + (size_t)ri * VEC) - p;
    Acc acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = Acc(0);
    // A thread whose word straddles a column boundary must mask the elements of the neighbouring column.  The choice between the plain
    // and the masked loop is made per WARP (a lane taking its own loop would double the warp's time, and with one wave of CTAs the
    // slowest warp is the kernel's time); the masked loop issues the same 16-byte loads.
    const bool active = rowbase < (long long)m;
    const bool interior = rowbase >= 0 && rowbase + VEC <= (long long)m;
    const bool plain = __all_sync(0xffffffffu, interior || !active);
    if (active) {
        const T* base = A + rowbase + (long long)klass * (long long)m;   // the thread's word in the class's first column
        const size_t cstride = (size_t)VEC * m;                          // elements between two columns of a class
        const T* xk = x + klass;
        size_t j = jlo + cl;
        const size_t step = (size_t)CL;
        if (plain) {
            for (; j + (U - 1) * step < jhi; j += U * step) {
                GvVec<T, VEC> a[U];
                T xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    a[u] = gv_load_stream<T, VEC>(base + (j + u * step) * cstride);
                    xv[u] = __ldg(xk + (j + u * step) * VEC);
                }
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) gv_mac(acc[v], (Acc)a[u].v[v], (Acc)xv[u]);
            }
            for (; j < jhi; j += step) {
                const GvVec<T, VEC> a = gv_load_stream<T, VEC>(base + j * cstride);
                const Acc xj = (Acc)__ldg(xk + j * VEC);
#pragma unroll
                for (int v = 0; v < VEC; ++v) gv_mac(acc[v], (Acc)a.v[v], xj);
            }
        } else {
            bool ok[VEC];
#pragma unroll
            for (int v = 0; v < VEC; ++v) ok[v] = rowbase + v >= 0 && rowbase + v < (long long)m;
            // The only words that reach outside the matrix are the head of column 0 and the tail of column n-1: the lane that meets
            // one of them takes it element-wise BEFORE the sweep, so that the sweep itself stays branch-free (same loads in flight as
            // the plain loop).
            size_t jend = jhi;
            if (j < jhi) {
                const Acc zero = Acc(0);
                if (rowbase < 0 && klass == 0 && j == 0) {                                       // column 0 is this lane's first
#pragma unroll
                    for (int v = 0; v < VEC; ++v) gv_mac(acc[v], ok[v] ? (Acc)__ldcs(base + v) : zero, (Acc)__ldg(xk));
                    j += step;
                }
                const size_t jl = nk - 1;                                                        // class index of column n-1, if ours
                if (rowbase + VEC > (long long)m && (size_t)klass == (n - 1) % VEC && jhi == nk && jl >= j && (jl - j) % step == 0) {
#pragma unroll
                    for (int v = 0; v < VEC; ++v)
                        gv_mac(acc[v], ok[v] ? (Acc)__ldcs(base + jl * cstride + v) : zero, (Acc)__ldg(xk + jl * VEC));
                    jend = jl;                                                                   // the lane's sweep stops before it
                }
            }
            for (; j + (U - 1) * step < jend; j += U * step) {
                GvVec<T, VEC> a[U];
                T xv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    a[u] = gv_load_stream<T, VEC>(base + (j + u * step) * cstride);
                    xv[u] = __ldg(xk + (j + u * step) * VEC);
                }
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) gv_mac(acc[v], ok[v] ? (Acc)a[u].v[v] : Acc(0), (Acc)xv[u]);
            }
            for (; j < jend; j += step) {
                const GvVec<T, VEC> a = gv_load_stream<T, VEC>(base + j * cstride);
                const Acc xj = (Acc)__ldg(xk + j * VEC);
#pragma unroll
                for (int v = 0; v < VEC; ++v) gv_mac(acc[v], ok[v] ? (Acc)a.v[v] : Acc(0), xj);
            }
        }
    }
    if (CL > 1) {  // fold the column lanes in lane order
#pragma unroll
        for (int v = 0; v < VEC; ++v) sh[threadIdx.x * VEC + v] = acc[v];
        __syncthreads();
        if (cl == 0)
            for (int c = 1; c < CL; ++c)
#pragma unroll
                for (int v = 0; v < VEC; ++v) acc[v] += sh[((c << lrt) + ri) * VEC + v];
    }
    if (cl == 0) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            const long long row = rowbase + v;
            if (row >= 0 && row < (long long)m) part[(size_t)blockIdx.y * m + (size_t)row] = acc[v];
        }
    }
}

// ---- r = A' x ---------------------------------------------------------------------------------------------------------------
// grid (column tiles, row splits); lli = log2(LI); a CTA covers G consecutive groups of (256 / LI) * COLS columns
template <typename T, int VEC, int COLS>
__global__ void __launch_bounds__(GV_THREADS) gemv_t_kernel(const T* __restrict__ A, size_t m, size_t n, const T* __restrict__ x, int lli,
                                                            int G, size_t rows_per_split, typename GvAcc<T>::type* __restrict__ part,
                                                            T* __restrict__ y) {
    using Acc = typename GvAcc<T>::type;
    __shared__ Acc sh[(GV_THREADS / 32) * COLS];
    const int LI = 1 << lli, CB = GV_THREADS >> lli;
    const int li = threadIdx.x & (LI - 1), cb = threadIdx.x >> lli;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t ilo = (size_t)blockIdx.y * rows_per_split;
    const size_t ihi = (ilo + rows_per_split < m) ? ilo + rows_per_split : m;
    const size_t step = (size_t)LI * VEC;
    for (int g = 0; g < G; ++g) {
        const size_t col0 = (((size_t)blockIdx.x * G + g) * CB + cb) * COLS;
        Acc acc[COLS];
#pragma unroll
        for (int c = 0; c < COLS; ++c) acc[c] = Acc(0);
        if (col0 < n) {
            const int nc = (n - col0 < (size_t)COLS) ? (int)(n - col0) : COLS;
            // UI sweep steps per batch: the unit-wise (unaligned) variant needs the extra loads in flight
            constexpr int UI = (VEC == 1) ? 32 / (int)sizeof(T) : 1;
            size_t i = ilo + (size_t)li * VEC;
            if (nc == COLS) {
                const T* p0 = A + col0 * m;
                for (; i + (UI - 1) * step < ihi; i += UI * step) {
                    GvVec<T, VEC> a[UI][COLS], xv[UI];
#pragma unroll
                    for (int u = 0; u < UI; ++u) {
#pragma unroll
                        for (int c = 0; c < COLS; ++c) a[u][c] = gv_load_stream<T, VEC>(p0 + c * m + i + u * step);
                        xv[u] = gv_load_cached<T, VEC>(x + i + u * step);
                    }
#pragma unroll
                    for (int u = 0; u < UI; ++u)
#pragma unroll
                        for (int c = 0; c < COLS; ++c)
#pragma unroll
                            for (int v = 0; v < VEC; ++v) gv_mac(acc[c], (Acc)a[u][c].v[v], (Acc)xv[u].v[v]);
                }
            }
            for (; i < ihi; i += step) {  // sweep tail, and the last (partial) column group
                const GvVec<T, VEC> xv = gv_load_cached<T, VEC>(x + i);
#pragma unroll
                for (int c = 0; c < COLS; ++c)
                    if (c < nc) {
                        GvVec<T, VEC> a = gv_load_stream<T, VEC>(A + (col0 + c) * m + i);
#pragma unroll
                        for (int v = 0; v < VEC; ++v) gv_mac(acc[c], (Acc)a.v[v], (Acc)xv.v[v]);
                    }
            }
        }
        // fold the LI lanes of each column group: fixed shuffle tree inside a warp (a group never straddles warps unless it is a
        // whole number of them), then the group's warps in warp order through shared memory
        const int W = LI < 32 ? LI : 32;
        for (int s = W >> 1; s > 0; s >>= 1)
#pragma unroll
            for (int c = 0; c < COLS; ++c) acc[c] += __shfl_down_sync(0xffffffffu, acc[c], s, W);
        if (LI > 32) {
            if (lane == 0)
#pragma unroll
                for (int c = 0; c < COLS; ++c) sh[warp * COLS + c] = acc[c];
            __syncthreads();
            if (li == 0) {
                const int nw = LI >> 5;
                for (int w = 1; w < nw; ++w)
#pragma unroll
                    for (int c = 0; c < COLS; ++c) acc[c] += sh[(warp + w) * COLS + c];
            }
            __syncthreads();
        }
        if (li == 0 && col0 < n) {
#pragma unroll
            for (int c = 0; c < COLS; ++c)
                if (col0 + c < n) {
                    if (part) part[(size_t)blockIdx.y * n + col0 + c] = acc[c];
                    else y[col0 + c] = (T)acc[c];
                }
        }
    }
}

// ---- r = A' x, columns NOT 16-byte aligned -----------------------------------------------------------------------------------------
// Same dealing of the columns into VEC phase classes as gemv_n_phase_kernel: a thread carries COLS columns of ONE class (klass, klass +
// VEC, ...), so the first 16-byte boundary lies `head` = (VEC - phase) % VEC rows below the top of every one of them.  The sweep runs over
// the words that lie entirely inside the column (16-byte loads; the matching x elements start at x + head, which is in general not
// 16-byte aligned: element-wise cached loads, or one 16-byte load when it happens to be); the <= VEC-1 rows above the first and below
// the last full word are added element-wise by two lanes of the first row split.  No load ever leaves the column.
template <typename T, int VEC, int COLS>
__global__ void __launch_bounds__(GV_THREADS) gemv_t_phase_kernel(const T* __restrict__ A, size_t m, size_t n, const T* __restrict__ x, int lli,
                                                                  int G, size_t words_per_split, int a0,
                                                                  typename GvAcc<T>::type* __restrict__ part, T* __restrict__ y) {
    using Acc = typename GvAcc<T>::type;
    __shared__ Acc sh[(GV_THREADS / 32) * COLS];
    const int LI = 1 << lli, CB = GV_THREADS >> lli;
    const int li = threadIdx.x & (LI - 1), cb = threadIdx.x >> lli;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int klass = blockIdx.x % VEC;
    const size_t gblock = blockIdx.x / VEC;
    const int p = (int)(((size_t)a0 + (size_t)klass * (m % VEC)) % VEC);
    const size_t head = (size_t)((VEC - p) % VEC);
    const size_t nfull = (m - head) / VEC;                                   // whole 16-byte words inside a column of this class
    const size_t tail0 = head + nfull * VEC;                                 // first row below the last full word
    const size_t nk = n > (size_t)klass ? (n - klass + VEC - 1) / VEC : 0;   // columns of this class
    const size_t wlo = (size_t)blockIdx.y * words_per_split;
    const size_t whi = (wlo + words_per_split < nfull) ? wlo + words_per_split : nfull;
    const size_t cstride = (size_t)VEC * m;                                  // elements between two columns of a class
    const T* xh = x + head;
    const bool xal = ((uintptr_t)xh % (sizeof(T) * VEC)) == 0;
    for (int g = 0; g < G; ++g) {
        const size_t jj0 = ((gblock * G + g) * CB + cb) * COLS;              // class index of the thread's first column
        Acc acc[COLS];
#pragma unroll
        for (int c = 0; c < COLS; ++c) acc[c] = Acc(0);
        if (jj0 < nk) {
            const int nc = (nk - jj0 < (size_t)COLS) ? (int)(nk - jj0) : COLS;
            const T* c0 = A + ((size_t)klass + (size_t)VEC * jj0) * m;      // top of the first column
            const T* p0 = c0 + head;                                         // its first full word (16-byte aligned)
            size_t w = wlo + li;
            if (nc == COLS) {
                for (; w < whi; w += LI) {
                    GvVec<T, VEC> a[COLS], xv;
#pragma unroll
                    for (int c = 0; c < COLS; ++c) a[c] = gv_load_stream<T, VEC>(p0 + c * cstride + w * VEC);
                    if (xal) xv = gv_load_cached<T, VEC>(xh + w * VEC);
                    else {
#pragma unroll
                        for (int v = 0; v < VEC; ++v) xv.v[v] = __ldg(xh + w * VEC + v);
                    }
#pragma unroll
                    for (int c = 0; c < COLS; ++c)
#pragma unroll
                        for (int v = 0; v < VEC; ++v) gv_mac(acc[c], (Acc)a[c].v[v], (Acc)xv.v[v]);
                }
            } else {
                for (; w < whi; w += LI) {
#pragma unroll
                    for (int c = 0; c < COLS; ++c)
                        if (c < nc) {
                            const GvVec<T, VEC> a = gv_load_stream<T, VEC>(p0 + c * cstride + w * VEC);
#pragma unroll
                            for (int v = 0; v < VEC; ++v) gv_mac(acc[c], (Acc)a.v[v], (Acc)__ldg(xh + w * VEC + v));
                        }
                }
            }
            if (blockIdx.y == 0) {  // the rows outside the full words: lane 0 the head, the next lane the tail
                if (li == 0)
                    for (size_t i = 0; i < head; ++i) {
                        const Acc xi = (Acc)__ldg(x + i);
#pragma unroll
                        for (int c = 0; c < COLS; ++c)
                            if (c < nc) gv_mac(acc[c], (Acc)__ldcs(c0 + c * cstride + i), xi);
                    }
                if (li == (LI > 1 ? 1 : 0))
                    for (size_t i = tail0; i < m; ++i) {
                        const Acc xi = (Acc)__ldg(x + i);
#pragma unroll
                        for (int c = 0; c < COLS; ++c)
                            if (c < nc) gv_mac(acc[c], (Acc)__ldcs(c0 + c * cstride + i), xi);
                    }
            }
        }
        // fold the LI lanes of each column group (same tree as gemv_t_kernel)
        const int W = LI < 32 ? LI : 32;
        for (int s = W >> 1; s > 0; s >>= 1)
#pragma unroll
            for (int c = 0; c < COLS; ++c) acc[c] += __shfl_down_sync(0xffffffffu, acc[c], s, W);
        if (LI > 32) {
            if (lane == 0)
#pragma unroll
                for (int c = 0; c < COLS; ++c) sh[warp * COLS + c] = acc[c];
            __syncthreads();
            if (li == 0) {
                const int nw = LI >> 5;
                for (int w2 = 1; w2 < nw; ++w2)
#pragma unroll
                    for (int c = 0; c < COLS; ++c) acc[c] += sh[(warp + w2) * COLS + c];
            }
            __syncthreads();
        }
        if (li == 0 && jj0 < nk) {
#pragma unroll
            for (int c = 0; c < COLS; ++c)
                if (jj0 + c < nk) {
                    const size_t j = (size_t)klass + (size_t)VEC * (jj0 + c);
                    if (part) part[(size_t)blockIdx.y * n + j] = acc[c];
                    else y[j] = (T)acc[c];
                }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(GV_THREADS) gemv_finish_kernel(const typename GvAcc<T>::type* __restrict__ part, size_t nout, int nsplit,
                                                                 T* __restrict__ y) {
    using Acc = typename GvAcc<T>::type;
    const size_t k = (size_t)blockIdx.x * GV_THREADS + threadIdx.x;
    if (k >= nout) return;
    Acc acc = part[k];
#pragma unroll 8
    for (int s = 1; s < nsplit; ++s) acc += part[(size_t)s * nout + k];   // split order; unrolled so that the loads overlap
    y[k] = (T)acc;
}

int ceil_log2(size_t v) {
    int l = 0;
    while (((size_t)1 << l) < v) ++l;
    return l;
}

template <typename T, int VEC>
int32_t launch_n(dab_ctx* ctx, const T* A, size_t m, size_t n, const T* x, T* y) {
    using Acc = typename GvAcc<T>::type;
    constexpr int U = GV_N_U, R = GV_N_R;
    const size_t rvecs = (m + (size_t)VEC * R - 1) / ((size_t)VEC * R);   // row groups-of-R
    int lrt = ceil_log2(rvecs);
    if (lrt > 8) lrt = 8;
    const int RT = 1 << lrt, CL = GV_THREADS >> lrt;
    const size_t gx = (rvecs + RT - 1) / RT;
    // one full wave of resident CTAs (no partial second wave), but every CTA keeps >= 16 column steps per lane
    const size_t slots = (size_t)ctx->sm_count * (size_t)dab_resident_ctas((const void*)gemv_n_kernel<T, VEC>, GV_THREADS);
    const size_t want = slots / gx > 0 ? slots / gx : 1;
    size_t max_split = n / ((size_t)CL * U * 4);
    if (max_split < 1) max_split = 1;
    size_t nsplit = want < max_split ? want : max_split;
    if (nsplit > 65535) nsplit = 65535;
    size_t cps = (n + nsplit - 1) / nsplit;
    nsplit = (n + cps - 1) / cps;
    Acc* part = nullptr;
    if (nsplit > 1) {
        int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, nsplit * m * sizeof(Acc), false);
        if (st != DAB_OK) return st;
        part = (Acc*)ctx->dim_scratch;
    }
    DAB_REQUIRE(ctx, gx <= 0x7fffffffull, DAB_ERR_ARG, "dab_gemv: too many row tiles");
    dim3 grid((unsigned)gx, (unsigned)nsplit);
    gemv_n_kernel<T, VEC><<<grid, GV_THREADS, 0, ctx->stream>>>(A, m, n, x, lrt, cps, part, y);
    DAB_LAUNCHED(ctx);
    if (part) {
        gemv_finish_kernel<T><<<(unsigned)((m + GV_THREADS - 1) / GV_THREADS), GV_THREADS, 0, ctx->stream>>>(part, m, (int)nsplit, y);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

// the phase-class variant (columns not 16-byte aligned): VEC classes x nsplit column splits in gridDim.y, always through the partials
template <typename T, int VEC>
int32_t launch_n_phase(dab_ctx* ctx, const T* A, size_t m, size_t n, const T* x, T* y) {
    using Acc = typename GvAcc<T>::type;
    constexpr int U = 4;
    const size_t rvecs = (m + 2 * (VEC - 1)) / VEC;   // words a column can touch at the worst phase
    int lrt = ceil_log2(rvecs);
    if (lrt > 8) lrt = 8;
    const int RT = 1 << lrt, CL = GV_THREADS >> lrt;
    const size_t gx = (rvecs + RT - 1) / RT;
    const size_t slots = (size_t)ctx->sm_count * (size_t)dab_resident_ctas((const void*)gemv_n_phase_kernel<T, VEC, U>, GV_THREADS);
    // four waves of CTAs rather than one: the CTAs holding a masked warp run a little longer and a single wave would wait for them
    // (tools/sweep_gemv.cu sweeps it); the partial vectors stay below 1/32 of the matrix bytes
    size_t want = 4 * slots / (gx * VEC);
    if (want > n / (32 * VEC * (sizeof(Acc) / sizeof(T)))) want = n / (32 * VEC * (sizeof(Acc) / sizeof(T)));
    if (want < 1) want = 1;
    const size_t nk = (n + VEC - 1) / VEC;            // columns of the largest class
    size_t max_split = nk / ((size_t)CL * U * 4);
    if (max_split < 1) max_split = 1;
    size_t nsplit = want < max_split ? want : max_split;
    if (nsplit * VEC > 65535) nsplit = 65535 / VEC;
    size_t cps = (nk + nsplit - 1) / nsplit;
    nsplit = (nk + cps - 1) / cps;
    const size_t ny = nsplit * VEC;
    int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, ny * m * sizeof(Acc), false);
    if (st != DAB_OK) return st;
    Acc* part = (Acc*)ctx->dim_scratch;
    DAB_REQUIRE(ctx, gx <= 0x7fffffffull, DAB_ERR_ARG, "dab_gemv: too many row tiles");
    const int a0 = (int)(((uintptr_t)A / sizeof(T)) % VEC);
    dim3 grid((unsigned)gx, (unsigned)ny);
    gemv_n_phase_kernel<T, VEC, U><<<grid, GV_THREADS, 0, ctx->stream>>>(A, m, n, x, lrt, cps, a0, part);
    DAB_LAUNCHED(ctx);
    gemv_finish_kernel<T><<<(unsigned)((m + GV_THREADS - 1) / GV_THREADS), GV_THREADS, 0, ctx->stream>>>(part, m, (int)ny, y);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

template <typename T, int VEC, int COLS>
int32_t launch_t(dab_ctx* ctx, const T* A, size_t m, size_t n, const T* x, T* y) {
    using Acc = typename GvAcc<T>::type;
    const size_t rvecs = (m + VEC - 1) / VEC;
    int lli = ceil_log2(rvecs);
    if (lli > 8) lli = 8;
    const int LI = 1 << lli, CB = GV_THREADS >> lli;
    // short columns: a CTA walks G consecutive column groups so that it still moves >= 64 KiB
    const size_t group_bytes = (size_t)CB * COLS * m * sizeof(T);
    size_t Gs = group_bytes ? (65536 + group_bytes - 1) / group_bytes : 1;
    if (Gs > 16) Gs = 16;
    if (Gs < 1) Gs = 1;
    const int G = (int)Gs;
    const size_t cols_per_cta = (size_t)CB * COLS * G;
    const size_t gx = (n + cols_per_cta - 1) / cols_per_cta;
    const size_t slots = (size_t)ctx->sm_count * (size_t)dab_resident_ctas((const void*)gemv_t_kernel<T, VEC, COLS>, GV_THREADS);
    const size_t waves = n >= 64 ? 4 : 1;
    const size_t want = waves * slots / gx > 0 ? waves * slots / gx : 1;
    const size_t unit = (size_t)LI * VEC;  // rows one sweep step covers; splits start on a multiple of it (keeps 16-B alignment)
    size_t max_split = m / (unit * 16);
    if (max_split < 1) max_split = 1;
    size_t nsplit = want < max_split ? want : max_split;
    if (nsplit > 65535) nsplit = 65535;
    size_t rps = (m + nsplit - 1) / nsplit;
    rps = (rps + unit - 1) / unit * unit;
    nsplit = (m + rps - 1) / rps;
    Acc* part = nullptr;
    if (nsplit > 1) {
        int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, nsplit * n * sizeof(Acc), false);
        if (st != DAB_OK) return st;
        part = (Acc*)ctx->dim_scratch;
    }
    DAB_REQUIRE(ctx, gx <= 0x7fffffffull, DAB_ERR_ARG, "dab_gemv: too many column tiles");
    dim3 grid((unsigned)gx, (unsigned)nsplit);
    gemv_t_kernel<T, VEC, COLS><<<grid, GV_THREADS, 0, ctx->stream>>>(A, m, n, x, lli, G, rps, part, y);
    DAB_LAUNCHED(ctx);
    if (part) {
        gemv_finish_kernel<T><<<(unsigned)((n + GV_THREADS - 1) / GV_THREADS), GV_THREADS, 0, ctx->stream>>>(part, n, (int)nsplit, y);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

// the phase-class variant of A' x (columns not 16-byte aligned)
template <typename T, int VEC, int COLS>
int32_t launch_t_phase(dab_ctx* ctx, const T* A, size_t m, size_t n, const T* x, T* y) {
    using Acc = typename GvAcc<T>::type;
    const size_t words = m / VEC;                                  // full words of a column at phase 0 (an upper bound for the others)
    int lli = ceil_log2(words);
    if (lli > 8) lli = 8;
    const int LI = 1 << lli, CB = GV_THREADS >> lli;
    const size_t group_bytes = (size_t)CB * COLS * m * sizeof(T);
    size_t Gs = group_bytes ? (65536 + group_bytes - 1) / group_bytes : 1;
    if (Gs > 16) Gs = 16;
    if (Gs < 1) Gs = 1;
    const int G = (int)Gs;
    const size_t nk = (n + VEC - 1) / VEC;                         // columns of the largest class
    const size_t cols_per_cta = (size_t)CB * COLS * G;
    const size_t gx = ((nk + cols_per_cta - 1) / cols_per_cta) * VEC;
    const size_t slots = (size_t)ctx->sm_count * (size_t)dab_resident_ctas((const void*)gemv_t_phase_kernel<T, VEC, COLS>, GV_THREADS);
    const size_t waves = 4;
    const size_t want = waves * slots / gx > 0 ? waves * slots / gx : 1;
    size_t max_split = words / ((size_t)LI * 16);
    if (max_split < 1) max_split = 1;
    size_t nsplit = want < max_split ? want : max_split;
    if (nsplit > 65535) nsplit = 65535;
    size_t wps = (words + nsplit - 1) / nsplit;
    wps = (wps + LI - 1) / LI * LI;
    nsplit = (words + wps - 1) / wps;
    Acc* part = nullptr;
    if (nsplit > 1) {
        int32_t st = dab_scratch_grow(ctx, &ctx->dim_scratch, &ctx->dim_scratch_bytes, nsplit * n * sizeof(Acc), false);
        if (st != DAB_OK) return st;
        part = (Acc*)ctx->dim_scratch;
    }
    DAB_REQUIRE(ctx, gx <= 0x7fffffffull, DAB_ERR_ARG, "dab_gemv: too many column tiles");
    const int a0 = (int)(((uintptr_t)A / sizeof(T)) % VEC);
    dim3 grid((unsigned)gx, (unsigned)nsplit);
    gemv_t_phase_kernel<T, VEC, COLS><<<grid, GV_THREADS, 0, ctx->stream>>>(A, m, n, x, lli, G, wps, a0, part, y);
    DAB_LAUNCHED(ctx);
    if (part) {
        gemv_finish_kernel<T><<<(unsigned)((n + GV_THREADS - 1) / GV_THREADS), GV_THREADS, 0, ctx->stream>>>(part, n, (int)nsplit, y);
        DAB_LAUNCHED(ctx);
    }
    return DAB_OK;
}

template <typename T>
__global__ void gv_zero_kernel(T* y, size_t n) {
    const size_t k = (size_t)blockIdx.x * GV_THREADS + threadIdx.x;
    if (k < n) y[k] = T(0);
}

template <typename T>
int32_t gemv_t(dab_ctx* ctx, int32_t trans, const T* A, size_t m, size_t n, const T* x, T* y) {
    constexpr int VEC = 16 / sizeof(T);
    const size_t nout = trans ? n : m, nred = trans ? m : n;
    if (nout == 0) return DAB_OK;
    if (nred == 0) {  // empty sum: zeros(T, nout), as Base's generic and BLAS matvec both give
        gv_zero_kernel<T><<<(unsigned)((nout + GV_THREADS - 1) / GV_THREADS), GV_THREADS, 0, ctx->stream>>>(y, nout);
        DAB_LAUNCHED(ctx);
        return DAB_OK;
    }
    // 16-byte loads need every column start 16-byte aligned: base aligned and m a multiple of VEC (x too for the A' x sweep)
    const bool vec = ((uintptr_t)A % 16 == 0) && (m % VEC == 0) && (!trans || (uintptr_t)x % 16 == 0);
    if (!trans) {
        // The phase-class kernel serves every chunk big enough to matter: 16-byte loads whatever the alignment of the columns, and
        // four waves of CTAs (faster than the single-wave kernel on aligned chunks and than unit-wise loads on misaligned ones when it
        // was designed).
        // Where it pays: the VEC class partials cost 2*VEC*m carriers of traffic (16/n of the Float32 matrix bytes) and a short column
        // leaves row lanes idle -- an aligned chunk switches kernels only when that is below 2 % (measured 4194304 x 128: 5.8 vs 6.4
        // TB/s, 128 x 4194304: 3.0 vs 5.4), a misaligned one as soon as it beats the unit-wise loads' -35 %.
        const bool phase_ok = (uintptr_t)A % sizeof(T) == 0;
        if (phase_ok && (vec ? (m >= 4096 && n >= 1024) : (m >= 256 && n >= 64))) return launch_n_phase<T, VEC>(ctx, A, m, n, x, y);
        if (vec) return launch_n<T, VEC>(ctx, A, m, n, x, y);
        return launch_n<T, 1>(ctx, A, m, n, x, y);
    }
    // columns a thread carries (x is loaded once per COLS column elements): 8 with 16-byte loads (faster than 4 on a large Float32
    // chunk when it was designed)
    if (vec && n >= 64) return launch_t<T, VEC, 8>(ctx, A, m, n, x, y);
    // misaligned columns: the phase-class kernel keeps the 16-byte loads
    if (!vec && (uintptr_t)A % sizeof(T) == 0 && (uintptr_t)x % sizeof(T) == 0 && m >= 256 && n >= 64)
        return launch_t_phase<T, VEC, 4>(ctx, A, m, n, x, y);   // 4 columns per thread: 8 cost 128 registers here (6.4-6.8 vs 5.4-6.1 TB/s)
    return vec ? launch_t<T, VEC, 4>(ctx, A, m, n, x, y) : launch_t<T, 1, 4>(ctx, A, m, n, x, y);
}

}  // namespace

extern "C" int32_t dab_gemv(dab_ctx* ctx, int32_t dtype, int32_t trans, const void* A, size_t m, size_t n, const void* x, void* r) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, trans == 0 || trans == 1, DAB_ERR_ARG, "dab_gemv: trans %d", trans);
    DAB_REQUIRE(ctx, (A || m * n == 0) && (x || (trans ? m : n) == 0) && (r || (trans ? n : m) == 0), DAB_ERR_ARG, "dab_gemv: null pointer");
    switch (dtype) {
        case DAB_F32: return gemv_t<float>(ctx, trans, (const float*)A, m, n, (const float*)x, (float*)r);
        case DAB_F64: return gemv_t<double>(ctx, trans, (const double*)A, m, n, (const double*)x, (double*)r);
        case DAB_I32: return gemv_t<int32_t>(ctx, trans, (const int32_t*)A, m, n, (const int32_t*)x, (int32_t*)r);
        case DAB_I64: return gemv_t<int64_t>(ctx, trans, (const int64_t*)A, m, n, (const int64_t*)x, (int64_t*)r);
        default: return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_gemv: dtype %d", dtype);
    }
}

// ---- transpose of one box (K10) -----------------------------------------------------------------------------------------------
namespace {

// TR_TILE x TR_TILE element tile (64 for units up to 4 bytes, 32 above: static shared memory budget); 256 threads = TR_TILE x TY
template <typename U, int TR_TILE>
__global__ void __launch_bounds__(256) transpose_box_kernel(U* __restrict__ dst, size_t dst_ld, const U* __restrict__ src, size_t src_ld,
                                                            size_t rows, size_t cols, unsigned tiles_r) {
    // +1 padding: the transposed read walks a tile column, i.e. stride TR_TILE+1 words -> conflict-free for 4-byte units
    __shared__ U tile[TR_TILE][TR_TILE + 1];
    const size_t tr = blockIdx.x % tiles_r, tc = blockIdx.x / tiles_r;  // consecutive CTAs walk down the source rows (address order)
    const size_t r0 = tr * TR_TILE, c0 = tc * TR_TILE;
    constexpr int TY = 256 / TR_TILE;
    constexpr int NK = TR_TILE / TY;                       // tile rows a thread moves: all NK loads are issued before the first store
    const int tx = threadIdx.x & (TR_TILE - 1), ty = threadIdx.x / TR_TILE;
    U v[NK];
#pragma unroll
    for (int q = 0; q < NK; ++q) {
        const size_t r = r0 + tx, c = c0 + ty + q * TY;
        v[q] = (r < rows && c < cols) ? src[r + c * src_ld] : U{};
    }
#pragma unroll
    for (int q = 0; q < NK; ++q) tile[ty + q * TY][tx] = v[q];
    __syncthreads();
#pragma unroll 4
    for (int k = ty; k < TR_TILE; k += TY) {
        const size_t c = c0 + tx, r = r0 + k;  // dst is (cols x rows): element (c, r)
        if (r < rows && c < cols) dst[c + r * dst_ld] = tile[tx][k];
    }
}

// 4-byte units with everything 16-byte aligned: 16-byte global loads down the source rows and 16-byte global stores down the
// destination rows (4x fewer LSU instructions than the unit-wise kernel); the 64 x 64 tile is transposed through shared memory
// with scalar accesses (pitch 65 words: at most 2-way bank conflicts on either side).
__global__ void __launch_bounds__(256) transpose_box_vec4_kernel(uint32_t* __restrict__ dst, size_t dst_ld, const uint32_t* __restrict__ src,
                                                                 size_t src_ld, size_t rows, size_t cols, unsigned tiles_r) {
    __shared__ uint32_t tile[64][65];
    const size_t tr = blockIdx.x % tiles_r, tc = blockIdx.x / tiles_r;
    const size_t r0 = tr * 64, c0 = tc * 64;
    const int q = threadIdx.x & 15, k0 = threadIdx.x >> 4;
    uint4 v[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const size_t r = r0 + 4 * q, c = c0 + k0 + 16 * it;
        if (r < rows && c < cols) v[it] = __ldcs(reinterpret_cast<const uint4*>(src + r + c * src_ld));
    }
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int k = k0 + 16 * it;
        tile[k][4 * q + 0] = v[it].x;
        tile[k][4 * q + 1] = v[it].y;
        tile[k][4 * q + 2] = v[it].z;
        tile[k][4 * q + 3] = v[it].w;
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int k = k0 + 16 * it;                       // source row inside the tile = destination column
        const size_t c = c0 + 4 * q, r = r0 + k;
        if (r < rows && c < cols) {
            uint4 o;
            o.x = tile[4 * q + 0][k];
            o.y = tile[4 * q + 1][k];
            o.z = tile[4 * q + 2][k];
            o.w = tile[4 * q + 3][k];
            __stcs(reinterpret_cast<uint4*>(dst + c + r * dst_ld), o);
        }
    }
}

template <typename U>
int32_t launch_transpose(dab_ctx* ctx, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows, size_t cols) {
    constexpr int TR_TILE = sizeof(U) <= 4 ? 64 : 32;
    const size_t tiles_r = (rows + TR_TILE - 1) / TR_TILE, tiles_c = (cols + TR_TILE - 1) / TR_TILE;
    DAB_REQUIRE(ctx, tiles_r * tiles_c <= 0x7fffffffull && tiles_r <= 0xffffffffull, DAB_ERR_ARG, "dab_transpose_box: too many tiles");
    if constexpr (sizeof(U) == 4) {
        if (rows % 4 == 0 && cols % 4 == 0 && src_ld % 4 == 0 && dst_ld % 4 == 0 && (uintptr_t)src % 16 == 0 && (uintptr_t)dst % 16 == 0) {
            transpose_box_vec4_kernel<<<(unsigned)(tiles_r * tiles_c), 256, 0, ctx->stream>>>((uint32_t*)dst, dst_ld, (const uint32_t*)src,
                                                                                            src_ld, rows, cols, (unsigned)tiles_r);
            DAB_LAUNCHED(ctx);
            return DAB_OK;
        }
    }
    transpose_box_kernel<U, TR_TILE><<<(unsigned)(tiles_r * tiles_c), 256, 0, ctx->stream>>>((U*)dst, dst_ld, (const U*)src, src_ld, rows, cols,
                                                                                   (unsigned)tiles_r);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

// Julia's conj negates the imaginary part by flipping its sign bit, so a NaN keeps its payload; an arithmetic negation would give the
// canonical NaN on the GPU.
__device__ __forceinline__ float flip_sign(float x) { return __uint_as_float(__float_as_uint(x) ^ 0x80000000u); }
__device__ __forceinline__ double flip_sign(double x) { return __longlong_as_double(__double_as_longlong(x) ^ (long long)0x8000000000000000ull); }

// conj(transpose) of one box of Complex{T}: transpose_box_kernel's tile walk with 8- / 16-byte elements, the imaginary component's
// sign bit flipped between the shared-memory tile and the store.
template <typename T, int TR_TILE>
__global__ void __launch_bounds__(256) adjoint_box_kernel(Cplx<T>* __restrict__ dst, size_t dst_ld, const Cplx<T>* __restrict__ src,
                                                          size_t src_ld, size_t rows, size_t cols, unsigned tiles_r) {
    __shared__ Cplx<T> tile[TR_TILE][TR_TILE + 1];
    const size_t tr = blockIdx.x % tiles_r, tc = blockIdx.x / tiles_r;
    const size_t r0 = tr * TR_TILE, c0 = tc * TR_TILE;
    constexpr int TY = 256 / TR_TILE;
    constexpr int NK = TR_TILE / TY;
    const int tx = threadIdx.x & (TR_TILE - 1), ty = threadIdx.x / TR_TILE;
    Cplx<T> v[NK];
#pragma unroll
    for (int q = 0; q < NK; ++q) {
        const size_t r = r0 + tx, c = c0 + ty + q * TY;
        v[q] = (r < rows && c < cols) ? src[r + c * src_ld] : Cplx<T>{};
    }
#pragma unroll
    for (int q = 0; q < NK; ++q) tile[ty + q * TY][tx] = v[q];
    __syncthreads();
#pragma unroll 4
    for (int k = ty; k < TR_TILE; k += TY) {
        const size_t c = c0 + tx, r = r0 + k;
        if (r < rows && c < cols) {
            Cplx<T> z = tile[tx][k];
            z.im = flip_sign(z.im);
            dst[c + r * dst_ld] = z;
        }
    }
}

template <typename T>
int32_t launch_adjoint(dab_ctx* ctx, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows, size_t cols) {
    constexpr int TR_TILE = 32;  // as dab_transpose_box for 8- and 16-byte units
    DAB_REQUIRE(ctx, (uintptr_t)dst % sizeof(Cplx<T>) == 0 && (uintptr_t)src % sizeof(Cplx<T>) == 0, DAB_ERR_ARG,
                "dab_adjoint_box: data must be aligned to the element size");
    const size_t tiles_r = (rows + TR_TILE - 1) / TR_TILE, tiles_c = (cols + TR_TILE - 1) / TR_TILE;
    DAB_REQUIRE(ctx, tiles_r * tiles_c <= 0x7fffffffull && tiles_r <= 0xffffffffull, DAB_ERR_ARG, "dab_adjoint_box: too many tiles");
    adjoint_box_kernel<T, TR_TILE><<<(unsigned)(tiles_r * tiles_c), 256, 0, ctx->stream>>>((Cplx<T>*)dst, dst_ld, (const Cplx<T>*)src, src_ld, rows,
                                                                                         cols, (unsigned)tiles_r);
    DAB_LAUNCHED(ctx);
    return DAB_OK;
}

}  // namespace

extern "C" int32_t dab_adjoint_box(dab_ctx* ctx, int32_t dtype, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows,
                                   size_t cols) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, dtype == DAB_C64 || dtype == DAB_C128, DAB_ERR_UNSUPPORTED,
                "dab_adjoint_box: dtype %d is not complex (the adjoint of a real matrix is dab_transpose_box)", dtype);
    if (rows == 0 || cols == 0) return DAB_OK;
    DAB_REQUIRE(ctx, dst && src, DAB_ERR_ARG, "dab_adjoint_box: null pointer");
    DAB_REQUIRE(ctx, src_ld >= rows && dst_ld >= cols, DAB_ERR_DIM_MISMATCH, "dab_adjoint_box: leading dimension smaller than the box");
    if (dtype == DAB_C64) return launch_adjoint<float>(ctx, dst, dst_ld, src, src_ld, rows, cols);
    return launch_adjoint<double>(ctx, dst, dst_ld, src, src_ld, rows, cols);
}

extern "C" int32_t dab_transpose_box(dab_ctx* ctx, int32_t elem_bytes, void* dst, size_t dst_ld, const void* src, size_t src_ld, size_t rows,
                                     size_t cols) {
    DAB_ENTER(ctx);
    if (rows == 0 || cols == 0) return DAB_OK;
    DAB_REQUIRE(ctx, dst && src, DAB_ERR_ARG, "dab_transpose_box: null pointer");
    DAB_REQUIRE(ctx, src_ld >= rows && dst_ld >= cols, DAB_ERR_DIM_MISMATCH, "dab_transpose_box: leading dimension smaller than the box");
    switch (elem_bytes) {
        case 1: return launch_transpose<uint8_t>(ctx, dst, dst_ld, src, src_ld, rows, cols);
        case 2: return launch_transpose<uint16_t>(ctx, dst, dst_ld, src, src_ld, rows, cols);
        case 4: return launch_transpose<uint32_t>(ctx, dst, dst_ld, src, src_ld, rows, cols);
        case 8: return launch_transpose<uint64_t>(ctx, dst, dst_ld, src, src_ld, rows, cols);
        case 16: return launch_transpose<int4>(ctx, dst, dst_ld, src, src_ld, rows, cols);
        default: return dab_fail(ctx, DAB_ERR_ARG, "dab_transpose_box: elem_bytes %d", elem_bytes);
    }
}
