// dab_slices_core.cuh -- the per-element arithmetic of the slice kernels (dab_slices.cu) as __host__ __device__ functions, so that the
// very same code runs inside the kernels and inside tools/slices_host_check.cu (a host-only replay of the bitonic network against
// std::sort and of the Jacobi sweeps against numpy.linalg.svd; built and run by the CPU test tier).
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "dab_sort_key.cuh"

// ---- segmented sort: bitonic network over B fibres of one CTA, each padded to P2 = 2^log2p2 keys -------------------------------------
// Compare/exchange p of a (k, j) stage: positions i < i + j inside the group.  Every fibre is sorted ascending: inside a fibre the usual
// bitonic directions, and the last merge (k == P2) ascending for all fibres -- (i & P2) would otherwise alternate with the fibre's parity.
__host__ __device__ inline unsigned int slices_bitonic_lo(unsigned int p, unsigned int j) { return ((p & ~(j - 1u)) << 1) | (p & (j - 1u)); }
__host__ __device__ inline bool slices_bitonic_asc(unsigned int i, unsigned int k, unsigned int p2) { return k == p2 || (i & k) == 0u; }

// position of key i of the group in shared memory: fibre (i >> log2p2) starts every P2 + 1 keys (one pad key against bank conflicts of
// the transposed staging when inner > 1)
__host__ __device__ inline unsigned int slices_smem_index(unsigned int i, unsigned int log2p2) {
    return (i >> log2p2) * ((1u << log2p2) + 1u) + (i & ((1u << log2p2) - 1u));
}

template <typename U>
__host__ __device__ inline void slices_cmpx(U& a, U& b, bool asc) {
    if ((a > b) == asc) {
        const U t = a;
        a = b;
        b = t;
    }
}

// the padding key: above every key except an equal all-ones key, whose bits are the same
template <typename U>
__host__ __device__ inline U slices_pad_key() { return (U)~(U)0; }

__host__ __device__ inline unsigned int slices_log2_ceil(size_t n) {
    unsigned int l = 0;
    while (((size_t)1 << l) < n) ++l;
    return l;
}

// ---- batched singular values: one-sided (Hestenes) Jacobi ---------------------------------------------------------------------------
// Round-robin ("circle") pairing of np (even) columns: round r < np - 1, pair k < np / 2.  Column 0 stays, the others rotate; every pair of
// columns meets exactly once per sweep and the pairs of one round are disjoint, so they are rotated in parallel.
__host__ __device__ inline void slices_rr_pair(int np, int r, int k, int* p, int* q) {
    const int m = np - 1;
    *p = k == 0 ? 0 : (k - 1 + r) % m + 1;
    *q = (np - 2 - k + r) % m + 1;
}

// Rotation that makes columns p and q orthogonal, from alpha = |a_p|^2, beta = |a_q|^2, gamma = a_p . a_q:
//   a_p <- c a_p - s a_q,  a_q <- s a_p + c a_q  (the smaller root t = s / c of t^2 + 2 zeta t - 1 = 0).
// Returns false when the pair is already orthogonal to the tolerance |gamma| <= tol * |a_p| |a_q|.
__host__ __device__ inline bool slices_jacobi_rotation(double alpha, double beta, double gamma, double tol, double* c, double* s) {
    if (!(fabs(gamma) > tol * sqrt(alpha) * sqrt(beta))) return false;
    const double zeta = (beta - alpha) / (2.0 * gamma);
    double t;
    if (fabs(zeta) > 1e150) t = 0.5 / zeta;   // 1 + zeta^2 would overflow; t = 1 / (2 zeta) to working precision
    else t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    *c = 1.0 / sqrt(1.0 + t * t);
    *s = *c * t;
    return true;
}

__host__ __device__ inline void slices_jacobi_apply(double* ap, double* aq, double c, double s) {
    const double x = *ap, y = *aq;
    *ap = c * x - s * y;
    *aq = s * x + c * y;
}

// The matrix is scaled by 2^-e, amax * 2^-e in [0.5, 1), before the sweeps and the column norms by 2^e after them (exact: powers of
// two), so that the sums of squares neither overflow nor underflow for any finite input whose entries lie within ~1e150 of its largest
// (LAPACK's dgesvj scales its input too).
__host__ __device__ inline int slices_scale_exp(double amax) {
    int e = 0;
    if (amax > 0.0) frexp(amax, &e);
    return e;
}

constexpr int DAB_SVD_MAX_SWEEPS = 40;

// pair tolerance of a sweep over columns of `rows` entries (LAPACK dgesvj's sqrt(m) * eps)
__host__ __device__ inline double slices_jacobi_tol(int rows) { return 2.220446049250313e-16 * sqrt((double)rows); }

// ---- batched symmetric eigenvalues: two-sided cyclic Jacobi ---------------------------------------------------------------------------
// A round takes the round-robin pairs of slices_rr_pair: every rotation is computed from the current 2x2 pivots first, then all rows
// p, q are rotated (J^T A), then all columns (A J); the pairs of a round are disjoint, so this is J^T A J exactly.  A sweep is np - 1
// rounds; sweeps stop when no pair needed a rotation, or after DAB_EIG_MAX_SWEEPS.
constexpr int DAB_EIG_MAX_SWEEPS = 40;
// relative off-diagonal test: |a_pq| <= eps sqrt(|a_pp| |a_qq|) counts as zero ...
constexpr double DAB_EIG_TOL = 2.220446049250313e-16;
// ... and so does |a_pq| <= 2^-80 once the matrix is scaled to max |a| in [0.5, 1): by Weyl's bound that moves no eigenvalue by more than
// 2^-80 of the largest entry, and it keeps the rounding noise around eigenvalues near 0 (rank-deficient input) from being rotated forever
constexpr double DAB_EIG_ABS_FLOOR = 8.271806125530277e-25;

// Rotation (c, s) that zeroes a_pq of J^T A J, J = [c s; -s c] in rows / columns (p, q): t = s / c is the smaller root of
// t^2 + 2 zeta t - 1 = 0, zeta = (a_qq - a_pp) / (2 a_pq) (Golub & Van Loan, sym.schur2).  Returns false when a_pq counts as zero.
__host__ __device__ inline bool slices_sym_rotation(double app, double aqq, double apq, double* c, double* s) {
    const double g = fabs(apq);
    if (!(g > DAB_EIG_TOL * sqrt(fabs(app)) * sqrt(fabs(aqq)) && g > DAB_EIG_ABS_FLOOR)) return false;
    const double zeta = (aqq - app) / (2.0 * apq);
    double t;
    if (fabs(zeta) > 1e150) t = 0.5 / zeta;   // 1 + zeta^2 would overflow; t = 1 / (2 zeta) to working precision
    else t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    *c = 1.0 / sqrt(1.0 + t * t);
    *s = *c * t;
    return true;
}

// position of d[i] among d[0 .. n) in ascending order, ties by index (the eigenvalues are written at their rank)
__host__ __device__ inline int slices_rank_asc(const double* d, int n, int i) {
    const double v = d[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += d[j] < v || (d[j] == v && j < i);
    return rank;
}
