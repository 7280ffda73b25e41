// dab_lu_core.cuh -- the per-element arithmetic of K27 (dab_lu_batched.cu: batched `A \ B` and `det(A)` of small dense slices) as
// __host__ __device__ functions, so that the very same code runs inside the kernels and inside tools/lu_host_check.cu (a host-only replay
// of the path choice, the pivoting, the substitutions and the determinant against NumPy / SciPy; built and run by the CPU test tier).
//
// Julia's dispatch, restated from LinearAlgebra (Julia 1.10, generic.jl):
//   A \ B:   istril(A) && istriu(A): Diagonal(A) \ B, x = b ./ d, SingularException(i) for the first d_i == 0;
//            istril(A) / istriu(A):  forward / backward substitution, SingularException(i) for the first zero diagonal entry (trtrs!);
//            otherwise lu(A) \ B:    partial pivoting (idamax), ArgumentError for a NaN / Inf anywhere in A (getrf!'s chkfinite),
//                                    SingularException(info) for the first exactly-zero pivot.
//   det(A):  istriu(A) || istril(A): prod(diag(A)) in index order; otherwise det(lu(A; check=false)): the product of U's diagonal in index
//            order, negated for an odd number of row swaps, +0.0 when a pivot is exactly zero.  det never raises.
// The structure tests are exact `== 0` comparisons (iszero): -0.0 is zero, NaN is not.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>

enum LuPath : int { LU_PATH_LU = 0, LU_PATH_LOWER = 1, LU_PATH_UPPER = 2, LU_PATH_DIAG = 3 };

// entry a_ij (0-based) keeps A from being lower triangular / upper triangular
__host__ __device__ inline bool lu_breaks_lower(int i, int j, double v) { return j > i && v != 0.0; }
__host__ __device__ inline bool lu_breaks_upper(int i, int j, double v) { return j < i && v != 0.0; }

// the path of `A \ B` from "some entry above the diagonal is nonzero" (not_lower) and "some entry below it is nonzero" (not_upper)
__host__ __device__ inline int lu_ldiv_path(bool not_lower, bool not_upper) {
    if (!not_lower) return not_upper ? LU_PATH_LOWER : LU_PATH_DIAG;
    return not_upper ? LU_PATH_LU : LU_PATH_UPPER;
}

// det takes the diagonal product for either triangle
__host__ __device__ inline bool lu_det_triangular(bool not_lower, bool not_upper) { return !not_lower || !not_upper; }

// ---- pivot choice: LAPACK's idamax over the candidates at positions k, k+1, ... of column k ----------------------------------------------
// idamax keeps the first index whose |x| is strictly larger than every earlier one, starting from position k.  A NaN never compares larger,
// so it is skipped -- unless it sits at position k itself, where it stays the maximum.  As a key: larger wins, equal keys go to the lower
// position.  A row that is no longer a candidate has key -2.
__host__ __device__ inline double lu_pivot_key(double v, int pos, int k) {
    if (v != v) return pos == k ? INFINITY : -1.0;
    return fabs(v);
}

__host__ __device__ inline bool lu_pivot_wins(double key_a, int pos_a, double key_b, int pos_b) {
    return key_a > key_b || (key_a == key_b && pos_a < pos_b);
}

// ---- elimination -------------------------------------------------------------------------------------------------------------------------
// dgetrf2 scales the column below the pivot by 1 / pivot when |pivot| >= sfmin and divides otherwise
__host__ __device__ inline bool lu_use_reciprocal(double piv) { return fabs(piv) >= DBL_MIN; }

__host__ __device__ inline double lu_multiplier(double aik, double piv, double rpiv, bool recip) { return recip ? aik * rpiv : aik / piv; }

// a_ij - l_i * u_kj with one rounding (the rank-1 update of dger / dgemm on an FMA machine)
__host__ __device__ inline double lu_update(double aij, double l, double ukj) { return fma(-l, ukj, aij); }

// ---- substitutions ---------------------------------------------------------------------------------------------------------------------
// y_i - a_is * x_s (dtrsm's column sweep) ...
__host__ __device__ inline double lu_subst(double yi, double ais, double xs) { return fma(-ais, xs, yi); }
// ... and the division by the diagonal entry (also the whole of the diagonal path, b ./ d)
__host__ __device__ inline double lu_divide(double y, double d) { return y / d; }

// ---- determinant ---------------------------------------------------------------------------------------------------------------------
__host__ __device__ inline double lu_det_step(double acc, double d) { return acc * d; }

// det(F::LU): zero(T) unless issuccess (info == 0), otherwise the diagonal product times (-1)^swaps
__host__ __device__ inline double lu_det_finish(double prod, int swaps, int info) {
    if (info != 0) return 0.0;
    return (swaps & 1) ? prod * -1.0 : prod;
}

// ---- status word -----------------------------------------------------------------------------------------------------------------------
// One uint64 per call, all ones when no slice failed.  A failing slice b writes (b << 8) | low with atomicMin, low = info (1-based, <= 64)
// for a SingularException or LU_STATUS_NONFINITE for the ArgumentError of a NaN / Inf on the LU path: the word ends as the lowest failing b.
constexpr unsigned long long LU_STATUS_CLEAR = ~0ull;
constexpr unsigned int LU_STATUS_NONFINITE = 0x80u;

__host__ __device__ inline unsigned long long lu_status_key(size_t b, int info, bool nonfinite) {
    return ((unsigned long long)b << 8) | (nonfinite ? LU_STATUS_NONFINITE : (unsigned int)info);
}
