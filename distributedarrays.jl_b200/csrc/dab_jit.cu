// dab_jit.cu -- general fused broadcast: ONE kernel per localpart for an arbitrary expression tree, compiled at run time.
//
// Replaces what Julia's JIT does for  copyto!(localpart(dest), lbc::Broadcasted)  (reference src/broadcast.jl:80) and
// copy(lbc) (:96): the whole tree  f.(args...)  is fused into a single pass over the chunk -- N-ary, nested, with size-1
// ("extruded", src/broadcast.jl:112-113) dims and mixed element types.  The host runtime (distributedarrays.jl_b200/
// _broadcast.py) traces the user's function into C source for ONE element (Julia promotion already applied); this file
// wraps it into two sm_90a kernels with NVRTC (-fmad=false: no FMA contraction, Julia semantics):
//   dab_bc_linear  : every array argument is dense and has the destination's shape -> 4 consecutive elements per thread,
//                    16/32-byte vector loads and stores, grid-stride (HBM roofline: sum of element sizes per element);
//   dab_bc_general : per-argument strides (0 = extruded dim), coalesced along dim 0.
// Kernels are cached per (device, expression, element types, argument kinds).  NVRTC and the driver entry points are
// resolved at run time (dlopen / cudaGetDriverEntryPoint), so libdab200.so loads on a machine without a GPU.
#include <cuda.h>
#include <dlfcn.h>
#include <nvrtc.h>

#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "dab_common.cuh"

namespace {

const char* kPrelude = R"PRELUDE(
typedef unsigned long long u64;
typedef long long i64;
#define DEV __device__ __forceinline__
// ---- Julia scalar semantics: one IEEE rounding per operation, never contracted ----
DEV float jl_add(float a, float b) { return __fadd_rn(a, b); }
DEV float jl_sub(float a, float b) { return __fsub_rn(a, b); }
DEV float jl_mul(float a, float b) { return __fmul_rn(a, b); }
DEV float jl_div(float a, float b) { return __fdiv_rn(a, b); }
DEV double jl_add(double a, double b) { return __dadd_rn(a, b); }
DEV double jl_sub(double a, double b) { return __dsub_rn(a, b); }
DEV double jl_mul(double a, double b) { return __dmul_rn(a, b); }
DEV double jl_div(double a, double b) { return __ddiv_rn(a, b); }
DEV int jl_add(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
DEV int jl_sub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }
DEV int jl_mul(int a, int b) { return (int)((unsigned)a * (unsigned)b); }
DEV i64 jl_add(i64 a, i64 b) { return (i64)((u64)a + (u64)b); }
DEV i64 jl_sub(i64 a, i64 b) { return (i64)((u64)a - (u64)b); }
DEV i64 jl_mul(i64 a, i64 b) { return (i64)((u64)a * (u64)b); }
DEV float jl_max(float a, float b) { float r; asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
DEV float jl_min(float a, float b) { float r; asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
DEV double jl_max(double a, double b) {
    if (a != a || b != b) return __longlong_as_double(0x7ff8000000000000ll);
    if (a == b) return (__double_as_longlong(a) < 0) ? b : a;
    return a > b ? a : b;
}
DEV double jl_min(double a, double b) {
    if (a != a || b != b) return __longlong_as_double(0x7ff8000000000000ll);
    if (a == b) return (__double_as_longlong(a) < 0) ? a : b;
    return a < b ? a : b;
}
DEV int jl_max(int a, int b) { return a > b ? a : b; }
DEV int jl_min(int a, int b) { return a < b ? a : b; }
DEV i64 jl_max(i64 a, i64 b) { return a > b ? a : b; }
DEV i64 jl_min(i64 a, i64 b) { return a < b ? a : b; }
DEV bool jl_max(bool a, bool b) { return a || b; }
DEV bool jl_min(bool a, bool b) { return a && b; }
DEV float jl_rem(float a, float b) { return fmodf(a, b); }
DEV double jl_rem(double a, double b) { return fmod(a, b); }
DEV int jl_rem(int a, int b) { return (b == 0 || b == -1) ? 0 : a % b; }
DEV i64 jl_rem(i64 a, i64 b) { return (b == 0 || b == -1) ? 0 : a % b; }
DEV float jl_mod(float x, float y) { float r = fmodf(x, y); if (r == 0.f) return copysignf(r, y); return ((r > 0.f) != (y > 0.f)) ? __fadd_rn(r, y) : r; }
DEV double jl_mod(double x, double y) { double r = fmod(x, y); if (r == 0.0) return copysign(r, y); return ((r > 0.0) != (y > 0.0)) ? __dadd_rn(r, y) : r; }
DEV int jl_mod(int a, int b) { if (b == 0 || b == -1) return 0; int r = a % b; return (r != 0 && ((r < 0) != (b < 0))) ? r + b : r; }
DEV i64 jl_mod(i64 a, i64 b) { if (b == 0 || b == -1) return 0; i64 r = a % b; return (r != 0 && ((r < 0) != (b < 0))) ? r + b : r; }
DEV int jl_idiv(int a, int b) { if (b == 0) return 0; if (b == -1) return (int)(0u - (unsigned)a); return a / b; }
DEV i64 jl_idiv(i64 a, i64 b) { if (b == 0) return 0; if (b == -1) return (i64)(0ull - (u64)a); return a / b; }
DEV float jl_pow(float a, float b) { return powf(a, b); }
DEV double jl_pow(double a, double b) { return pow(a, b); }
DEV int jl_and(int a, int b) { return a & b; }
DEV int jl_or(int a, int b) { return a | b; }
DEV int jl_xor(int a, int b) { return a ^ b; }
DEV i64 jl_and(i64 a, i64 b) { return a & b; }
DEV i64 jl_or(i64 a, i64 b) { return a | b; }
DEV i64 jl_xor(i64 a, i64 b) { return a ^ b; }
DEV bool jl_and(bool a, bool b) { return a && b; }
DEV bool jl_or(bool a, bool b) { return a || b; }
DEV bool jl_xor(bool a, bool b) { return a != b; }
template <typename T> DEV bool jl_lt(T a, T b) { return a < b; }
template <typename T> DEV bool jl_le(T a, T b) { return a <= b; }
template <typename T> DEV bool jl_gt(T a, T b) { return a > b; }
template <typename T> DEV bool jl_ge(T a, T b) { return a >= b; }
template <typename T> DEV bool jl_eq(T a, T b) { return a == b; }
template <typename T> DEV bool jl_ne(T a, T b) { return a != b; }
DEV float jl_neg(float a) { return -a; }
DEV double jl_neg(double a) { return -a; }
DEV int jl_neg(int a) { return (int)(0u - (unsigned)a); }
DEV i64 jl_neg(i64 a) { return (i64)(0ull - (u64)a); }
DEV float jl_abs(float a) { return fabsf(a); }
DEV double jl_abs(double a) { return fabs(a); }
DEV int jl_abs(int a) { return a < 0 ? (int)(0u - (unsigned)a) : a; }
DEV i64 jl_abs(i64 a) { return a < 0 ? (i64)(0ull - (u64)a) : a; }
template <typename T> DEV T jl_abs2(T a) { return jl_mul(a, a); }
DEV float jl_sqrt(float a) { return __fsqrt_rn(a); }
DEV double jl_sqrt(double a) { return __dsqrt_rn(a); }
DEV float jl_inv(float a) { return __fdiv_rn(1.0f, a); }
DEV double jl_inv(double a) { return __ddiv_rn(1.0, a); }
DEV float jl_floor(float a) { return floorf(a); }
DEV double jl_floor(double a) { return floor(a); }
DEV float jl_ceil(float a) { return ceilf(a); }
DEV double jl_ceil(double a) { return ceil(a); }
template <typename T> DEV T jl_floor(T a) { return a; }
template <typename T> DEV T jl_ceil(T a) { return a; }
template <typename T> DEV T jl_sign(T a) { return a > (T)0 ? (T)1 : (a < (T)0 ? (T)(-1) : a); }
template <typename T> DEV bool jl_isnan(T a) { return a != a; }
template <typename T> DEV bool jl_isinf(T a) { return (a == a) && ((a - a) != (a - a)); }
template <typename T> DEV bool jl_isfinite(T a) { return (a - a) == (a - a); }
// transcendental functions: CUDA's libdevice (<= 1-2 ulp); NOT bit-identical to Julia's openlibm-derived kernels
#define JL_F1(name, ff, fd) DEV float jl_##name(float a) { return ff(a); } DEV double jl_##name(double a) { return fd(a); }
JL_F1(sin, sinf, sin) JL_F1(cos, cosf, cos) JL_F1(tan, tanf, tan) JL_F1(exp, expf, exp) JL_F1(exp2, exp2f, exp2)
JL_F1(log, logf, log) JL_F1(log2, log2f, log2) JL_F1(log10, log10f, log10) JL_F1(tanh, tanhf, tanh) JL_F1(sinh, sinhf, sinh)
JL_F1(cosh, coshf, cosh) JL_F1(atan, atanf, atan) JL_F1(asin, asinf, asin) JL_F1(acos, acosf, acos) JL_F1(expm1, expm1f, expm1)
JL_F1(log1p, log1pf, log1p) JL_F1(cbrt, cbrtf, cbrt)

struct BcParams {
    void* out;
    u64 shape[4];
    i64 ostr[4];
    const void* ptr[8];
    i64 str[8][4];
    u64 scalar[8];
};
template <typename T, int N> struct __align__(sizeof(T) * N) VecN { T v[N]; };
template <typename T> DEV T bits_as(u64 b) { T r; memcpy(&r, &b, sizeof(T)); return r; }
)PRELUDE";

// Int128 as the VALUE type of a fused map + reduce (f widens its argument: x -> Int128(x)^2 + 2 Int128(x) - 1, test/darray.jl:286-294).
// Appended to the prelude -- and NVRTC's --device-int128 switched on -- only for sources that mention the type, so every other generated
// kernel is byte-for-byte what it was.
const char* kPreludeI128 = R"PRELUDE(
typedef __int128 i128;
typedef unsigned __int128 u128;
DEV i128 jl_add(i128 a, i128 b) { return (i128)((u128)a + (u128)b); }
DEV i128 jl_sub(i128 a, i128 b) { return (i128)((u128)a - (u128)b); }
DEV i128 jl_mul(i128 a, i128 b) { return (i128)((u128)a * (u128)b); }
DEV i128 jl_neg(i128 a) { return (i128)((u128)0 - (u128)a); }
DEV i128 jl_abs(i128 a) { return a < 0 ? (i128)((u128)0 - (u128)a) : a; }
DEV i128 jl_max(i128 a, i128 b) { return a > b ? a : b; }
DEV i128 jl_min(i128 a, i128 b) { return a < b ? a : b; }
DEV i128 jl_and(i128 a, i128 b) { return a & b; }
DEV i128 jl_or(i128 a, i128 b) { return a | b; }
DEV i128 jl_xor(i128 a, i128 b) { return a ^ b; }
)PRELUDE";

bool mentions_i128(const char* expr) { return expr && strstr(expr, "i128") != nullptr; }

// Further unary functions of the reference's "scalar math" test (test/darray.jl:775-797) that CUDA's libdevice provides; same accuracy
// note as the transcendental block of the prelude (<= 1-2 ulp, not bit-identical to Julia's openlibm / SpecialFunctions kernels).  The
// tracer spells them jl_x_*; the block is appended only to sources that use one, so every other generated kernel stays byte-identical.
const char* kPreludeExt = R"PRELUDE(
#define JL_X1(name, ff, fd) DEV float jl_x_##name(float a) { return ff(a); } DEV double jl_x_##name(double a) { return fd(a); }
JL_X1(asinh, asinhf, asinh) JL_X1(acosh, acoshf, acosh) JL_X1(atanh, atanhf, atanh) JL_X1(exp10, exp10f, exp10)
JL_X1(sinpi, sinpif, sinpi) JL_X1(cospi, cospif, cospi) JL_X1(trunc, truncf, trunc) JL_X1(round, rintf, rint)
JL_X1(erf, erff, erf) JL_X1(erfc, erfcf, erfc) JL_X1(erfinv, erfinvf, erfinv) JL_X1(erfcinv, erfcinvf, erfcinv) JL_X1(erfcx, erfcxf, erfcx)
JL_X1(gamma, tgammaf, tgamma) JL_X1(loggamma, lgammaf, lgamma)
template <typename T> DEV T jl_x_trunc(T a) { return a; }
template <typename T> DEV T jl_x_round(T a) { return a; }
// x << n, x >> n (test/darray.jl:863-867) with Julia's semantics: the result has the type of x; n counts bits as an Int64; a negative n
// shifts the other way; shifting out every bit gives 0 (<<) or the sign fill (>>, arithmetic).
DEV i64 jl_x_shr(i64 a, i64 n);
DEV i64 jl_x_shl(i64 a, i64 n) {
    if (n < 0) return n <= -64 ? (a < 0 ? -1ll : 0ll) : (a >> (int)(-n));
    return n >= 64 ? 0ll : (i64)((u64)a << (int)n);
}
DEV i64 jl_x_shr(i64 a, i64 n) {
    if (n < 0) return n <= -64 ? 0ll : (i64)((u64)a << (int)(-n));
    return n >= 64 ? (a < 0 ? -1ll : 0ll) : (a >> (int)n);
}
DEV int jl_x_shl(int a, i64 n) {
    if (n < 0) return n <= -32 ? (a < 0 ? -1 : 0) : (a >> (int)(-n));
    return n >= 32 ? 0 : (int)((unsigned)a << (int)n);
}
DEV int jl_x_shr(int a, i64 n) {
    if (n < 0) return n <= -32 ? 0 : (int)((unsigned)a << (int)(-n));
    return n >= 32 ? (a < 0 ? -1 : 0) : (a >> (int)n);
}
)PRELUDE";

bool mentions_ext(const char* expr) { return expr && strstr(expr, "jl_x_") != nullptr; }

// Julia methods that are not "promote both operands, then operate" (the tracer spells them jl_m_*).  Appended only to sources that use
// one, so every other generated kernel stays byte-identical.
//   copysign        -- Bool * x = ifelse(b, x, copysign(zero(x), x)) for a float x (base/bool.jl)
//   eq ne lt le ... -- Int64 against Float32 / Float64 compares the values exactly (base/float.jl), without rounding the Int64
//   powi            -- ^(x::Float32, n::Integer) (base/math.jl): n == -2 is inv(x)^2 and n == 3 is x*x*x in Float32, otherwise
//                      Float32(power_by_squaring(Float64(x), n)), from inv(Float64(x)) when n < 0; the magnitude of a typemin n is 2^63
const char* kPreludeMethods = R"PRELUDE(
DEV float jl_m_copysign(float a, float b) { return copysignf(a, b); }
DEV double jl_m_copysign(double a, double b) { return copysign(a, b); }
// three-way comparison of an Int64 with a Float64 value: -1, 0, 1, or 2 when f is NaN
DEV int jl_m_cmp(i64 a, double f) {
    if (f != f) return 2;
    if (f >= 0x1p63) return -1;
    if (f < -0x1p63) return 1;
    const double t = trunc(f);
    const i64 ti = (i64)t;                          // exact: |t| < 2^63 or t == -2^63
    if (a != ti) return a < ti ? -1 : 1;
    const double fr = f - t;                        // exact
    return fr > 0.0 ? -1 : (fr < 0.0 ? 1 : 0);
}
DEV int jl_m_cmp(double f, i64 a) { const int c = jl_m_cmp(a, f); return c == 2 ? 2 : -c; }
DEV int jl_m_cmp(i64 a, float f) { return jl_m_cmp(a, (double)f); }
DEV int jl_m_cmp(float f, i64 a) { return jl_m_cmp((double)f, a); }
template <typename A, typename B> DEV bool jl_m_eq(A a, B b) { return jl_m_cmp(a, b) == 0; }
template <typename A, typename B> DEV bool jl_m_ne(A a, B b) { return jl_m_cmp(a, b) != 0; }
template <typename A, typename B> DEV bool jl_m_lt(A a, B b) { return jl_m_cmp(a, b) == -1; }
template <typename A, typename B> DEV bool jl_m_le(A a, B b) { const int c = jl_m_cmp(a, b); return c == -1 || c == 0; }
template <typename A, typename B> DEV bool jl_m_gt(A a, B b) { return jl_m_cmp(a, b) == 1; }
template <typename A, typename B> DEV bool jl_m_ge(A a, B b) { const int c = jl_m_cmp(a, b); return c == 1 || c == 0; }
// Base.power_by_squaring(x, p) for p >= 0, operation by operation (a shift by the full width gives 0)
DEV double jl_m_pbs(double x, u64 p) {
    if (p == 1) return x;
    if (p == 0) return 1.0;
    if (p == 2) return __dmul_rn(x, x);
    int t = __ffsll((long long)p);                  // trailing_zeros(p) + 1
    p = t >= 64 ? 0 : p >> t;
    while (--t > 0) x = __dmul_rn(x, x);
    double y = x;
    while (p > 0) {
        t = __ffsll((long long)p);
        p = t >= 64 ? 0 : p >> t;
        while (--t >= 0) x = __dmul_rn(x, x);
        y = __dmul_rn(y, x);
    }
    return y;
}
DEV float jl_m_powi(float x, i64 n) {
    if (n == -2) { const float i = __fdiv_rn(1.0f, x); return __fmul_rn(i, i); }
    if (n == 3) return __fmul_rn(__fmul_rn(x, x), x);
    if (n < 0) return (float)jl_m_pbs(__ddiv_rn(1.0, (double)x), 0ull - (u64)n);
    return (float)jl_m_pbs((double)x, (u64)n);
}
)PRELUDE";

bool mentions_methods(const char* expr) { return expr && strstr(expr, "jl_m_") != nullptr; }

// ComplexF32 / ComplexF64 values (jl_c64 / jl_c128: interleaved (re, im), Julia's Complex{T} layout), with Julia's definitions of the
// operations the tracer serves on them.  Appended only to sources that use a complex type (an argument, output or value dtype, or one of
// the names below in the expression), so every other generated kernel is byte-for-byte what it was.
const char* kPreludeCplx = R"PRELUDE(
struct jl_c128;
struct __align__(8) jl_c64 {
    float re, im;
    jl_c64() = default;
    DEV jl_c64(float r, float i) : re(r), im(i) {}
    DEV jl_c64(float r) : re(r), im(0.f) {}
    DEV jl_c64(double r) : re((float)r), im(0.f) {}
    DEV jl_c64(int r) : re((float)r), im(0.f) {}
    DEV jl_c64(i64 r) : re((float)r), im(0.f) {}
    DEV jl_c64(bool r) : re(r ? 1.f : 0.f), im(0.f) {}
    DEV explicit jl_c64(const jl_c128& z);
};
struct __align__(16) jl_c128 {
    double re, im;
    jl_c128() = default;
    DEV jl_c128(double r, double i) : re(r), im(i) {}
    DEV jl_c128(double r) : re(r), im(0.0) {}
    DEV jl_c128(float r) : re((double)r), im(0.0) {}
    DEV jl_c128(int r) : re((double)r), im(0.0) {}
    DEV jl_c128(i64 r) : re((double)r), im(0.0) {}
    DEV jl_c128(bool r) : re(r ? 1.0 : 0.0), im(0.0) {}
    DEV jl_c128(const jl_c64& z) : re((double)z.re), im((double)z.im) {}
};
DEV jl_c64::jl_c64(const jl_c128& z) : re((float)z.re), im((float)z.im) {}
// the 16-byte result slot of a ComplexF32 reduction: the value, then zeros
struct __align__(16) jl_c64_slot {
    jl_c64 v;
    float pad[2];
    jl_c64_slot() = default;
    DEV jl_c64_slot(const jl_c128& z) : v(z), pad{0.f, 0.f} {}
    DEV jl_c64_slot(bool b) : v(b), pad{0.f, 0.f} {}
};
DEV bool operator==(jl_c64 a, jl_c64 b) { return a.re == b.re && a.im == b.im; }
DEV bool operator!=(jl_c64 a, jl_c64 b) { return !(a == b); }
DEV bool operator==(jl_c128 a, jl_c128 b) { return a.re == b.re && a.im == b.im; }
DEV bool operator!=(jl_c128 a, jl_c128 b) { return !(a == b); }
DEV float jl_real(jl_c64 z) { return z.re; }
DEV double jl_real(jl_c128 z) { return z.re; }
DEV float jl_imag(jl_c64 z) { return z.im; }
DEV double jl_imag(jl_c128 z) { return z.im; }
DEV jl_c64 jl_conj(jl_c64 z) { return jl_c64(z.re, -z.im); }
DEV jl_c128 jl_conj(jl_c128 z) { return jl_c128(z.re, -z.im); }
DEV jl_c64 jl_neg(jl_c64 z) { return jl_c64(-z.re, -z.im); }
DEV jl_c128 jl_neg(jl_c128 z) { return jl_c128(-z.re, -z.im); }
DEV bool jl_isnan(jl_c64 z) { return z.re != z.re || z.im != z.im; }
DEV bool jl_isnan(jl_c128 z) { return z.re != z.re || z.im != z.im; }
DEV bool jl_isinf(jl_c64 z) { return jl_isinf(z.re) || jl_isinf(z.im); }
DEV bool jl_isinf(jl_c128 z) { return jl_isinf(z.re) || jl_isinf(z.im); }
DEV bool jl_isfinite(jl_c64 z) { return jl_isfinite(z.re) && jl_isfinite(z.im); }
DEV bool jl_isfinite(jl_c128 z) { return jl_isfinite(z.re) && jl_isfinite(z.im); }
// + - * between complex values; * is (ac - bd, ad + bc), every operation rounded separately
#define JL_CPLX_ARITH(C, R)                                                                                        \
DEV C jl_add(C a, C b) { return C(jl_add(a.re, b.re), jl_add(a.im, b.im)); }                                        \
DEV C jl_sub(C a, C b) { return C(jl_sub(a.re, b.re), jl_sub(a.im, b.im)); }                                        \
DEV C jl_mul(C a, C b) { return C(jl_sub(jl_mul(a.re, b.re), jl_mul(a.im, b.im)), jl_add(jl_mul(a.re, b.im), jl_mul(a.im, b.re))); } \
/* mixed real / complex: Julia's specialised methods, the real operand is NOT promoted to complex first */          \
DEV C jl_add(R x, C z) { return C(jl_add(x, z.re), z.im); }                                                         \
DEV C jl_add(C z, R x) { return C(jl_add(z.re, x), z.im); }                                                         \
DEV C jl_sub(R x, C z) { return C(jl_sub(x, z.re), -z.im); }                                                        \
DEV C jl_sub(C z, R x) { return C(jl_sub(z.re, x), z.im); }                                                         \
DEV C jl_mul(R x, C z) { return C(jl_mul(x, z.re), jl_mul(x, z.im)); }                                              \
DEV C jl_mul(C z, R x) { return C(jl_mul(z.re, x), jl_mul(z.im, x)); }                                              \
DEV C jl_div(C z, R x) { return C(jl_div(z.re, x), jl_div(z.im, x)); }                                              \
DEV R jl_abs2(C z) { return jl_add(jl_mul(z.re, z.re), jl_mul(z.im, z.im)); }
JL_CPLX_ARITH(jl_c64, float)
JL_CPLX_ARITH(jl_c128, double)
// ComplexF64 division: Baudin & Smith's robust algorithm with Julia's scaling of operands near the overflow / underflow thresholds
// (halve above floatmax/2; multiply by bs = 2/eps^2 = 2^105 below 2 floatmin/eps, so that subnormal operands are brought well inside the
// normal range and b*r cannot underflow again)
DEV double jl_cdiv2_(double a, double b, double c, double d, double r, double t) {
    if (r != 0.0) {
        const double br = __dmul_rn(b, r);
        return br != 0.0 ? __dmul_rn(__dadd_rn(a, br), t) : __dadd_rn(__dmul_rn(a, t), __dmul_rn(__dmul_rn(b, t), r));
    }
    return __dmul_rn(__dadd_rn(a, __dmul_rn(d, __ddiv_rn(b, c))), t);
}
DEV void jl_cdiv1_(double a, double b, double c, double d, double* p, double* q) {
    const double r = __ddiv_rn(d, c), t = __ddiv_rn(1.0, __dadd_rn(c, __dmul_rn(d, r)));
    *p = jl_cdiv2_(a, b, c, d, r, t);
    *q = jl_cdiv2_(b, -a, c, d, r, t);
}
DEV jl_c128 jl_div(jl_c128 z, jl_c128 w) {
    double a = z.re, b = z.im, c = w.re, d = w.im;
    const double ab = fmax(fabs(a), fabs(b)), cd = fmax(fabs(c), fabs(d));
    const double halfov = 0x1p1023, twoun = 0x1p-969, be = 0x1p105;   // floatmax/2, 2 floatmin/eps, 2/eps^2
    double s = 1.0;
    if (ab >= halfov) { a *= 0.5; b *= 0.5; s *= 2.0; }
    if (cd >= halfov) { c *= 0.5; d *= 0.5; s *= 0.5; }
    if (ab <= twoun) { a *= be; b *= be; s /= be; }
    if (cd <= twoun) { c *= be; d *= be; s *= be; }
    double p, q;
    if (fabs(d) <= fabs(c)) {
        jl_cdiv1_(a, b, c, d, &p, &q);
    } else {
        jl_cdiv1_(b, a, d, c, &p, &q);
        q = -q;
    }
    return jl_c128(__dmul_rn(p, s), __dmul_rn(q, s));
}
DEV jl_c128 jl_inv(jl_c128 w) { return jl_div(jl_c128(1.0, 0.0), w); }
// ComplexF32 / and inv: widened to ComplexF64 and rounded once, as Julia does
DEV jl_c64 jl_div(jl_c64 z, jl_c64 w) { return jl_c64(jl_div(jl_c128(z), jl_c128(w))); }
DEV jl_c64 jl_inv(jl_c64 w) { return jl_c64(jl_inv(jl_c128(w))); }
DEV jl_c64 jl_div(float x, jl_c64 z) { return jl_mul(x, jl_inv(z)); }
DEV jl_c128 jl_div(double x, jl_c128 z) { return jl_mul(x, jl_inv(z)); }
// abs = hypot: Float32 through exact Float64 squares, Float64 with CUDA's hypot (no intermediate overflow); Inf if a component is Inf
DEV float jl_abs(jl_c64 z) {
    if (isinf(z.re) || isinf(z.im)) return __int_as_float(0x7f800000);   // hypot(Inf, NaN) = Inf
    const double x = z.re, y = z.im;
    return (float)__dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
}
DEV double jl_abs(jl_c128 z) { return hypot(z.re, z.im); }
// angle(z) = atan(imag z, real z); angle(x::Real) = atan(0, x); cis(x) = Complex(cos x, sin x) (libdevice, <= 2 ulp)
DEV float jl_angle(jl_c64 z) { return atan2f(z.im, z.re); }
DEV double jl_angle(jl_c128 z) { return atan2(z.im, z.re); }
DEV float jl_angle(float x) { return atan2f(0.f, x); }
DEV double jl_angle(double x) { return atan2(0.0, x); }
DEV jl_c64 jl_cis(float x) { return jl_c64(cosf(x), sinf(x)); }
DEV jl_c128 jl_cis(double x) { return jl_c128(cos(x), sin(x)); }
)PRELUDE";

// Float16 values (jl_f16: the IEEE binary16 bits).  Julia defines Float16 arithmetic as "widen to Float32, operate, round to Float16"
// (base/float.jl); for + - * / and sqrt that IS the correctly rounded binary16 result (24 >= 2*11 + 2).  Math functions are
// Float16(f(Float32(x))), as Julia's Float16 methods.  Conversions are single PTX cvt instructions: Float64 -> Float16 rounds once
// (never through Float32); Int32 / Int64 values go through an exact or already-overflowing Float32.  Appended only to sources that use
// the type (an argument, output or value dtype, or the name in the expression), so every other generated kernel is byte-for-byte what it
// was; no toolkit header is needed.
const char* kPreludeF16 = R"PRELUDE(
struct __align__(2) jl_f16 {
    unsigned short b;
    jl_f16() = default;
    DEV jl_f16(float x) { asm("cvt.rn.f16.f32 %0, %1;" : "=h"(b) : "f"(x)); }
    DEV jl_f16(double x) { asm("cvt.rn.f16.f64 %0, %1;" : "=h"(b) : "d"(x)); }
    DEV jl_f16(int x) : jl_f16((float)x) {}   // exact below 2^24; larger values overflow to +-Inf either way
    DEV jl_f16(i64 x) : jl_f16((float)x) {}
    DEV jl_f16(bool x) : b(x ? 0x3c00 : 0) {}
    // Float32(x) / Float64(x): exact; a NaN keeps its sign and payload bits (the cvt instruction would return the canonical NaN)
    DEV explicit operator float() const {
        float f;
        asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(b));
        return (b & 0x7fff) > 0x7c00 ? __int_as_float(((unsigned)(b & 0x8000) << 16) | 0x7f800000u | ((unsigned)(b & 0x3ff) << 13)) : f;
    }
    DEV explicit operator double() const {
        double d;
        asm("cvt.f64.f16 %0, %1;" : "=d"(d) : "h"(b));
        return (b & 0x7fff) > 0x7c00 ? __longlong_as_double(((i64)(b & 0x8000) << 48) | 0x7ff0000000000000ll | ((i64)(b & 0x3ff) << 42)) : d;
    }
};
DEV jl_f16 jl_f16_bits(unsigned short b) { jl_f16 r; r.b = b; return r; }
// the operand of an arithmetic operation (its NaN results are canonical anyway)
DEV float jl_w(jl_f16 a) { float f; asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(a.b)); return f; }
DEV jl_f16 jl_add(jl_f16 a, jl_f16 b) { return jl_f16(__fadd_rn(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_sub(jl_f16 a, jl_f16 b) { return jl_f16(__fsub_rn(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_mul(jl_f16 a, jl_f16 b) { return jl_f16(__fmul_rn(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_div(jl_f16 a, jl_f16 b) { return jl_f16(__fdiv_rn(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_max(jl_f16 a, jl_f16 b) { return jl_f16(jl_max(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_min(jl_f16 a, jl_f16 b) { return jl_f16(jl_min(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_rem(jl_f16 a, jl_f16 b) { return jl_f16(jl_rem(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_mod(jl_f16 a, jl_f16 b) { return jl_f16(jl_mod(jl_w(a), jl_w(b))); }
DEV jl_f16 jl_pow(jl_f16 a, jl_f16 b) { return jl_f16(powf(jl_w(a), jl_w(b))); }
DEV bool jl_lt(jl_f16 a, jl_f16 b) { return jl_w(a) < jl_w(b); }
DEV bool jl_le(jl_f16 a, jl_f16 b) { return jl_w(a) <= jl_w(b); }
DEV bool jl_gt(jl_f16 a, jl_f16 b) { return jl_w(a) > jl_w(b); }
DEV bool jl_ge(jl_f16 a, jl_f16 b) { return jl_w(a) >= jl_w(b); }
DEV bool jl_eq(jl_f16 a, jl_f16 b) { return jl_w(a) == jl_w(b); }
DEV bool jl_ne(jl_f16 a, jl_f16 b) { return jl_w(a) != jl_w(b); }
DEV jl_f16 jl_neg(jl_f16 a) { return jl_f16_bits(a.b ^ 0x8000); }
DEV jl_f16 jl_abs(jl_f16 a) { return jl_f16_bits(a.b & 0x7fff); }
DEV jl_f16 jl_sqrt(jl_f16 a) { return jl_f16(__fsqrt_rn(jl_w(a))); }
DEV jl_f16 jl_inv(jl_f16 a) { return jl_f16(__fdiv_rn(1.0f, jl_w(a))); }
DEV jl_f16 jl_floor(jl_f16 a) { return jl_f16(floorf(jl_w(a))); }
DEV jl_f16 jl_ceil(jl_f16 a) { return jl_f16(ceilf(jl_w(a))); }
DEV jl_f16 jl_sign(jl_f16 a) { return jl_f16(jl_sign(jl_w(a))); }
DEV bool jl_isnan(jl_f16 a) { return (a.b & 0x7fff) > 0x7c00; }
DEV bool jl_isinf(jl_f16 a) { return (a.b & 0x7fff) == 0x7c00; }
DEV bool jl_isfinite(jl_f16 a) { return (a.b & 0x7c00) != 0x7c00; }
#define JL_H1(name) DEV jl_f16 jl_##name(jl_f16 a) { return jl_f16(jl_##name(jl_w(a))); }
JL_H1(sin) JL_H1(cos) JL_H1(tan) JL_H1(exp) JL_H1(exp2) JL_H1(log) JL_H1(log2) JL_H1(log10) JL_H1(tanh) JL_H1(sinh) JL_H1(cosh)
JL_H1(atan) JL_H1(asin) JL_H1(acos) JL_H1(expm1) JL_H1(log1p) JL_H1(cbrt)
DEV jl_f16 jl_angle(jl_f16 a) { return jl_f16(atan2f(0.f, jl_w(a))); }   // angle(x::Real) = atan(zero(x), x)
)PRELUDE";

// The Float16 methods of kPreludeExt's and kPreludeMethods' names, appended after those blocks when a source uses both.
const char* kPreludeF16Ext = R"PRELUDE(
JL_H1(x_asinh) JL_H1(x_acosh) JL_H1(x_atanh) JL_H1(x_exp10) JL_H1(x_sinpi) JL_H1(x_cospi) JL_H1(x_trunc) JL_H1(x_round)
JL_H1(x_erf) JL_H1(x_erfc) JL_H1(x_erfinv) JL_H1(x_erfcinv) JL_H1(x_erfcx) JL_H1(x_gamma) JL_H1(x_loggamma)
)PRELUDE";
const char* kPreludeF16Methods = R"PRELUDE(
DEV jl_f16 jl_m_copysign(jl_f16 a, jl_f16 b) { return jl_f16_bits((a.b & 0x7fff) | (b.b & 0x8000)); }
)PRELUDE";

bool uses_f16(const char* expr, int32_t dt0, int nargs, const int32_t* dts) {
    if (dt0 == DAB_F16) return true;
    for (int k = 0; k < nargs; ++k)
        if (dts[k] == DAB_F16) return true;
    return expr && strstr(expr, "jl_f16") != nullptr;
}

// the Float16 block and its companions for the blocks already in s
void append_f16(std::string& s, const char* expr) {
    s += kPreludeF16;
    if (mentions_ext(expr)) s += kPreludeF16Ext;
    if (mentions_methods(expr)) s += kPreludeF16Methods;
}

// elements per thread step of the linear kernel: 8 when an array argument or the output is Float16 (16-byte accesses), else 4
int lin_width(int32_t out_dt, int nargs, const int32_t* dts) {
    if (out_dt == DAB_F16) return 8;
    for (int k = 0; k < nargs; ++k)
        if (dts[k] == DAB_F16) return 8;
    return 4;
}

bool is_cplx_dt(int32_t dt) { return dt == DAB_C64 || dt == DAB_C128; }

bool uses_cplx(const char* expr, int32_t dt0, int nargs, const int32_t* dts) {
    if (is_cplx_dt(dt0)) return true;
    for (int k = 0; k < nargs; ++k)
        if (is_cplx_dt(dts[k])) return true;
    const char* names[] = {"jl_c64", "jl_c128", "jl_cis(", "jl_angle(", nullptr};
    for (int i = 0; expr && names[i]; ++i)
        if (strstr(expr, names[i])) return true;
    return false;
}

const char* ctype_of(int32_t dt) {
    switch (dt) {
        case DAB_F32: return "float";
        case DAB_F64: return "double";
        case DAB_I32: return "int";
        case DAB_I64: return "long long";
        case DAB_U8: return "bool";
        case DAB_C64: return "jl_c64";
        case DAB_C128: return "jl_c128";
        case DAB_F16: return "jl_f16";
        default: return nullptr;
    }
}

// value type of dab_mapreduce_expr: the array element types plus Int128
const char* vtype_of(int32_t dt) { return dt == DAB_I128 ? "i128" : ctype_of(dt); }

struct BcParamsHost {
    void* out;
    unsigned long long shape[4];
    long long ostr[4];
    const void* ptr[8];
    long long str[8][4];
    unsigned long long scalar[8];
};

struct Nvrtc {
    void* h = nullptr;
    nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
    const char* (*GetErrorString)(nvrtcResult) = nullptr;
    bool ok = false;
    char why[256] = "";
};

Nvrtc& nvrtc() {
    static Nvrtc api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    const char* names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", nullptr};
    for (int i = 0; names[i] && !api.h; ++i) api.h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
    if (!api.h) {
        snprintf(api.why, sizeof(api.why), "dlopen(libnvrtc.so.12) failed: %s", dlerror());
        return api;
    }
#define SYM(f, n)                                                                  \
    do {                                                                           \
        *(void**)(&api.f) = dlsym(api.h, n);                                       \
        if (!api.f) {                                                              \
            snprintf(api.why, sizeof(api.why), "libnvrtc lacks symbol %s", n);     \
            return api;                                                            \
        }                                                                          \
    } while (0)
    SYM(CreateProgram, "nvrtcCreateProgram");
    SYM(CompileProgram, "nvrtcCompileProgram");
    SYM(GetCUBINSize, "nvrtcGetCUBINSize");
    SYM(GetCUBIN, "nvrtcGetCUBIN");
    SYM(GetProgramLogSize, "nvrtcGetProgramLogSize");
    SYM(GetProgramLog, "nvrtcGetProgramLog");
    SYM(DestroyProgram, "nvrtcDestroyProgram");
    SYM(GetErrorString, "nvrtcGetErrorString");
#undef SYM
    api.ok = true;
    return api;
}

struct Driver {
    CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
    CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
    CUresult (*OccupancyMaxActiveBlocksPerMultiprocessor)(int*, CUfunction, int, size_t) = nullptr;
    CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
    bool ok = false;
    char why[256] = "";
};

Driver& driver() {
    static Driver d;
    static bool tried = false;
    if (tried) return d;
    tried = true;
#define ENTRY(f, n)                                                                                       \
    do {                                                                                                  \
        cudaDriverEntryPointQueryResult qr;                                                               \
        if (cudaGetDriverEntryPoint(n, (void**)&d.f, cudaEnableDefault, &qr) != cudaSuccess || !d.f) {    \
            cudaGetLastError();                                                                           \
            snprintf(d.why, sizeof(d.why), "driver entry point %s unavailable", n);                       \
            return d;                                                                                     \
        }                                                                                                 \
    } while (0)
    ENTRY(ModuleLoadData, "cuModuleLoadData");
    ENTRY(ModuleGetFunction, "cuModuleGetFunction");
    ENTRY(LaunchKernel, "cuLaunchKernel");
    ENTRY(OccupancyMaxActiveBlocksPerMultiprocessor, "cuOccupancyMaxActiveBlocksPerMultiprocessor");
    ENTRY(GetErrorString, "cuGetErrorString");
#undef ENTRY
    d.ok = true;
    return d;
}

struct Compiled {
    CUfunction linear = nullptr, general = nullptr, rows = nullptr;
    int occ_linear = 1, occ_general = 1, occ_rows = 1;
};

std::mutex g_mu;
std::unordered_map<std::string, Compiled> g_cache;

std::string build_source(const char* expr, int32_t out_dt, int nargs, const int32_t* dts, const bool* is_arr) {
    std::string s = kPrelude;
    if (mentions_ext(expr)) s += kPreludeExt;
    if (mentions_methods(expr)) s += kPreludeMethods;
    if (uses_cplx(expr, out_dt, nargs, dts)) s += kPreludeCplx;
    if (uses_f16(expr, out_dt, nargs, dts)) append_f16(s, expr);
    const std::string W = std::to_string(lin_width(out_dt, nargs, dts));   // "4" except in Float16 kernels
    s += "typedef ";
    s += ctype_of(out_dt);
    s += " OUT_T;\n";
    for (int k = 0; k < nargs; ++k) s += std::string("typedef ") + ctype_of(dts[k]) + " T" + std::to_string(k) + ";\n";
    s += "#define DAB_EXPR (";
    s += expr;
    s += ")\n";
    // ---- linear kernel: flat grid, one CTA per 2 x 256 vectors of W elements (4; 8 in Float16 kernels) (same shape as ew1_kernel, which beat
    // the persistent grid-stride form); the extra last CTA takes the remainder vectors and the scalar tail
    s += "extern \"C\" __global__ void __launch_bounds__(256) dab_bc_linear(BcParams p) {\n"
         "  const u64 n = p.shape[0] * p.shape[1] * p.shape[2] * p.shape[3];\n"
         "  const u64 nv = n / " + W + ";\n"
         "  const u64 ntiles = nv / 512;\n"
         "  OUT_T* o = (OUT_T*)p.out;\n";
    for (int k = 0; k < nargs; ++k) {
        std::string K = std::to_string(k);
        if (is_arr[k]) s += "  const T" + K + "* q" + K + " = (const T" + K + "*)p.ptr[" + K + "];\n";
        else s += "  const T" + K + " a" + K + " = bits_as<T" + K + ">(p.scalar[" + K + "]);\n";
    }
    s += "  if ((u64)blockIdx.x < ntiles) {\n"
         "    const u64 i0 = (u64)blockIdx.x * 512 + threadIdx.x;\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const VecN<T" + K + ", " + W + "> v" + K + "_0 = *(const VecN<T" + K + ", " + W + ">*)(q" + K + " + " + W + " * i0);\n";
            s += "    const VecN<T" + K + ", " + W + "> v" + K + "_1 = *(const VecN<T" + K + ", " + W + ">*)(q" + K + " + " + W + " * (i0 + 256));\n";
        }
    for (int u = 0; u < 2; ++u) {
        std::string U = std::to_string(u);
        s += "    { VecN<OUT_T, " + W + "> r;\n"
             "#pragma unroll\n"
             "      for (int j = 0; j < " + W + "; ++j) {\n";
        for (int k = 0; k < nargs; ++k)
            if (is_arr[k]) {
                std::string K = std::to_string(k);
                s += "        const T" + K + " a" + K + " = v" + K + "_" + U + ".v[j];\n";
            }
        s += "        r.v[j] = (OUT_T)DAB_EXPR;\n"
             "      }\n"
             "      *(VecN<OUT_T, " + W + ">*)(o + " + W + " * (i0 + " + std::to_string(256 * u) + ")) = r; }\n";
    }
    s += "    return;\n"
         "  }\n"
         "  for (u64 i = ntiles * 512 + threadIdx.x; i < nv; i += blockDim.x) {\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const VecN<T" + K + ", " + W + "> v" + K + " = *(const VecN<T" + K + ", " + W + ">*)(q" + K + " + " + W + " * i);\n";
        }
    s += "    VecN<OUT_T, " + W + "> r;\n"
         "#pragma unroll\n"
         "    for (int j = 0; j < " + W + "; ++j) {\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "      const T" + K + " a" + K + " = v" + K + ".v[j];\n";
        }
    s += "      r.v[j] = (OUT_T)DAB_EXPR;\n"
         "    }\n"
         "    *(VecN<OUT_T, " + W + ">*)(o + " + W + " * i) = r;\n"
         "  }\n"
         "  for (u64 i = nv * " + W + " + threadIdx.x; i < n; i += blockDim.x) {\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const T" + K + " a" + K + " = q" + K + "[i];\n";
        }
    s += "    o[i] = (OUT_T)DAB_EXPR;\n"
         "  }\n"
         "}\n";
    // ---- general (strided / extruded) kernel
    s += "extern \"C\" __global__ void __launch_bounds__(256) dab_bc_general(BcParams p) {\n"
         "  const u64 n0 = p.shape[0], n1 = p.shape[1], n2 = p.shape[2];\n"
         "  const u64 n = n0 * n1 * n2 * p.shape[3];\n"
         "  OUT_T* o = (OUT_T*)p.out;\n";
    for (int k = 0; k < nargs; ++k) {
        std::string K = std::to_string(k);
        if (is_arr[k]) s += "  const T" + K + "* q" + K + " = (const T" + K + "*)p.ptr[" + K + "];\n";
        else s += "  const T" + K + " a" + K + " = bits_as<T" + K + ">(p.scalar[" + K + "]);\n";
    }
    s += "  const u64 stride = (u64)gridDim.x * blockDim.x;\n"
         "  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {\n"
         "    const u64 i0 = i % n0, t0 = i / n0, i1 = t0 % n1, t1 = t0 / n1, i2 = t1 % n2, i3 = t1 / n2;\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const T" + K + " a" + K + " = q" + K + "[(i64)i0 * p.str[" + K + "][0] + (i64)i1 * p.str[" + K + "][1] + (i64)i2 * p.str[" + K +
                 "][2] + (i64)i3 * p.str[" + K + "][3]];\n";
        }
    s += "    o[(i64)i0 * p.ostr[0] + (i64)i1 * p.ostr[1] + (i64)i2 * p.ostr[2] + (i64)i3 * p.ostr[3]] = (OUT_T)DAB_EXPR;\n"
         "  }\n"
         "}\n";
    // ---- "rows" kernel: the destination is dense, every array argument is either dense along dim 0 (stride 1, 16-byte aligned
    // rows) or extruded along dim 0 (stride 0): each thread produces 4 consecutive elements of one row with vector accesses and
    // decomposes the index once per 4 elements.  Serves  a .- m  with a 1 x n  m,  a .* v  with a column vector v, ... (the
    // extrusion cases of reference src/broadcast.jl:103-120) at streaming speed.
    s += "extern \"C\" __global__ void __launch_bounds__(256) dab_bc_rows(BcParams p) {\n"
         "  const u64 n0v = p.shape[0] / 4, n1 = p.shape[1], n2 = p.shape[2];\n"
         "  const u64 total = n0v * n1 * n2 * p.shape[3];\n"
         "  OUT_T* o = (OUT_T*)p.out;\n";
    for (int k = 0; k < nargs; ++k) {
        std::string K = std::to_string(k);
        if (is_arr[k]) s += "  const T" + K + "* q" + K + " = (const T" + K + "*)p.ptr[" + K + "];\n  const bool d" + K + " = p.str[" + K + "][0] != 0;\n";
        else s += "  const T" + K + " a" + K + " = bits_as<T" + K + ">(p.scalar[" + K + "]);\n";
    }
    s += "  const u64 stride = (u64)gridDim.x * blockDim.x;\n"
         "  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {\n"
         "    const u64 i0 = (i % n0v) * 4, t0 = i / n0v, i1 = t0 % n1, t1 = t0 / n1, i2 = t1 % n2, i3 = t1 / n2;\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const i64 f" + K + " = (i64)i1 * p.str[" + K + "][1] + (i64)i2 * p.str[" + K + "][2] + (i64)i3 * p.str[" + K + "][3];\n";
            s += "    VecN<T" + K + ", 4> v" + K + ";\n";
            s += "    if (d" + K + ") v" + K + " = *(const VecN<T" + K + ", 4>*)(q" + K + " + f" + K + " + (i64)i0);\n";
            s += "    else { const T" + K + " b = q" + K + "[f" + K + "]; v" + K + ".v[0] = b; v" + K + ".v[1] = b; v" + K + ".v[2] = b; v" + K + ".v[3] = b; }\n";
        }
    s += "    VecN<OUT_T, 4> r;\n"
         "#pragma unroll\n"
         "    for (int j = 0; j < 4; ++j) {\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "      const T" + K + " a" + K + " = v" + K + ".v[j];\n";
        }
    s += "      r.v[j] = (OUT_T)DAB_EXPR;\n"
         "    }\n"
         "    *(VecN<OUT_T, 4>*)(o + (i64)i0 + (i64)i1 * p.ostr[1] + (i64)i2 * p.ostr[2] + (i64)i3 * p.ostr[3]) = r;\n"
         "  }\n"
         "}\n";
    return s;
}

int32_t compile_cubin(dab_ctx* ctx, const std::string& src, std::vector<char>* cubin_out, bool int128 = false) {
    Nvrtc& rt = nvrtc();
    if (!rt.ok) return dab_fail(ctx, DAB_ERR_NVRTC, "NVRTC unavailable: %s", rt.why);
    nvrtcProgram prog;
    nvrtcResult r = rt.CreateProgram(&prog, src.c_str(), "dab_broadcast.cu", 0, nullptr, nullptr);
    if (r != NVRTC_SUCCESS) return dab_fail(ctx, DAB_ERR_NVRTC, "nvrtcCreateProgram: %s", rt.GetErrorString(r));
    const char* opts[] = {"--gpu-architecture=sm_90a", "-fmad=false", "--std=c++17", "-lineinfo", "-default-device", "--device-int128"};
    r = rt.CompileProgram(prog, int128 ? 6 : 5, opts);
    if (r != NVRTC_SUCCESS) {
        size_t ls = 0;
        rt.GetProgramLogSize(prog, &ls);
        std::string log(ls + 1, '\0');
        if (ls) rt.GetProgramLog(prog, &log[0]);
        rt.DestroyProgram(&prog);
        if (log.size() > 400) log.resize(400);
        return dab_fail(ctx, DAB_ERR_NVRTC, "NVRTC compile failed (%s): %s", rt.GetErrorString(r), log.c_str());
    }
    size_t cs = 0;
    rt.GetCUBINSize(prog, &cs);
    cubin_out->resize(cs);
    rt.GetCUBIN(prog, cubin_out->data());
    rt.DestroyProgram(&prog);
    return DAB_OK;
}

int32_t compile(dab_ctx* ctx, const std::string& src, Compiled* out) {
    Driver& drv = driver();
    if (!drv.ok) return dab_fail(ctx, DAB_ERR_NVRTC, "CUDA driver API unavailable: %s", drv.why);
    std::vector<char> cubin;
    int32_t st = compile_cubin(ctx, src, &cubin);
    if (st != DAB_OK) return st;
    CUmodule mod;
    CUresult cr = drv.ModuleLoadData(&mod, cubin.data());
    if (cr != CUDA_SUCCESS) {
        const char* es = "?";
        drv.GetErrorString(cr, &es);
        return dab_fail(ctx, DAB_ERR_NVRTC, "cuModuleLoadData failed: %s", es);
    }
    if (drv.ModuleGetFunction(&out->linear, mod, "dab_bc_linear") != CUDA_SUCCESS ||
        drv.ModuleGetFunction(&out->general, mod, "dab_bc_general") != CUDA_SUCCESS ||
        drv.ModuleGetFunction(&out->rows, mod, "dab_bc_rows") != CUDA_SUCCESS)
        return dab_fail(ctx, DAB_ERR_NVRTC, "cuModuleGetFunction failed");
    if (drv.OccupancyMaxActiveBlocksPerMultiprocessor(&out->occ_rows, out->rows, 256, 0) != CUDA_SUCCESS || out->occ_rows < 1) out->occ_rows = 1;
    if (drv.OccupancyMaxActiveBlocksPerMultiprocessor(&out->occ_linear, out->linear, 256, 0) != CUDA_SUCCESS || out->occ_linear < 1)
        out->occ_linear = 1;
    if (drv.OccupancyMaxActiveBlocksPerMultiprocessor(&out->occ_general, out->general, 256, 0) != CUDA_SUCCESS || out->occ_general < 1)
        out->occ_general = 1;
    return DAB_OK;
}


// ------------------------------------------------------------------------------------------------------------------------------
// Fused map + reduce for an arbitrary traced expression:  mapreduce(f, op, args...)  on one localpart in ONE pass over HBM
// (reference src/mapreduce.jl:31 with a general closure f; also dot = mapreduce(*, +, x, y), isequal = all(x .== y), ...).
// Same structure as the hand-written reduce_kernel: flat grid, 2 x 16/32-byte vector loads per argument in flight, 8-value tree in
// the value type, wide (fp64 / int64) carrier, one partial per CTA; a second tiny launch folds the <= 16384 partials in a fixed
// order (deterministic) and writes the 16-byte result slot.
struct MrSpec {
    const char *tile_t, *acc_t, *out_t, *tile_comb, *acc_comb, *acc_id;
};

bool mr_spec(int32_t val_dt, int32_t op, MrSpec* sp) {
    const bool flt = val_dt == DAB_F32 || val_dt == DAB_F64, boolean = val_dt == DAB_U8;
    const char* vt = vtype_of(val_dt);
    if (val_dt == DAB_I128) {  // tile, carrier and result are all Int128; + and * wrap, so any grouping gives the same bits
        switch (op) {
            case DAB_SUM: *sp = {vt, vt, vt, "jl_add(a, b)", "jl_add(a, b)", "0"}; return true;
            case DAB_PROD: *sp = {vt, vt, vt, "jl_mul(a, b)", "jl_mul(a, b)", "1"}; return true;
            case DAB_MAX: *sp = {vt, vt, vt, "jl_max(a, b)", "jl_max(a, b)", "((u128)1 << 127)"}; return true;
            case DAB_MIN: *sp = {vt, vt, vt, "jl_min(a, b)", "jl_min(a, b)", "(~((u128)1 << 127))"}; return true;
            default: return false;
        }
    }
    if (val_dt == DAB_F16) {  // Float16 values: Float32 tile (exact widening), fp64 carrier, one rounding to Float16 (the slot's first 2 bytes)
        switch (op) {
            case DAB_SUM: *sp = {"float", "double", vt, "jl_add(a, b)", "jl_add(a, b)", "0.0"}; return true;
            case DAB_PROD: *sp = {"float", "double", vt, "jl_mul(a, b)", "jl_mul(a, b)", "1.0"}; return true;
            case DAB_MAX: *sp = {"float", "float", vt, "jl_max(a, b)", "jl_max(a, b)", "(-__int_as_float(0x7f800000))"}; return true;
            case DAB_MIN: *sp = {"float", "float", vt, "jl_min(a, b)", "jl_min(a, b)", "__int_as_float(0x7f800000)"}; return true;
            default: return false;
        }
    }
    if (is_cplx_dt(val_dt)) {  // complex fp64 carrier; sums add componentwise in the value type inside a tile, products widen first
        const char* out = val_dt == DAB_C64 ? "jl_c64_slot" : "jl_c128";
        switch (op) {
            case DAB_SUM: *sp = {vt, "jl_c128", out, "jl_add(a, b)", "jl_add(a, b)", "jl_c128(0.0, 0.0)"}; return true;
            case DAB_PROD: *sp = {"jl_c128", "jl_c128", out, "jl_mul(a, b)", "jl_mul(a, b)", "jl_c128(1.0, 0.0)"}; return true;
            default: return false;
        }
    }
    switch (op) {
        case DAB_SUM:
        case DAB_COUNT:
            if (op == DAB_COUNT && !boolean) return false;
            if (flt) *sp = {vt, "double", vt, "jl_add(a, b)", "jl_add(a, b)", "0.0"};
            else if (boolean) *sp = {"int", "long long", "long long", "(a + b)", "jl_add(a, b)", "0ll"};
            else *sp = {"long long", "long long", "long long", "jl_add(a, b)", "jl_add(a, b)", "0ll"};
            return true;
        case DAB_PROD:
            if (boolean) return false;
            if (flt) *sp = {vt, "double", vt, "jl_mul(a, b)", "jl_mul(a, b)", "1.0"};
            else *sp = {"long long", "long long", "long long", "jl_mul(a, b)", "jl_mul(a, b)", "1ll"};
            return true;
        case DAB_MAX:
        case DAB_MIN: {
            if (boolean) return false;
            const bool mx = op == DAB_MAX;
            const char* id = val_dt == DAB_F32   ? (mx ? "(-__int_as_float(0x7f800000))" : "__int_as_float(0x7f800000)")
                             : val_dt == DAB_F64 ? (mx ? "(-__longlong_as_double(0x7ff0000000000000ll))" : "__longlong_as_double(0x7ff0000000000000ll)")
                             : val_dt == DAB_I32 ? (mx ? "((int)0x80000000)" : "0x7fffffff")
                                                 : (mx ? "((long long)0x8000000000000000ll)" : "0x7fffffffffffffffll");
            *sp = {vt, vt, vt, mx ? "jl_max(a, b)" : "jl_min(a, b)", mx ? "jl_max(a, b)" : "jl_min(a, b)", id};
            return true;
        }
        case DAB_ALL:
        case DAB_ANY:
            if (!boolean) return false;
            *sp = {"int", "long long", "long long", "(a + b)", "jl_add(a, b)", "0ll"};
            return true;
        default: return false;
    }
}

struct MrParamsHost {
    const void* ptr[8];
    unsigned long long scalar[8];
    unsigned long long n;
    void* partials;
    int tiles_per_cta;
};
struct MrFinalHost {
    const void* partials;
    void* out;
    long long n;
    unsigned int nparts;
    int mode;
};

std::string build_mr_source(const char* expr, int32_t val_dt, int32_t op, int nargs, const int32_t* dts, const bool* is_arr, const MrSpec& sp) {
    std::string s = kPrelude;
    if (val_dt == DAB_I128 || mentions_i128(expr)) s += kPreludeI128;
    if (mentions_ext(expr)) s += kPreludeExt;
    if (mentions_methods(expr)) s += kPreludeMethods;
    if (uses_cplx(expr, val_dt, nargs, dts)) s += kPreludeCplx;
    if (uses_f16(expr, val_dt, nargs, dts)) append_f16(s, expr);
    if (val_dt == DAB_I128 || is_cplx_dt(val_dt)) s += "#define DAB_ACC16 1\n";   // 16-byte carrier: shuffles and the result slot move four words
    s += std::string("typedef ") + vtype_of(val_dt) + " VAL_T;\n";
    for (int k = 0; k < nargs; ++k) s += std::string("typedef ") + ctype_of(dts[k]) + " T" + std::to_string(k) + ";\n";
    s += std::string("typedef ") + sp.tile_t + " TILE_T;\ntypedef " + sp.acc_t + " ACC_T;\ntypedef " + sp.out_t + " OUT_T;\n";
    s += "#define DAB_EXPR (";
    s += expr;
    s += ")\n";
    s += std::string("DEV TILE_T tile_comb(TILE_T a, TILE_T b) { return ") + sp.tile_comb + "; }\n";
    s += std::string("DEV ACC_T acc_comb(ACC_T a, ACC_T b) { return ") + sp.acc_comb + "; }\n";
    s += std::string("#define ACC_ID ((ACC_T)") + sp.acc_id + ")\n";
    s += R"MR(
struct MrParams { const void* ptr[8]; u64 scalar[8]; u64 n; void* partials; int tiles_per_cta; };
struct MrFinal { const void* partials; void* out; i64 n; unsigned int nparts; int mode; };
DEV ACC_T acc_shfl(ACC_T v, int d) {
#ifdef DAB_ACC16
    int w[4]; memcpy(w, &v, 16);
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = __shfl_down_sync(0xffffffffu, w[k], d);
    ACC_T r; memcpy(&r, w, 16); return r;
#else
    if (sizeof(ACC_T) == 8) {
        i64 x; memcpy(&x, &v, 8);
        int lo = __shfl_down_sync(0xffffffffu, (int)(x & 0xffffffffll), d), hi = __shfl_down_sync(0xffffffffu, (int)(x >> 32), d);
        x = ((i64)hi << 32) | (unsigned int)lo;
        ACC_T r; memcpy(&r, &x, 8); return r;
    } else {
        int x = 0; memcpy(&x, &v, sizeof(ACC_T));
        x = __shfl_down_sync(0xffffffffu, x, d);
        ACC_T r; memcpy(&r, &x, sizeof(ACC_T)); return r;
    }
#endif
}
DEV ACC_T block_reduce(ACC_T acc, ACC_T* smem) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc = acc_comb(acc, acc_shfl(acc, d));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) smem[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < 8 ? smem[lane] : ACC_ID;
#pragma unroll
        for (int d = 4; d > 0; d >>= 1) acc = acc_comb(acc, acc_shfl(acc, d));
    }
    return acc;
}
extern "C" __global__ void __launch_bounds__(256) dab_mr_final(MrFinal p) {
    __shared__ ACC_T smem[8];
    const ACC_T* parts = (const ACC_T*)p.partials;
    ACC_T acc = ACC_ID;
    unsigned int i = threadIdx.x;
    for (; i + 768 < p.nparts; i += 1024) {   // 4 independent loads in flight
        ACC_T a0 = parts[i], a1 = parts[i + 256], a2 = parts[i + 512], a3 = parts[i + 768];
        acc = acc_comb(acc, acc_comb(acc_comb(a0, a1), acc_comb(a2, a3)));
    }
    for (; i < p.nparts; i += 256) acc = acc_comb(acc, parts[i]);
    acc = block_reduce(acc, smem);
    if (threadIdx.x == 0) {
        OUT_T res;
        if (p.mode == 1) res = (OUT_T)(acc == (ACC_T)p.n);
        else if (p.mode == 2) res = (OUT_T)(acc != (ACC_T)0);
        else res = (OUT_T)acc;
#ifdef DAB_ACC16
        memcpy(p.out, &res, 16);
#else
        u64 w0 = 0, w1 = 0;
        memcpy(&w0, &res, sizeof(OUT_T));
        memcpy(&w1, &acc, sizeof(ACC_T));
        ((u64*)p.out)[0] = w0;
        ((u64*)p.out)[1] = w1;
#endif
    }
}
)MR";
    // ---- partial kernel: tiles of 2 x 256 vectors of W elements (4; 8 in Float16 kernels, 16-byte accesses)
    const int wi = lin_width(DAB_F32, nargs, dts);
    const std::string W = std::to_string(wi), W2 = std::to_string(2 * wi), WT = std::to_string(512 * wi);
    s += "extern \"C\" __global__ void __launch_bounds__(256) dab_mr_partial(MrParams p) {\n"
         "  __shared__ ACC_T smem[8];\n"
         "  const u64 n = p.n, nv = n / " + W + ", ntiles = nv / 512;\n";
    for (int k = 0; k < nargs; ++k) {
        std::string K = std::to_string(k);
        if (is_arr[k]) s += "  const T" + K + "* q" + K + " = (const T" + K + "*)p.ptr[" + K + "];\n";
        else s += "  const T" + K + " a" + K + " = bits_as<T" + K + ">(p.scalar[" + K + "]);\n";
    }
    s += "  ACC_T acc = ACC_ID;\n"
         "  u64 t_end = ((u64)blockIdx.x + 1) * (u64)p.tiles_per_cta;\n"
         "  if (t_end > ntiles) t_end = ntiles;\n"
         "#pragma unroll 1\n"
         "  for (u64 t = (u64)blockIdx.x * (u64)p.tiles_per_cta; t < t_end; ++t) {\n"
         "    const u64 i0 = t * 512 + threadIdx.x;\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "    const VecN<T" + K + ", " + W + "> v" + K + "_0 = *(const VecN<T" + K + ", " + W + ">*)(q" + K + " + " + W + " * i0);\n";
            s += "    const VecN<T" + K + ", " + W + "> v" + K + "_1 = *(const VecN<T" + K + ", " + W + ">*)(q" + K + " + " + W + " * (i0 + 256));\n";
        }
    s += "    TILE_T m[" + W2 + "];\n";
    for (int u = 0; u < 2; ++u) {
        std::string U = std::to_string(u);
        s += "#pragma unroll\n    for (int j = 0; j < " + W + "; ++j) {\n";
        for (int k = 0; k < nargs; ++k)
            if (is_arr[k]) {
                std::string K = std::to_string(k);
                s += "      const T" + K + " a" + K + " = v" + K + "_" + U + ".v[j];\n";
            }
        s += "      m[" + std::to_string(wi * u) + " + j] = (TILE_T)((VAL_T)DAB_EXPR);\n    }\n";
    }
    s += "#pragma unroll\n"
         "    for (int w = " + W2 + "; w > 1; w >>= 1)\n"
         "#pragma unroll\n"
         "      for (int k = 0; k < w / 2; ++k) m[k] = tile_comb(m[k], m[k + w / 2]);\n"
         "    acc = acc_comb(acc, (ACC_T)m[0]);\n"
         "  }\n"
         "  if (blockIdx.x == gridDim.x - 1) {\n"
         "    for (u64 i = ntiles * " + WT + " + threadIdx.x; i < n; i += blockDim.x) {\n";
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k]) {
            std::string K = std::to_string(k);
            s += "      const T" + K + " a" + K + " = q" + K + "[i];\n";
        }
    s += "      acc = acc_comb(acc, (ACC_T)(TILE_T)((VAL_T)DAB_EXPR));\n"
         "    }\n"
         "  }\n"
         "  acc = block_reduce(acc, smem);\n"
         "  if (threadIdx.x == 0) ((ACC_T*)p.partials)[blockIdx.x] = acc;\n"
         "}\n";
    return s;
}

struct CompiledMr {
    CUfunction partial = nullptr, final_ = nullptr;
};
std::unordered_map<std::string, CompiledMr> g_mr_cache;

}  // namespace

extern "C" {

// Diagnostic (no GPU needed): run the same source generation + NVRTC compilation as dab_broadcast_expr and report the size
// of the sm_90a cubin.  Lets the host-side tests validate the tracer's code generation on a CPU-only machine.
int32_t dab_jit_compile_check(const char* expr, int32_t out_dtype, int32_t nargs, const int32_t* arg_dtypes,
                              const int32_t* arg_is_array, size_t* cubin_bytes) {
    if (!expr || !ctype_of(out_dtype) || nargs < 0 || nargs > 8 || (nargs && (!arg_dtypes || !arg_is_array)))
        return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_compile_check: bad argument");
    bool is_arr[8] = {false};
    for (int k = 0; k < nargs; ++k) {
        if (!ctype_of(arg_dtypes[k])) return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_compile_check: bad dtype of arg %d", k);
        is_arr[k] = arg_is_array[k] != 0;
        if (!is_arr[k] && arg_dtypes[k] == DAB_C128) return dab_fail(nullptr, DAB_ERR_ARG, "a ComplexF64 scalar does not fit the 8-byte scalar slot of arg %d (pass complex(re, im) of two Float64 scalars)", k);
    }
    std::vector<char> cubin;
    int32_t st = compile_cubin(nullptr, build_source(expr, out_dtype, nargs, arg_dtypes, is_arr), &cubin);
    if (st != DAB_OK) return st;
    if (cubin_bytes) *cubin_bytes = cubin.size();
    return DAB_OK;
}

int32_t dab_broadcast_expr(dab_ctx* ctx, const char* expr, int32_t out_dtype, void* out, const size_t shape[4],
                           const size_t out_strides[4], int32_t nargs, const int32_t* arg_dtypes, const void* const* arg_ptrs,
                           const size_t* arg_strides, const uint64_t* arg_scalars) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, expr && out && shape && out_strides, DAB_ERR_ARG, "dab_broadcast_expr: null pointer");
    DAB_REQUIRE(ctx, nargs >= 0 && nargs <= 8, DAB_ERR_ARG, "dab_broadcast_expr: nargs %d (max 8)", nargs);
    DAB_REQUIRE(ctx, ctype_of(out_dtype), DAB_ERR_ARG, "dab_broadcast_expr: bad out dtype %d", out_dtype);
    DAB_REQUIRE(ctx, nargs == 0 || (arg_dtypes && arg_ptrs && arg_strides && arg_scalars), DAB_ERR_ARG, "dab_broadcast_expr: null arg table");
    size_t n = shape[0] * shape[1] * shape[2] * shape[3];
    if (n == 0) return DAB_OK;
    bool is_arr[8] = {false};
    std::string key = std::to_string(ctx->device) + "|" + std::to_string(out_dtype) + "|";
    for (int k = 0; k < nargs; ++k) {
        DAB_REQUIRE(ctx, ctype_of(arg_dtypes[k]), DAB_ERR_ARG, "dab_broadcast_expr: bad dtype of arg %d", k);
        is_arr[k] = arg_ptrs[k] != nullptr;
        DAB_REQUIRE(ctx, is_arr[k] || arg_dtypes[k] != DAB_C128, DAB_ERR_ARG, "dab_broadcast_expr: a ComplexF64 scalar does not fit the 8-byte scalar slot of arg %d (pass complex(re, im) of two Float64 scalars)", k);
        key += std::to_string(arg_dtypes[k]) + (is_arr[k] ? "a" : "s");
    }
    key += "|";
    key += expr;
    Compiled comp;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_cache.find(key);
        if (it == g_cache.end()) {
            DAB_CUDA(ctx, cudaFree(0));  // make sure the primary context is current for the driver calls
            int32_t st = compile(ctx, build_source(expr, out_dtype, nargs, arg_dtypes, is_arr), &comp);
            if (st != DAB_OK) return st;
            g_cache[key] = comp;
        } else {
            comp = it->second;
        }
    }
    BcParamsHost p;
    memset(&p, 0, sizeof(p));
    p.out = out;
    size_t dense[4], acc = 1;
    for (int d = 0; d < 4; ++d) {
        p.shape[d] = shape[d];
        p.ostr[d] = (long long)out_strides[d];
        dense[d] = acc;
        acc *= shape[d];
    }
    bool linear = true;
    for (int d = 0; d < 4; ++d)
        if (shape[d] > 1 && out_strides[d] != dense[d]) linear = false;
    const size_t lw = (size_t)lin_width(out_dtype, nargs, arg_dtypes);   // elements per vector of the linear kernel
    if ((uintptr_t)out % (lw * dab_dtype_size(out_dtype))) linear = false;
    for (int k = 0; k < nargs; ++k) {
        p.ptr[k] = arg_ptrs[k];
        p.scalar[k] = arg_scalars[k];
        for (int d = 0; d < 4; ++d) {
            p.str[k][d] = (long long)arg_strides[4 * k + d];
            if (is_arr[k] && shape[d] > 1 && arg_strides[4 * k + d] != dense[d]) linear = false;
        }
        if (is_arr[k] && ((uintptr_t)arg_ptrs[k] % (lw * dab_dtype_size(arg_dtypes[k])))) linear = false;
    }
    // rows kernel: dense destination, 4 | shape[0], every array argument dense-along-dim-0 with 4-element-aligned rows, or extruded
    bool rows = !linear && shape[0] % 4 == 0 && out_strides[0] == 1 && ((uintptr_t)out % (4 * dab_dtype_size(out_dtype))) == 0;
    for (int d = 1; d < 4 && rows; ++d)
        if (shape[d] > 1 && out_strides[d] % 4) rows = false;
    for (int k = 0; k < nargs && rows; ++k) {
        if (!is_arr[k]) continue;
        if (arg_strides[4 * k] == 0) continue;  // extruded along dim 0: scalar load per row
        if (arg_strides[4 * k] != 1 || ((uintptr_t)arg_ptrs[k] % (4 * dab_dtype_size(arg_dtypes[k])))) rows = false;
        for (int d = 1; d < 4 && rows; ++d)
            if (shape[d] > 1 && arg_strides[4 * k + d] % 4) rows = false;
    }
    Driver& drv = driver();
    void* args[] = {&p};
    CUfunction fn = linear ? comp.linear : (rows ? comp.rows : comp.general);
    size_t work = rows ? (n / 4 + 255) / 256 : (n + 255) / 256;
    size_t grid = linear ? (n / lw) / 512 + 1 : (size_t)dab_grid_for(ctx, work, rows ? comp.occ_rows : comp.occ_general);
    if (grid > 0x7fffffffull) return dab_fail(ctx, DAB_ERR_ARG, "array too large for one launch");
    CUresult cr = drv.LaunchKernel(fn, (unsigned)grid, 1, 1, 256, 1, 1, 0, (CUstream)ctx->stream, args, nullptr);
    if (cr != CUDA_SUCCESS) {
        const char* es = "?";
        drv.GetErrorString(cr, &es);
        return dab_fail(ctx, DAB_ERR_CUDA, "cuLaunchKernel failed: %s", es);
    }
    ctx->launches++;
    return DAB_OK;
}


int32_t dab_mapreduce_expr(dab_ctx* ctx, const char* expr, int32_t val_dtype, int32_t op, size_t n, int32_t nargs, const int32_t* arg_dtypes,
                           const void* const* arg_ptrs, const uint64_t* arg_scalars, void* out_dev) {
    DAB_ENTER(ctx);
    DAB_REQUIRE(ctx, expr && out_dev, DAB_ERR_ARG, "dab_mapreduce_expr: null pointer");
    DAB_REQUIRE(ctx, nargs >= 1 && nargs <= 8 && arg_dtypes && arg_ptrs && arg_scalars, DAB_ERR_ARG, "dab_mapreduce_expr: bad argument table");
    DAB_REQUIRE(ctx, vtype_of(val_dtype), DAB_ERR_ARG, "dab_mapreduce_expr: bad value dtype %d", val_dtype);
    DAB_REQUIRE(ctx, n > 0, DAB_ERR_EMPTY, "dab_mapreduce_expr: empty input (the host runtime handles n == 0)");
    MrSpec sp;
    if (!mr_spec(val_dtype, op, &sp))
        return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "mapreduce op %d on value dtype %d is not served (no host fallback)", op, val_dtype);
    bool is_arr[8] = {false};
    bool vec_ok = true;
    std::string key = "mr|" + std::to_string(ctx->device) + "|" + std::to_string(val_dtype) + "|" + std::to_string(op) + "|";
    for (int k = 0; k < nargs; ++k) {
        DAB_REQUIRE(ctx, ctype_of(arg_dtypes[k]), DAB_ERR_ARG, "dab_mapreduce_expr: bad dtype of arg %d", k);
        is_arr[k] = arg_ptrs[k] != nullptr;
        DAB_REQUIRE(ctx, is_arr[k] || arg_dtypes[k] != DAB_C128, DAB_ERR_ARG, "dab_mapreduce_expr: a ComplexF64 scalar does not fit the 8-byte scalar slot of arg %d (pass complex(re, im) of two Float64 scalars)", k);
        key += std::to_string(arg_dtypes[k]) + (is_arr[k] ? "a" : "s");
    }
    const size_t lw = (size_t)lin_width(DAB_F32, nargs, arg_dtypes);   // elements per vector of the partial kernel (8 with Float16 arguments)
    for (int k = 0; k < nargs; ++k)
        if (is_arr[k] && ((uintptr_t)arg_ptrs[k] % (lw * dab_dtype_size(arg_dtypes[k])))) vec_ok = false;
    if (!vec_ok) return dab_fail(ctx, DAB_ERR_UNSUPPORTED, "dab_mapreduce_expr: arguments must be aligned to %d elements", (int)lw);
    key += "|";
    key += expr;
    CompiledMr comp;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_mr_cache.find(key);
        if (it == g_mr_cache.end()) {
            DAB_CUDA(ctx, cudaFree(0));
            Driver& drv = driver();
            if (!drv.ok) return dab_fail(ctx, DAB_ERR_NVRTC, "CUDA driver API unavailable: %s", drv.why);
            std::vector<char> cubin;
            int32_t st = compile_cubin(ctx, build_mr_source(expr, val_dtype, op, nargs, arg_dtypes, is_arr, sp), &cubin,
                                       val_dtype == DAB_I128 || mentions_i128(expr));
            if (st != DAB_OK) return st;
            CUmodule mod;
            if (drv.ModuleLoadData(&mod, cubin.data()) != CUDA_SUCCESS) return dab_fail(ctx, DAB_ERR_NVRTC, "cuModuleLoadData failed");
            if (drv.ModuleGetFunction(&comp.partial, mod, "dab_mr_partial") != CUDA_SUCCESS ||
                drv.ModuleGetFunction(&comp.final_, mod, "dab_mr_final") != CUDA_SUCCESS)
                return dab_fail(ctx, DAB_ERR_NVRTC, "cuModuleGetFunction failed");
            g_mr_cache[key] = comp;
        } else {
            comp = it->second;
        }
    }
    const size_t ntiles = (n / lw) / 512;
    size_t k = 2;
    const size_t max_parts = 16384;
    if ((ntiles + k - 1) / k > max_parts) k = (ntiles + max_parts - 1) / max_parts;
    size_t grid = (ntiles + k - 1) / k;
    if (grid < 1) grid = 1;
    MrParamsHost p;
    memset(&p, 0, sizeof(p));
    for (int a = 0; a < nargs; ++a) {
        p.ptr[a] = arg_ptrs[a];
        p.scalar[a] = arg_scalars[a];
    }
    p.n = n;
    p.partials = ctx->block_partials;
    p.tiles_per_cta = (int)k;
    MrFinalHost f;
    f.partials = ctx->block_partials;
    f.out = out_dev;
    f.n = (long long)n;
    f.nparts = (unsigned int)grid;
    f.mode = op == DAB_ALL ? 1 : (op == DAB_ANY ? 2 : 0);
    Driver& drv = driver();
    void* a1[] = {&p};
    void* a2[] = {&f};
    if (drv.LaunchKernel(comp.partial, (unsigned)grid, 1, 1, 256, 1, 1, 0, (CUstream)ctx->stream, a1, nullptr) != CUDA_SUCCESS ||
        drv.LaunchKernel(comp.final_, 1, 1, 1, 256, 1, 1, 0, (CUstream)ctx->stream, a2, nullptr) != CUDA_SUCCESS)
        return dab_fail(ctx, DAB_ERR_CUDA, "cuLaunchKernel failed (dab_mapreduce_expr)");
    ctx->launches += 2;
    return DAB_OK;
}

// Diagnostic (no GPU, no NVRTC): the generated source itself -- kind 0 the broadcast kernels of dab_broadcast_expr (dtype = output type),
// kind 1 the fused map + reduce kernels of dab_mapreduce_expr (dtype = value type, op).  Copies at most cap bytes to buf and the full
// length to *len; lets the tests pin the sources of existing expressions byte for byte.
int32_t dab_jit_source(int32_t kind, const char* expr, int32_t dtype, int32_t op, int32_t nargs, const int32_t* arg_dtypes,
                       const int32_t* arg_is_array, char* buf, size_t cap, size_t* len) {
    if (!expr || !len || nargs < 0 || nargs > 8 || (nargs && (!arg_dtypes || !arg_is_array)) || (kind != 0 && kind != 1))
        return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_source: bad argument");
    bool is_arr[8] = {false};
    for (int k = 0; k < nargs; ++k) {
        if (!ctype_of(arg_dtypes[k])) return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_source: bad dtype of arg %d", k);
        is_arr[k] = arg_is_array[k] != 0;
    }
    std::string src;
    if (kind == 0) {
        if (!ctype_of(dtype)) return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_source: bad out dtype %d", dtype);
        src = build_source(expr, dtype, nargs, arg_dtypes, is_arr);
    } else {
        MrSpec sp;
        if (!vtype_of(dtype) || !mr_spec(dtype, op, &sp)) return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "op %d on value dtype %d not served", op, dtype);
        src = build_mr_source(expr, dtype, op, nargs, arg_dtypes, is_arr, sp);
    }
    *len = src.size();
    if (buf && cap) memcpy(buf, src.data(), src.size() < cap ? src.size() : cap);
    return DAB_OK;
}

// Diagnostic twin of dab_jit_compile_check for the fused map+reduce kernels.
int32_t dab_jit_compile_check_reduce(const char* expr, int32_t val_dtype, int32_t op, int32_t nargs, const int32_t* arg_dtypes,
                                     const int32_t* arg_is_array, size_t* cubin_bytes) {
    if (!expr || !vtype_of(val_dtype) || nargs < 1 || nargs > 8 || !arg_dtypes || !arg_is_array)
        return dab_fail(nullptr, DAB_ERR_ARG, "dab_jit_compile_check_reduce: bad argument");
    MrSpec sp;
    if (!mr_spec(val_dtype, op, &sp)) return dab_fail(nullptr, DAB_ERR_UNSUPPORTED, "op %d on value dtype %d not served", op, val_dtype);
    bool is_arr[8] = {false};
    for (int k = 0; k < nargs; ++k) {
        if (!ctype_of(arg_dtypes[k])) return dab_fail(nullptr, DAB_ERR_ARG, "bad dtype of arg %d", k);
        is_arr[k] = arg_is_array[k] != 0;
        if (!is_arr[k] && arg_dtypes[k] == DAB_C128) return dab_fail(nullptr, DAB_ERR_ARG, "a ComplexF64 scalar does not fit the 8-byte scalar slot of arg %d (pass complex(re, im) of two Float64 scalars)", k);
    }
    std::vector<char> cubin;
    int32_t st = compile_cubin(nullptr, build_mr_source(expr, val_dtype, op, nargs, arg_dtypes, is_arr, sp), &cubin,
                               val_dtype == DAB_I128 || mentions_i128(expr));
    if (st != DAB_OK) return st;
    if (cubin_bytes) *cubin_bytes = cubin.size();
    return DAB_OK;
}

}  // extern "C"
