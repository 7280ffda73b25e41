"""CPU-only: the source generated for the fused map+reduce kernels (dab_mapreduce_expr) compiles with NVRTC for sm_90a for every
(op, value type) combination the host runtime can request, and unsupported combinations are refused, not silently served."""
import ctypes as C

import numpy as np
import pytest


def _check(dab, f, tags, op, arrays=None):
    from darray_b200 import _lib
    from darray_b200._broadcast import codegen, trace

    code = {"f32": 0, "f64": 1, "i32": 2, "i64": 3, "bool": 4}
    e = trace(f, tags)
    n = len(tags)
    dts = (C.c_int32 * n)(*[code[t] for t in tags])
    arr = (C.c_int32 * n)(*(arrays or [1] * n))
    sz = C.c_size_t()
    L = _lib.lib()
    st = L.dab_jit_compile_check_reduce(codegen(e).encode(), code[e.jt], op, n, dts, arr, C.byref(sz))
    return st, sz.value, (L.dab_last_error(None) or b"").decode()[:300]


def test_fused_mapreduce_codegen_compiles(dab):
    from darray_b200 import _lib, sqrt

    cases = [(lambda a, b: a * b, ["f32", "f32"], _lib.SUM), (lambda a, b: a * b, ["f64", "f64"], _lib.SUM),
             (lambda x: x ** 2 + 2 * x - 1, ["i64"], _lib.SUM), (lambda x: 2 * x, ["i32"], _lib.PROD), (lambda x: sqrt(x) * x + 1, ["f32"], _lib.SUM),
             (lambda a, b: a == b, ["f64", "f64"], _lib.ALL), (lambda v: (v > 0.25) & (v < 0.5), ["f32"], _lib.COUNT),
             (lambda v: v + 1 < 1, ["f32"], _lib.ANY), (lambda v: v > 0.5, ["f32"], _lib.SUM), (lambda x: 2 * x, ["i64"], _lib.MAX),
             (lambda x, s: x * s, ["f32", "f32"], _lib.MIN), (lambda x: -x, ["f64"], _lib.MAX), (lambda x: x % 3, ["i32"], _lib.MIN)]
    for f, tags, op in cases:
        st, size, err = _check(dab, f, tags, op, arrays=[1] + [0] * (len(tags) - 1) if len(tags) == 2 and tags[1] == "f32" and op == _lib.MIN else None)
        assert st == 0 and size > 2000, (tags, op, err)


def test_fused_mapreduce_refuses_unsupported(dab):
    from darray_b200 import _lib

    st, _, err = _check(dab, lambda v: v > 0.5, ["f32"], _lib.MAX)        # max of Bools: not served
    assert st == _lib.ERR_UNSUPPORTED
    st, _, err = _check(dab, lambda v: v * 2, ["f32"], _lib.ALL)          # all() of non-Bool values
    assert st == _lib.ERR_UNSUPPORTED


# ---- Int128 as the value type of mapreduce (reference test/darray.jl:286-294: exact mapreduce of Int128-valued f) -----------------------

def test_int128_tracer_and_kernels_compile():
    import ctypes as C

    import darray_b200 as dab
    from darray_b200 import _broadcast as bc
    from darray_b200 import _lib
    e = bc.trace(lambda x: dab.Int128(x) ** 2 + 2 * dab.Int128(x) - 1, ["i64"])
    assert e.jt == "i128" and bc.uses_tag(e, "i128")
    assert bc.trace(lambda x: dab.widen(x) * dab.widen(x), ["i64"]).jt == "i128"
    assert bc.trace(lambda x: dab.widen(x), ["i32"]).jt == "i64" and bc.trace(lambda x: dab.widen(x), ["f32"]).jt == "f64"
    assert bc.trace(lambda x: dab.Int128(x) * 1.5, ["i64"]).jt == "f64"            # promote_type(Int128, Float64) == Float64
    assert bc.trace(lambda x: dab.Int128(x) + x, ["i32"]).jt == "i128"
    with pytest.raises(dab.UnsupportedError):
        bc._NPT["i128"]                                                             # no arrays of Int128
    src = bc.codegen(e).encode()
    L = _lib.lib()
    for op in (_lib.SUM, _lib.PROD, _lib.MAX, _lib.MIN):
        nbytes = C.c_size_t()
        st = L.dab_jit_compile_check_reduce(src, _lib.I128, op, 1, (C.c_int32 * 1)(_lib.I64), (C.c_int32 * 1)(1), C.byref(nbytes))
        assert st == 0 and nbytes.value > 1000, L.dab_last_error(None)
    assert L.dab_jit_compile_check_reduce(src, _lib.I128, _lib.ALL, 1, (C.c_int32 * 1)(_lib.I64), (C.c_int32 * 1)(1), C.byref(nbytes)) == _lib.ERR_UNSUPPORTED
    # an Int128 intermediate under a Float64 value: the i128 prelude rides along
    src2 = bc.codegen(bc.trace(lambda x: (dab.Int128(x) * dab.Int128(x)) * 1.0, ["i64"])).encode()
    assert L.dab_jit_compile_check_reduce(src2, _lib.F64, _lib.SUM, 1, (C.c_int32 * 1)(_lib.I64), (C.c_int32 * 1)(1), C.byref(nbytes)) == 0
    # literals wider than 64 bits and negative ones survive the two-word spelling
    lit = bc._lit("i128", -3)
    assert "0xffffffffffffffffULL << 64" in lit and "0xfffffffffffffffdULL" in lit


def test_int128_fold_wraps_like_julia():
    from darray_b200 import _lib
    from darray_b200._mapreduce import fold128, wrap128
    assert wrap128(2 ** 127) == -2 ** 127 and wrap128(-2 ** 127 - 1) == 2 ** 127 - 1 and wrap128(5) == 5
    assert fold128([2 ** 126, 2 ** 126], _lib.SUM) == -2 ** 127
    assert fold128([34 ** 20, 34 ** 10], _lib.PROD) == wrap128(34 ** 30)
    assert fold128([-5, 7, 3], _lib.MAX) == 7 and fold128([-5, 7, 3], _lib.MIN) == -5


def test_int128_mapreduce_host_flow(hostmem, dab):
    """The reference's exactness test (test/darray.jl:286-294) through the host runtime on the host-memory ABI: random 1:5 vectors of
    length 2..30, f in {2x, x^2, x^2 + 2x - 1} widened to Int128, op in {+, *}; the result equals Python's exact integers wrapped
    to 128 bits (the product of 30 values up to 34 does not fit 64 bits)."""
    from darray_b200._mapreduce import wrap128
    rng = np.random.default_rng(286)
    fs = [(lambda x: 2 * dab.Int128(x), lambda v: 2 * v), (lambda x: dab.Int128(x) ** 2, lambda v: v * v),
          (lambda x: dab.Int128(x) ** 2 + 2 * dab.Int128(x) - 1, lambda v: v * v + 2 * v - 1)]
    for nw in (1, 2, 8):
        dab.init(workers_per_rank=nw, use_dist=False)
        for _ in range(8):
            a = rng.integers(1, 6, int(rng.integers(max(2, nw), 31))).astype(np.int64)
            d = dab.distribute(a)
            for tf, pf in fs:
                vals = [pf(int(v)) for v in a]
                assert dab.mapreduce(tf, "+", d) == wrap128(sum(vals))
                prod = 1
                for v in vals:
                    prod *= v
                got = dab.mapreduce(tf, "*", d)
                assert isinstance(got, int) and got == wrap128(prod)
            assert dab.mapreduce(lambda x: dab.Int128(x) * (2 ** 62), "max", d) == int(a.max()) * 2 ** 62     # beyond Int64
            assert dab.mapreduce(lambda x: -dab.Int128(x) * (2 ** 62), "min", d) == -int(a.max()) * 2 ** 62
            d.close()
    big = np.full(30, 5, dtype=np.int64)
    dab.init(workers_per_rank=2, use_dist=False)
    d = dab.distribute(big)
    assert dab.mapreduce(lambda x: dab.Int128(x) ** 2 + 2 * dab.Int128(x) - 1, "*", d) == wrap128(34 ** 30) != 34 ** 30


# ---- the rest of the reference's "scalar math" vocabulary (test/darray.jl:775-797) ---------------------------------------------------------

_EXT_NAMES = ["acos", "acosh", "acot", "acoth", "acsc", "acsch", "asec", "asech", "asin", "asinh", "atan", "atanh", "cbrt", "cosh", "cospi", "cot",
              "coth", "csc", "csch", "deg2rad", "erf", "erfc", "erfcinv", "erfcx", "erfinv", "exp10", "exp2", "expm1", "gamma", "isfinite", "isinf",
              "log10", "log1p", "log2", "loggamma", "rad2deg", "round_", "sec", "sech", "sinh", "sinpi", "trunc"]


def test_extended_unary_functions_trace_and_compile():
    """Every added unary function traces with Julia's result type and its broadcast kernel compiles for sm_90a (Float64 argument here; the
    Float32 / Int64 variants were compiled once when the functions were added).  Functions Julia defines by composition are composed the
    same way (sec = inv(cos), asec = acos(inv), deg2rad = x * (pi / 180) in the argument's type)."""
    import darray_b200 as dab
    from darray_b200 import _broadcast as bc
    from darray_b200 import _lib
    L = _lib.lib()
    for nm in _EXT_NAMES:
        f = getattr(dab, nm)
        e = bc.trace(lambda x: f(x), ["f64"])
        assert e.jt == ("bool" if nm in ("isfinite", "isinf") else "f64"), nm
        out = {"f64": _lib.F64, "bool": _lib.U8}[e.jt]
        nbytes = C.c_size_t()
        st = L.dab_jit_compile_check(bc.codegen(e).encode(), out, 1, (C.c_int32 * 1)(_lib.F64), (C.c_int32 * 1)(1), C.byref(nbytes))
        assert st == 0 and nbytes.value > 1000, (nm, L.dab_last_error(None))
    assert bc.codegen(bc.trace(lambda x: dab.sec(x), ["f32"])) == "jl_inv(jl_cos(a0))"
    assert bc.codegen(bc.trace(lambda x: dab.asec(x), ["f64"])) == "jl_acos(jl_inv(a0))"
    assert bc.codegen(bc.trace(lambda x: dab.acoth(x), ["f64"])) == "jl_x_atanh(jl_inv(a0))"
    d2r = bc.trace(lambda x: dab.deg2rad(x), ["f32"])
    assert d2r.op == "mul" and d2r.jt == "f32" and np.float32(d2r.args[1].val) == np.float32(np.pi) / np.float32(180)
    assert bc.trace(lambda x: dab.deg2rad(x), ["i64"]).jt == "f64" and bc.trace(lambda x: dab.asinh(x), ["i32"]).jt == "f64"   # float(::Int)
    assert bc.trace(lambda x: dab.round_(x), ["i64"]).jt == "i64" and bc.trace(lambda x: dab.trunc(x), ["f32"]).jt == "f32"
    # sources without an extension function do not carry the extension block: same cubin as before the block existed
    a, b = C.c_size_t(), C.c_size_t()
    assert L.dab_jit_compile_check(b"jl_sin(a0)", _lib.F64, 1, (C.c_int32 * 1)(_lib.F64), (C.c_int32 * 1)(1), C.byref(a)) == 0
    assert L.dab_jit_compile_check(b"jl_x_sinpi(a0)", _lib.F64, 1, (C.c_int32 * 1)(_lib.F64), (C.c_int32 * 1)(1), C.byref(b)) == 0
    assert a.value != b.value


def test_shift_operators_trace_and_compile():
    """``a .<< 2``, ``2 .<< a``, ``a .<< a`` and ``>>`` (test/darray.jl:863-867): the result has the type of the LEFT operand, the count is
    an Int64, floats are a MethodError; the kernels compile for sm_90a; the emulator's model follows Julia (negative counts, counts past
    the width)."""
    import darray_b200 as dab  # noqa: F401
    import hostmem_abi as hm
    from darray_b200 import _broadcast as bc
    from darray_b200 import _lib
    L = _lib.lib()
    code = {"i32": _lib.I32, "i64": _lib.I64}
    for f, tags, out in [(lambda a: a << 2, ["i64"], "i64"), (lambda a: 2 << a, ["i32"], "i64"), (lambda a: a >> 3, ["i32"], "i32"),
                         (lambda a, b: a << b, ["i32", "i64"], "i32"), (lambda a, b: a >> b, ["i64", "i32"], "i64"),
                         (lambda a: (a > 0) << 2, ["i64"], "i64")]:
        e = bc.trace(f, tags)
        assert e.jt == out
        n = len(tags)
        nbytes = C.c_size_t()
        st = L.dab_jit_compile_check(bc.codegen(e).encode(), code[out], n, (C.c_int32 * n)(*[code[t] for t in tags]), (C.c_int32 * n)(*[1] * n),
                                     C.byref(nbytes))
        assert st == 0 and nbytes.value > 1000, L.dab_last_error(None)
    with pytest.raises(TypeError):
        bc.trace(lambda a: a << 2, ["f64"])
    with pytest.raises(TypeError):
        bc.trace(lambda a: a << 2.0, ["i64"])
    # Julia: 1 << 2 == 4, 1 << 64 == 0, 1 << -1 == 0, -8 >> 1 == -4, -8 >> 70 == -1, -8 >> -2 == -32, typemin << 1 == 0, Int32(1) << 31 == typemin(Int32)
    assert [hm.jl_shift(1, 2, 64, True), hm.jl_shift(1, 64, 64, True), hm.jl_shift(1, -1, 64, True)] == [4, 0, 0]
    assert [hm.jl_shift(-8, 1, 64, False), hm.jl_shift(-8, 70, 64, False), hm.jl_shift(-8, -2, 64, False)] == [-4, -1, -32]
    assert hm.jl_shift(-2 ** 63, 1, 64, True) == 0 and hm.jl_shift(1, 31, 32, True) == -2 ** 31 and hm.jl_shift(3, 63, 64, True) == -2 ** 63
    args = [np.array([1, -8, 5], dtype=np.int64)]
    assert list(hm.eval_expr(bc.trace(lambda a: (a << 2) >> 1, ["i64"]), args)) == [2, -16, 10]


def test_shift_device_functions_on_the_host(tmp_path):
    """The text of the jl_x_shl / jl_x_shr device functions (the on-demand prelude block of dab_jit.cu) compiled for the host with g++ and
    compared with the Julia-semantics model over edge and random operands: the scalar code NVRTC will compile is checked on CPU."""
    import os
    import shutil
    import subprocess
    import hostmem_abi as hm
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "distributedarrays.jl_b200", "csrc", "dab_jit.cu")).read()
    ext = text[text.index('kPreludeExt = R"PRELUDE('):]
    ext = ext[:ext.index(')PRELUDE"')]
    body = ext[ext.index("DEV i64 jl_x_shr(i64 a, i64 n);"):]
    src = tmp_path / "shifts.cpp"
    src.write_text("typedef unsigned long long u64;\ntypedef long long i64;\n#define DEV static inline\n" + body + """
extern "C" {
i64 shl64(i64 a, i64 n) { return jl_x_shl(a, n); }
i64 shr64(i64 a, i64 n) { return jl_x_shr(a, n); }
int shl32(int a, i64 n) { return jl_x_shl(a, n); }
int shr32(int a, i64 n) { return jl_x_shr(a, n); }
}
""")
    so = str(tmp_path / "shifts.so")
    subprocess.check_call([gxx, "-O1", "-shared", "-fPIC", "-o", so, str(src)])
    L = C.CDLL(so)
    for f in (L.shl64, L.shr64):
        f.restype, f.argtypes = C.c_longlong, [C.c_longlong, C.c_longlong]
    for f in (L.shl32, L.shr32):
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_longlong]
    rng = np.random.default_rng(864)
    counts = [0, 1, 2, 31, 32, 33, 63, 64, 65, 1000, -1, -2, -31, -32, -33, -63, -64, -65, -1000, 2 ** 62, -2 ** 63]
    for bits, shl, shr in ((64, L.shl64, L.shr64), (32, L.shl32, L.shr32)):
        lo, hi = -2 ** (bits - 1), 2 ** (bits - 1) - 1
        xs = [0, 1, -1, 2, -8, lo, hi, lo + 1, 3] + [int(v) for v in rng.integers(lo, hi, 40)]
        for x in xs:
            for n in counts + [int(v) for v in rng.integers(-70, 70, 10)]:
                assert shl(x, n) == hm.jl_shift(x, n, bits, True), (bits, x, n)
                assert shr(x, n) == hm.jl_shift(x, n, bits, False), (bits, x, n)
