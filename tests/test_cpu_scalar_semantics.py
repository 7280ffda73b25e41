"""The model of Julia's scalar methods (tests/julia_scalar.py) against answers taken from the Base definitions, its vectorised forms
against its scalar methods, and the tracer's trees and result types for the methods that are not "promote, then operate"."""
import ctypes as C

import numpy as np
import pytest

import julia_scalar as jl

f32, f64, i32, i64, B = np.float32, np.float64, np.int32, np.int64, np.bool_
NAN, INF = np.nan, np.inf
IMAX, IMIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min


def same(got, want) -> bool:
    """``===``: same type and same bits (every NaN is the same)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype:
        return False
    if got.dtype.kind == "f":
        return bool(np.isnan(got) == np.isnan(want) and (np.isnan(got) or got.tobytes() == want.tobytes()))
    return bool(got == want)


# (expression, model value, Julia's answer) -- from base/bool.jl, base/int.jl, base/float.jl, base/number.jl, base/math.jl, base/intfuncs.jl
JULIA = [
    ("false*NaN === 0.0", jl.binop("mul", B(False), f64(NAN)), f64(0.0)),
    ("false*-NaN === -0.0", jl.binop("mul", B(False), f64(-NAN)), f64(-0.0)),
    ("false*-Inf === -0.0", jl.binop("mul", B(False), f64(-INF)), f64(-0.0)),
    ("true*-Inf === -Inf", jl.binop("mul", B(True), f64(-INF)), f64(-INF)),
    ("Inf32*false === 0f0", jl.binop("mul", f32(INF), B(False)), f32(0.0)),
    ("false + -0.0 === -0.0", jl.binop("add", B(False), f64(-0.0)), f64(-0.0)),
    ("-0f0 + false === -0f0", jl.binop("add", f32(-0.0), B(False)), f32(-0.0)),
    ("true + -0.0 === 1.0", jl.binop("add", B(True), f64(-0.0)), f64(1.0)),
    ("false - 0.0 === 0.0", jl.binop("sub", B(False), f64(0.0)), f64(0.0)),
    ("true*true === true", jl.binop("mul", B(True), B(True)), B(True)),
    ("true + true === 2", jl.binop("add", B(True), B(True)), i64(2)),
    ("abs(true) === true", jl.unop("abs", B(True)), B(True)),
    ("abs2(true) === true", jl.unop("abs2", B(True)), B(True)),
    ("sign(false) === false", jl.unop("sign", B(False)), B(False)),
    ("round(true) === true", jl.unop("round", B(True)), B(True)),
    ("-true === -1", jl.unop("neg", B(True)), i64(-1)),
    ("2^53+1 == 2.0^53 is false", jl.binop("eq", i64(2 ** 53 + 1), f64(2.0 ** 53)), B(False)),
    ("2^53+1 > 2.0^53", jl.binop("gt", i64(2 ** 53 + 1), f64(2.0 ** 53)), B(True)),
    ("typemax(Int) < 2.0^63", jl.binop("lt", i64(IMAX), f64(2.0 ** 63)), B(True)),
    ("typemin(Int) == -2.0^63", jl.binop("eq", i64(IMIN), f64(-2.0 ** 63)), B(True)),
    ("2^24+1 == 16777216f0 is false", jl.binop("eq", i64(2 ** 24 + 1), f32(2.0 ** 24)), B(False)),
    ("Int32(2^24+1) == 16777216f0 (promotes)", jl.binop("eq", i32(2 ** 24 + 1), f32(2.0 ** 24)), B(True)),
    ("3 < 3.5", jl.binop("lt", i64(3), f64(3.5)), B(True)),
    ("-3 > -3.5", jl.binop("gt", i64(-3), f64(-3.5)), B(True)),
    ("1 != NaN", jl.binop("ne", i64(1), f64(NAN)), B(True)),
    ("1 <= NaN is false", jl.binop("le", i64(1), f64(NAN)), B(False)),
    ("mod(-0.0, 1.0) === 0.0", jl.binop("mod", f64(-0.0), f64(1.0)), f64(0.0)),
    ("mod(0.0, -1.0) === -0.0", jl.binop("mod", f64(0.0), f64(-1.0)), f64(-0.0)),
    ("mod(-1f0, 3f0) === 2f0", jl.binop("mod", f32(-1.0), f32(3.0)), f32(2.0)),
    ("rem(-1.0, 3.0) === -1.0", jl.binop("rem", f64(-1.0), f64(3.0)), f64(-1.0)),
    ("mod(-7, 3) === 2", jl.binop("mod", i64(-7), i64(3)), i64(2)),
    ("rem(-7, 3) === -1", jl.binop("rem", i64(-7), i64(3)), i64(-1)),
    ("div(-7, 2) === -3", jl.binop("idiv", i64(-7), i64(2)), i64(-3)),
    ("div(typemax(Int), -7)", jl.binop("idiv", i64(IMAX), i64(-7)), i64(-(IMAX // 7))),
    ("max(-0.0, 0.0) === 0.0", jl.binop("max", f64(-0.0), f64(0.0)), f64(0.0)),
    ("min(0.0, -0.0) === -0.0", jl.binop("min", f64(0.0), f64(-0.0)), f64(-0.0)),
    ("max(NaN, Inf) is NaN", jl.binop("max", f64(NAN), f64(INF)), f64(NAN)),
    ("min(-Inf32, NaN32) is NaN", jl.binop("min", f32(-INF), f32(NAN)), f32(NAN)),
    ("sign(-0.0) === -0.0", jl.unop("sign", f64(-0.0)), f64(-0.0)),
    ("sign(NaN) is NaN", jl.unop("sign", f64(NAN)), f64(NAN)),
    ("sign(-3) === -1", jl.unop("sign", i64(-3)), i64(-1)),
    ("round(2.5) == 2.0", jl.unop("round", f64(2.5)), f64(2.0)),
    ("round(-0.5) === -0.0", jl.unop("round", f64(-0.5)), f64(-0.0)),
    ("trunc(-0.7f0) === -0f0", jl.unop("trunc", f32(-0.7)), f32(-0.0)),
    ("abs(typemin(Int32)) wraps", jl.unop("abs", i32(-2 ** 31)), i32(-2 ** 31)),
    ("inv(2) === 0.5", jl.unop("inv", i64(2)), f64(0.5)),
    ("sqrt(4) === 2.0", jl.unop("sqrt", i64(4)), f64(2.0)),
    ("Float32(2^53+2^29+1) rounds once", jl.convert(i64(2 ** 53 + 2 ** 29 + 1), "f32"), f32(2.0 ** 53 + 2 ** 30)),
    ("3 / 2 === 1.5", jl.binop("div", i64(3), i64(2)), f64(1.5)),
    ("Int32(1) + 1.0f0 === 2f0", jl.binop("add", i32(1), f32(1.0)), f32(2.0)),
    ("Int64 + Float32 is Float32", jl.binop("add", i64(1), f32(1.0)), f32(2.0)),
    ("x^0 === 1f0 for NaN32", jl.literal_pow(f32(NAN), 0), f32(1.0)),
    ("x^-1 === inv(x)", jl.literal_pow(f64(4.0), -1), f64(0.25)),
    ("x^-2 == inv(x)^2", jl.literal_pow(f32(3.0), -2), f32(1 / 3.0) * f32(1 / 3.0)),
    ("2f0^-3 === 0.125f0", jl.pow_f32_int(f32(2.0), -3), f32(0.125)),
    ("(-1f0)^typemin(Int) === 1f0", jl.pow_f32_int(f32(-1.0), IMIN), f32(1.0)),
    ("1.1f0^7 in Float64", jl.pow_f32_int(f32(1.1), 7), f32(float(f32(1.1)) ** 7)),
    ("Bool(1) from Int64", jl.convert(i64(1), "bool"), B(True)),
    ("Int32(-5) from Int64", jl.convert(i64(-5), "i32"), i32(-5)),
    ("ifelse(true, 1, 2.0) === 1.0", jl.ifelse(True, i64(1), f64(2.0)), f64(1.0)),
]


@pytest.mark.parametrize("name,got,want", JULIA, ids=[j[0] for j in JULIA])
def test_model_against_julia_answers(name, got, want):
    assert same(got, want), (name, got, want)


def test_documented_deviations():
    """The backend's answers where Julia throws: by-zero divisions give 0, typemin ÷ -1 wraps."""
    for t in (i32, i64):
        for op in ("idiv", "rem", "mod"):
            assert jl.binop(op, t(7), t(0)) == 0
        assert jl.binop("idiv", t(np.iinfo(t).min), t(-1)) == np.iinfo(t).min
        assert jl.binop("rem", t(np.iinfo(t).min), t(-1)) == 0


BIN_FLOAT = ("add", "sub", "mul", "div", "rem", "mod", "max", "min", "eq", "ne", "lt", "le", "gt", "ge")
BIN_INT = ("add", "sub", "mul", "rem", "mod", "idiv", "max", "min", "and", "or", "xor", "eq", "lt", "ge")
UN = ("abs", "abs2", "neg", "sign", "inv", "sqrt", "floor", "ceil", "trunc", "round")


def _same_arrays(got, want):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype.kind == "f":
        nan = np.isnan(want)
        return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint8), want[~nan].view(np.uint8))
    return np.array_equal(got, want)


@pytest.mark.parametrize("t", ["f32", "f64", "i32", "i64"])
def test_vectorised_forms_follow_the_scalar_methods(t):
    """``vbin`` / ``vun`` (used by the host-memory emulation) give the scalar methods' answers on the whole value grid."""
    g = jl.grid(t)
    x, y = jl.pairs(g, g)
    for op in BIN_FLOAT if t[0] == "f" else BIN_INT:
        want = jl.table2(op, x, y)
        got = jl.vbin(op, x, y)
        assert _same_arrays(np.asarray(got).astype(want.dtype), want), op
    for op in UN:
        if t[0] == "i" and op in ("inv", "sqrt"):
            continue
        want = jl.table1(op, g)
        assert _same_arrays(jl.vun(op, g), want), op
    if t[0] == "f":
        gi = jl.grid("i64")
        xi, yf = jl.pairs(gi, g)
        for op in ("eq", "ne", "lt", "le", "gt", "ge"):
            assert np.array_equal(jl.vcmp_exact(op, xi, yf), jl.table2(op, xi, yf)), op
            assert np.array_equal(jl.vcmp_exact(op, yf, xi), jl.table2(op, yf, xi)), op


def test_power_by_squaring_against_exact_powers():
    """For exponents whose powers are exact in Float64, power_by_squaring is the exact power."""
    for x in (2.0, -2.0, 0.5, 3.0, -1.0):
        for p in range(0, 30):
            assert jl.power_by_squaring(np.float64(x), p) == x ** p


# ---------------------------------------------------------------------------------------------------------- the tracer
def _tr(f, tags, out=None):
    from darray_b200._broadcast import codegen, convert, trace
    e = trace(f, tags)
    return e, codegen(convert(e, out or e.jt))


def test_tracer_bool_methods(dab):
    e, src = _tr(lambda x: (x > 0) * x, ["f64"])
    assert e.jt == "f64" and e.op == "ifelse" and "jl_m_copysign" in src and "jl_mul" not in src
    for tags in (["bool", "f32"], ["f32", "bool"]):
        e, src = _tr(lambda a, b: a * b, tags)
        assert e.jt == "f32" and e.op == "ifelse" and e.args[0].jt == "bool"
        e, _ = _tr(lambda a, b: a + b, tags)
        assert e.jt == "f32" and e.op == "ifelse" and e.args[2].op == "arg"     # false + x is x itself
    e, _ = _tr(lambda x: True * x, ["f64"])
    assert e.op == "ifelse" and e.args[0].op == "const"
    e, src = _tr(lambda a, b: a * b, ["bool", "bool"])
    assert e.jt == "bool" and src == "jl_and(a0, a1)"
    for f in (abs, dab.abs2, dab.round_, dab.trunc, dab.sign, lambda x: x * x, lambda x: x ** 2):
        e, _ = _tr(f, ["bool"])
        assert e.jt == "bool", f
    assert _tr(lambda x: -x, ["bool"])[0].jt == "i64"
    assert _tr(lambda a, b: a + b, ["bool", "bool"])[0].jt == "i64"
    assert _tr(lambda a, b: a * b, ["bool", "i32"])[0].jt == "i32"


def test_tracer_exact_int64_float_comparisons(dab):
    for ft in ("f32", "f64"):
        for op, f in (("lt", lambda a, b: a < b), ("eq", lambda a, b: a == b), ("ge", lambda a, b: a >= b)):
            e, src = _tr(f, ["i64", ft])
            assert e.op == "m_" + op and e.jt == "bool" and e.args[0].jt == "i64" and e.args[1].jt == ft
            assert src == f"jl_m_{op}(a0, a1)"
            e, _ = _tr(f, [ft, "i64"])
            assert e.op == "m_" + op and e.args[0].jt == ft
    # an Int64 constant the float type holds exactly keeps the converted comparison (the generated source is unchanged)
    assert _tr(lambda x: x > 1, ["f64"])[1] == "jl_gt(a0, __longlong_as_double((long long)0x3ff0000000000000ULL))"
    assert _tr(lambda x: x > 2 ** 53 + 1, ["f64"])[0].op == "m_gt"
    assert _tr(lambda x: x > 2 ** 24 + 1, ["f32"])[0].op == "m_gt"
    assert _tr(lambda x: x > 0.5, ["i64"])[0].op == "m_gt"
    assert _tr(lambda a, b: a < b, ["i32", "f32"])[0].op == "lt"                # Int32 with Float32 promotes in Julia too
    assert _tr(lambda a, b: dab.ifelse(a < b, a, b), ["i64", "f64"])[0].args[0].op == "m_lt"


def test_tracer_powers(dab):
    for t in ("f32", "f64"):
        e, src = _tr(lambda x: x ** 0, [t])
        assert e.op == "const" and e.val == 1.0 and e.jt == t
        e, src = _tr(lambda x: x ** -1, [t])
        assert src == "jl_inv(a0)"
        e, src = _tr(lambda x: x ** -2, [t])
        assert src == "jl_mul(jl_inv(a0), jl_inv(a0))"
        assert _tr(lambda x: x ** 3, [t])[1] == "jl_mul(jl_mul(a0, a0), a0)"
    assert _tr(lambda x: x ** 7, ["f32"])[1] == "jl_m_powi(a0, ((long long)7LL))"
    assert _tr(lambda x: x ** -5, ["f32"])[0].op == "m_powi"
    assert _tr(lambda x: x ** 7, ["f64"])[0].op == "pow"                          # Float64 ^ Integer stays a pow call
    e, src = _tr(lambda x, n: x ** n, ["f32", "i32"])
    assert e.op == "m_powi" and e.jt == "f32" and src == "jl_m_powi(a0, ((long long)(a1)))"
    assert _tr(lambda x, n: x ** n, ["f32", "i64"])[0].op == "m_powi"
    assert _tr(lambda x, n: x ** n, ["f32", "f32"])[0].op == "pow"
    assert _tr(lambda x: x ** -1, ["i64"])[0].jt == "f64"                         # inv(x::Integer) is Float64
    assert _tr(lambda x: x ** 0, ["i32"])[0].jt == "i32"
    assert _tr(lambda x: x ** -2, ["bool"])[0].jt == "f64"


NEW_SOURCES = [
    (lambda x: (x > 0) * x, ["f32"], "f32"), (lambda x: (x > 0) * x, ["f64"], "f64"), (lambda b, x: b * x, ["bool", "f64"], "f64"),
    (lambda b, x: x + b, ["bool", "f32"], "f32"), (lambda a, b: a * b, ["bool", "bool"], "bool"), (lambda x: abs(x), ["bool"], "bool"),
    (lambda a, b: a == b, ["i64", "f64"], "bool"), (lambda a, b: a <= b, ["f32", "i64"], "bool"), (lambda a, b: a != b, ["f64", "i64"], "bool"),
    (lambda a, b: a > b, ["i64", "f32"], "bool"), (lambda x: x ** 7, ["f32"], "f32"), (lambda x: x ** -9, ["f32"], "f32"),
    (lambda x, n: x ** n, ["f32", "i32"], "f32"), (lambda x, n: x ** n, ["f32", "i64"], "f32"), (lambda x: x ** -2, ["f64"], "f64"),
]
_CODE = {"f32": 0, "f64": 1, "i32": 2, "i64": 3, "bool": 4}


@pytest.mark.parametrize("k", range(len(NEW_SOURCES)))
def test_new_sources_compile_for_sm90a(dab, k):
    """Every source the new methods generate compiles for sm_90a (elementwise and fused map + reduce)."""
    from darray_b200 import _lib
    f, tags, out = NEW_SOURCES[k]
    _, src = _tr(f, tags, out)
    L = _lib.lib()
    dts = (C.c_int32 * len(tags))(*[_CODE[t] for t in tags])
    arr = (C.c_int32 * len(tags))(*[1] * len(tags))
    size = C.c_size_t()
    assert L.dab_jit_compile_check(src.encode(), _CODE[out], len(tags), dts, arr, C.byref(size)) == 0, L.dab_last_error(None)
    op = _lib.COUNT if out == "bool" else _lib.SUM
    assert L.dab_jit_compile_check_reduce(src.encode(), _CODE[out], op, len(tags), dts, arr, C.byref(size)) == 0, L.dab_last_error(None)
    assert size.value > 0


def test_methods_block_is_gated():
    """The jl_m_* helpers sit in their own prelude block, appended only to sources that name one."""
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    jit = open(os.path.join(root, "distributedarrays.jl_b200", "csrc", "dab_jit.cu")).read()
    prelude = jit[jit.index('const char* kPrelude = R"PRELUDE('):jit.index(')PRELUDE";')]
    assert "jl_m_" not in prelude
    assert jit.count("if (mentions_methods(expr)) s += kPreludeMethods;") == 2
