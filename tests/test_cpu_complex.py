"""CPU tier for the complex element types: the tracer's result types against a written-out promote_type table, NVRTC compilation of
complex trees for sm_90a, byte-identical sources for real trees, the C ABI tables, and the host-side refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = {"f32": 0, "f64": 1, "i32": 2, "i64": 3, "bool": 4, "c64": 6, "c128": 7}

# promote_type(A, B) as Julia defines it, for every pair involving ComplexF32 / ComplexF64
PROMOTE = {("c64", "bool"): "c64", ("c64", "i32"): "c64", ("c64", "i64"): "c64", ("c64", "f32"): "c64", ("c64", "f64"): "c128",
           ("c64", "c64"): "c64", ("c64", "c128"): "c128", ("c128", "bool"): "c128", ("c128", "i32"): "c128", ("c128", "i64"): "c128",
           ("c128", "f32"): "c128", ("c128", "f64"): "c128", ("c128", "c128"): "c128"}


def test_dtype_codes_and_tables(dab):
    from darray_b200 import _lib
    from darray_b200._darray import _DT, _NP
    hdr = open(os.path.join(ROOT, "include", "dab200.h")).read()
    assert re.search(r"DAB_C64 = 6\b", hdr) and re.search(r"DAB_C128 = 7\b", hdr)
    assert (_lib.C64, _lib.C128) == (6, 7)
    for dt in (np.complex64, np.complex128):
        assert _NP[_DT[np.dtype(dt)]] == np.dtype(dt) and dab.np_dtype(dab.dab_dtype(dt)) == np.dtype(dt)
    assert "dab_adjoint_box" in _lib.EXPORTS and "dab_adjoint_box" in hdr
    jl = open(os.path.join(ROOT, "julia", "DArrayB200.jl")).read()
    assert "dab_dtype(::Type{ComplexF32}) = Int32(6)" in jl and "dab_dtype(::Type{ComplexF64}) = Int32(7)" in jl


def test_reduce_result_dtypes(dab):
    from darray_b200 import _lib
    L = _lib.lib()
    out = C.c_int32()
    for dt, comp in ((_lib.C64, _lib.F32), (_lib.C128, _lib.F64)):
        for op, m, want in [(_lib.SUM, _lib.MAP_ID, dt), (_lib.PROD, _lib.MAP_ID, dt), (_lib.SUM, _lib.MAP_NEG, dt), (_lib.PROD, _lib.MAP_NEG, dt),
                            (_lib.SUM, _lib.MAP_ABS2, comp), (_lib.MAX, _lib.MAP_ABS, comp), (_lib.MIN, _lib.MAP_ABS2, comp),
                            (_lib.COUNT, _lib.MAP_ISNAN, _lib.I64), (_lib.ANY, _lib.MAP_NONZERO, _lib.I64), (_lib.ALL, _lib.MAP_ISNAN, _lib.I64)]:
            assert L.dab_reduce_result_dtype(dt, op, m, C.byref(out)) == _lib.OK and out.value == want, (dt, op, m)
        for op, m in [(_lib.MAX, _lib.MAP_ID), (_lib.MIN, _lib.MAP_ID), (_lib.EXTREMA, _lib.MAP_ID), (_lib.PROD, _lib.MAP_ABS), (_lib.SUM, _lib.MAP_SQRT)]:
            assert L.dab_reduce_result_dtype(dt, op, m, C.byref(out)) == _lib.ERR_UNSUPPORTED, (dt, op, m)


def test_combine_ordered_complex_is_a_left_fold(dab):
    from darray_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(0)
    for ct, T in ((np.complex64, np.float32), (np.complex128, np.float64)):
        v = (rng.standard_normal(7) + 1j * rng.standard_normal(7)).astype(ct) * T(1e3)
        out = np.zeros(1, dtype=ct)
        _lib.check(L.dab_combine_ordered(_lib.C64 if ct == np.complex64 else _lib.C128, _lib.SUM, C.c_void_p(v.ctypes.data), 7, C.c_void_p(out.ctypes.data)))
        re, im = v[0].real, v[0].imag
        for z in v[1:]:
            re, im = T(re + z.real), T(im + z.imag)
        assert out[0].real == re and out[0].imag == im
        _lib.check(L.dab_combine_ordered(_lib.C64 if ct == np.complex64 else _lib.C128, _lib.PROD, C.c_void_p(v.ctypes.data), 7, C.c_void_p(out.ctypes.data)))
        re, im = v[0].real, v[0].imag
        for z in v[1:]:
            re, im = T(T(re * z.real) - T(im * z.imag)), T(T(re * z.imag) + T(im * z.real))
        assert out[0].real == re and out[0].imag == im


def test_tracer_promotion_table():
    from darray_b200._broadcast import trace
    for (a, b), want in PROMOTE.items():
        for f in (lambda x, y: x + y, lambda x, y: x * y, lambda x, y: x - y, lambda x, y: x / y):
            assert trace(f, [a, b]).jt == want, (a, b)
            assert trace(f, [b, a]).jt == want, (b, a)
        assert trace(lambda x, y: x == y, [a, b]).jt == "bool"
    assert trace(lambda z: z + 1j, ["c64"]).jt == "c128"                                  # a Python complex literal is a ComplexF64
    assert trace(lambda z: z + np.complex64(1j), ["c64"]).jt == "c64"
    assert trace(lambda z: z * 2, ["c64"]).jt == "c64" and trace(lambda z: z * 2.0, ["c64"]).jt == "c128"
    assert trace(lambda z: z * np.float32(2), ["c64"]).jt == "c64"


def test_tracer_complex_functions():
    import darray_b200 as dab
    from darray_b200._broadcast import codegen, trace
    for f, tag, want in [(abs, "c64", "f32"), (dab.abs2, "c128", "f64"), (dab.real, "c64", "f32"), (dab.imag, "c128", "f64"),
                         (dab.angle, "c64", "f32"), (dab.conj, "c64", "c64"), (dab.inv, "c128", "c128"), (lambda z: -z, "c64", "c64"),
                         (dab.isnan, "c64", "bool"), (dab.isinf, "c128", "bool"), (dab.isfinite, "c64", "bool"), (dab.iszero, "c128", "bool"),
                         (dab.cis, "f32", "c64"), (dab.cis, "i64", "c128"), (dab.complex, "f64", "c128"), (dab.real, "f32", "f32"),
                         (dab.conj, "i64", "i64"), (dab.angle, "f64", "f64")]:
        assert trace(f, [tag]).jt == want, (f, tag)
    assert trace(lambda x, y: dab.complex(x, y), ["f32", "i64"]).jt == "c64"
    assert trace(lambda x: dab.imag(x), ["f64"]).op == "const"
    assert trace(lambda z, w: dab.ifelse(dab.isnan(z), z, w), ["c64", "c128"]).jt == "c128"
    # the mixed real/complex methods keep the real operand real (in the component type)
    e = trace(lambda x, z: x * z, ["f32", "c64"])
    assert e.args[0].jt == "f32" and e.args[1].jt == "c64"
    assert codegen(trace(lambda z: z * 2.0, ["c64"])) == "jl_mul(jl_c128(a0), __longlong_as_double((long long)0x4000000000000000ULL))"
    for f in (dab.exp, dab.sqrt, dab.sin, dab.log, dab.floor, dab.tanh, dab.gamma, lambda z: z ** 2, lambda z: dab.mod(z, 2.0),
              lambda z: z % 2, lambda z: z // 2, dab.cis, lambda z: z << 1):
        with pytest.raises(dab.UnsupportedError):
            trace(f, ["c64"])
    for f in (lambda z: z < 1, lambda z: z >= 0.5, lambda z, w: dab.jl_max(z, w), lambda z, w: dab.jl_min(z, w)):
        with pytest.raises(TypeError):
            trace(f, ["c128", "c128"][:f.__code__.co_argcount])
    with pytest.raises(dab.UnsupportedError):
        trace(lambda x: dab.complex(x), ["i64"])                                           # Complex{Int} is not served


def test_complex_trees_route_to_nvrtc_only():
    from darray_b200._broadcast import match_affine, trace, uses_complex
    e = trace(lambda z: 2 * z + 1, ["c64"])
    assert uses_complex(e)                                                                  # run_local skips every hand-written kernel
    assert match_affine(trace(lambda x: 2 * x + 1, ["f32"])) == (2.0, 1.0)


def _compile(L, src, out, tags, reduce_op=None, arr=None):
    n = len(tags)
    dts = (C.c_int32 * n)(*[CODE[t] for t in tags])
    isarr = (C.c_int32 * n)(*(arr if arr is not None else [1] * n))
    sz = C.c_size_t()
    if reduce_op is None:
        st = L.dab_jit_compile_check(src, CODE[out], n, dts, isarr, C.byref(sz))
    else:
        st = L.dab_jit_compile_check_reduce(src, CODE[out], reduce_op, n, dts, isarr, C.byref(sz))
    return st, sz.value


def test_complex_codegen_compiles_for_sm90a(dab):
    from darray_b200 import _lib
    from darray_b200._broadcast import codegen, convert, split_c128_scalars, trace, LocalArg
    L = _lib.lib()
    cases = [(lambda z, w: z * w + dab.conj(z) / w, ["c64", "c64"], "c64"), (lambda z, x: 2.0 * z - x, ["c64", "f32"], "c128"),
             (lambda z: abs(z) + dab.angle(z) + dab.abs2(z), ["c128"], "f64"), (lambda x: dab.cis(x), ["f64"], "c128"),
             (lambda z: dab.inv(z) - 1j, ["c64"], "c128"), (lambda x, y: dab.complex(x, y), ["f32", "f32"], "c64"),
             (lambda z, w: dab.ifelse(dab.isnan(z), w, z), ["c128", "c64"], "c128"), (lambda x: x * 3, ["f32"], "c64")]
    for f, tags, out in cases:
        src = codegen(convert(trace(f, tags), out)).encode()
        st, sz = _compile(L, src, out, tags, arr=[1] * (len(tags) - 1) + [0 if len(tags) > 1 and tags[-1] != "c128" else 1])
        assert st == 0 and sz > 1000, (src, L.dab_last_error(None))
    for f, tags, val, op in [(lambda z: z, ["c64"], "c64", _lib.SUM), (lambda z: z, ["c64"], "c64", _lib.PROD), (lambda z: z, ["c128"], "c128", _lib.SUM),
                             (lambda z, w: dab.conj(z) * w, ["c128", "c128"], "c128", _lib.SUM), (lambda z, w: z == w, ["c64", "c64"], "bool", _lib.ALL),
                             (lambda z: dab.isnan(z), ["c128"], "bool", _lib.COUNT), (lambda z: abs(z), ["c64"], "f32", _lib.PROD)]:
        src = codegen(trace(f, tags)).encode()
        st, sz = _compile(L, src, val, tags, reduce_op=op)
        assert st == 0 and sz > 1000, (src, L.dab_last_error(None))
    st, _ = _compile(L, b"a0", "c128", ["c128"], reduce_op=_lib.MAX)
    assert st == _lib.ERR_UNSUPPORTED
    st, _ = _compile(L, b"a0", "c128", ["c128"], arr=[0])                               # a ComplexF64 scalar does not fit 8 bytes ...
    assert st == _lib.ERR_ARG
    e, largs = split_c128_scalars(trace(lambda z, s: z * s, ["c128", "c128"]), [LocalArg(object(), None, "c128"), LocalArg(None, 1 - 2j, "c128")])
    assert [a.tag for a in largs] == ["c128", "f64", "f64"] and (largs[1].scalar, largs[2].scalar) == (1.0, -2.0)
    st, _ = _compile(L, codegen(e).encode(), "c128", ["c128", "f64", "f64"], arr=[1, 0, 0])  # ... it enters as complex(re, im)
    assert st == 0, L.dab_last_error(None)


def test_real_sources_unchanged(dab):
    """The complex prelude is appended only to sources that use a complex type: real trees generate exactly the source they did (a written-out
    corpus), still compile, and the library appends the complex block behind the ``uses_cplx`` gate only."""
    from darray_b200 import _lib
    from darray_b200._broadcast import codegen, convert, trace
    L = _lib.lib()
    corpus = [(lambda x: 2 * x + 1, ["f32"], "f32"), (lambda a, m, c: a - m * dab.sin(c), ["f64"] * 3, "f64"), (lambda x, y: x % y, ["i32", "i32"], "i32"),
              (lambda x: x > 1.0, ["f64"], "bool"), (lambda x: dab.erf(x) + dab.abs2(x), ["f32"], "f32"), (lambda x, y: dab.ifelse(x < y, x, y), ["i64", "i64"], "i64")]
    want = ["jl_add(jl_mul(__int_as_float((int)0x40000000), a0), __int_as_float((int)0x3f800000))",
            "jl_sub(a0, jl_mul(a1, jl_sin(a2)))", "jl_rem(a0, a1)", "jl_gt(a0, __longlong_as_double((long long)0x3ff0000000000000ULL))",
            "jl_add(jl_x_erf(a0), jl_abs2(a0))", "((jl_lt(a0, a1)) ? (a0) : (a1))"]
    for (f, tags, out), w in zip(corpus, want):
        src = codegen(convert(trace(f, tags), out))
        assert src == w and "jl_c" not in src
        st, _ = _compile(L, src.encode(), out, tags)
        assert st == 0
    # the library source: the complex block is gated, the real prelude itself does not mention the complex types
    jit = open(os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_jit.cu")).read()
    prelude = jit[jit.index('const char* kPrelude = R"PRELUDE('):jit.index(')PRELUDE";')]
    assert "jl_c64" not in prelude and "if (uses_cplx(expr, out_dt, nargs, dts)) s += kPreludeCplx;" in jit


def test_host_refusals_before_any_launch(dab, hostmem):
    """Refusals happen on the host: with the host-memory ABI installed, none of these reaches an entry point that launches."""
    rt = dab.init(workers_per_rank=2, use_dist=False)
    z = dab.distribute(np.ones((8, 8), np.complex128))
    v = dab.distribute(np.ones(8, np.complex64))
    with pytest.raises(TypeError):
        dab.maximum(z)
    with pytest.raises(TypeError):
        dab.extrema(z)
    with pytest.raises(TypeError):
        dab.sort(v)
    with pytest.raises(dab.UnsupportedError):
        z @ z
    with pytest.raises(dab.UnsupportedError):
        z @ np.ones(8, np.complex128)
    with pytest.raises(dab.UnsupportedError):
        dab.mapslices(dab.sort, z, dims=1)
    with pytest.raises(dab.UnsupportedError):
        dab.prod(z, dims=1)
    with pytest.raises(dab.UnsupportedError):
        dab.broadcast(dab.exp, z)
    with pytest.raises(dab.InexactError):
        dab.rmul_(dab.distribute(np.ones(8)), 1 + 1j)
    assert rt is not None


def test_reducedim_refuses_complex_ops_before_touching_the_device(dab):
    """dab_reducedim takes the complex codes for SUM with MAP_ID only (as the real SUM over 2*inner components); every other op or map is
    refused with DAB_ERR_UNSUPPORTED naming the type, before the context or any buffer is used (here: no context, null buffers)."""
    from darray_b200 import _lib
    L = _lib.lib()
    for dt, name in ((_lib.C64, b"ComplexF32"), (_lib.C128, b"ComplexF64")):
        for op, m, red in ((_lib.PROD, _lib.MAP_ID, 0), (_lib.PROD, _lib.MAP_ID, 1 << 16), (_lib.MAX, _lib.MAP_ID, 7), (_lib.SUM, _lib.MAP_ABS, 7),
                           (_lib.SUM, _lib.MAP_ABS2, 1 << 16), (_lib.MIN, _lib.MAP_NEG, 0)):
            assert L.dab_reducedim(None, dt, op, m, None, 1, red, 1, None, 0) == _lib.ERR_UNSUPPORTED
            assert name in L.dab_last_error(None)
        assert L.dab_reducedim(None, dt, _lib.SUM, _lib.MAP_ID, None, 1, 7, 1, None, 0) == _lib.ERR_ARG      # served: reaches the null-ctx check
