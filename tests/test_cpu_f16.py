"""Float16 on the host side, without a GPU: the dtype code agrees across the C header, the ctypes layer, the array layer and the Julia
binding; the tracer follows Julia's promotion for Float16 (np.float16 scalars are Float16 constants, Python floats Float64 literals);
Float16 expressions and fused map-reduce kernels compile for sm_90a through NVRTC; the host-side Float16 fold and result types."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16 = np.float16


def test_dtype_code_agrees_everywhere(dab):
    from darray_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dab200.h")).read()
    assert re.search(r"DAB_F16\s*=\s*8\b", hdr)
    assert _lib.F16 == 8
    assert dab.dab_dtype(np.float16) == 8 and dab.np_dtype(8) == np.dtype(np.float16)
    jl = open(os.path.join(ROOT, "julia", "DArrayB200.jl")).read()
    assert "dab_dtype(::Type{Float16}) = Int32(8)" in jl and 'ctype(::Type{Float16}) = "jl_f16"' in jl


def test_promotion_table():
    from darray_b200._broadcast import promote
    assert promote("f16", "bool") == "f16" and promote("f16", "i32") == "f16" and promote("i64", "f16") == "f16"
    assert promote("f16", "f32") == "f32" and promote("f64", "f16") == "f64" and promote("f16", "f16") == "f16"
    assert promote("f16", "c64") == "c64" and promote("c128", "f16") == "c128"


def test_tracer_result_types(dab):
    from darray_b200._broadcast import trace
    assert trace(lambda x: x * F16(1.5), ["f32"]).jt == "f32"            # np.float16 scalar: Float16 constant
    assert trace(lambda x: x * 1.5, ["f16"]).jt == "f64"                 # Python float: Float64 literal
    assert trace(lambda x: x * 2, ["f16"]).jt == "f16"
    assert trace(lambda x: x / 2, ["f16"]).jt == "f16"
    assert trace(lambda x: dab.sqrt(x) + dab.sin(x), ["f16"]).jt == "f16"
    assert trace(lambda x: x ** 3, ["f16"]).jt == "f16" and trace(lambda x: x ** 7, ["f16"]).jt == "f16"
    assert trace(lambda x: dab.Float16(x), ["f64"]).jt == "f16" and trace(lambda x: dab.Float16(x), ["i64"]).jt == "f16"
    assert trace(lambda x: dab.widen(x), ["f16"]).jt == "f32"
    assert trace(lambda x: x < 1, ["f16"]).jt == "bool"
    with pytest.raises(dab.UnsupportedError):
        trace(lambda x: dab.complex(x), ["f16"])                          # ComplexF16 is not served


def test_float64_constant_rounds_once():
    from darray_b200._broadcast import Expr, convert
    x = 1 + 2.0 ** -11 + 2.0 ** -40                                      # through Float32 this would tie and round to even (1.0)
    c = convert(Expr.wrap(x), "f16")
    assert c.val == float(F16(x)) == 1 + 2.0 ** -10


def _compile(dab, f, tags, out):
    from darray_b200 import _lib
    from darray_b200._broadcast import _NPT, codegen, convert, trace
    src = codegen(convert(trace(f, tags), out)).encode()
    n = len(tags)
    dts = (C.c_int32 * n)(*[dab.dab_dtype(_NPT[t]) for t in tags])
    sz = C.c_size_t()
    st = _lib.lib().dab_jit_compile_check(src, dab.dab_dtype(_NPT[out]), n, dts, (C.c_int32 * n)(*([1] * n)), C.byref(sz))
    return st, src


@pytest.mark.parametrize("f,tags,out", [
    (lambda x, y: x * y + F16(1.5), ["f16", "f16"], "f16"),
    (lambda x: dab_fns(x), ["f16"], "f16"),
    (lambda x, y: x + y, ["f16", "f64"], "f64"),
    (lambda x, y: x, ["f16", "f32"], "f32"),
    (lambda x, y: x * y, ["i64", "f16"], "f16"),
    (lambda x, y: (x < y) * x + x ** y, ["f16", "i32"], "f16"),
    (lambda x: x, ["f64"], "f16"),
    (lambda x: x, ["i32"], "f16"),
])
def test_float16_kernels_compile(dab, f, tags, out):
    st, src = _compile(dab, f, tags, out)
    assert st == 0, src


def dab_fns(x):
    import darray_b200 as dab
    return dab.sqrt(x) + dab.exp(x) + dab.erf(x) + dab.trunc(x) + abs(x) - dab.floor(x) + dab.jl_max(x, dab.ceil(x)) + dab.mod(x, x)


@pytest.mark.parametrize("op", ["SUM", "PROD", "MAX", "MIN"])
def test_float16_mapreduce_compiles(dab, op):
    from darray_b200 import _lib
    from darray_b200._broadcast import codegen, trace
    src = codegen(trace(lambda x, y: x * y, ["f16", "f16"])).encode()
    sz = C.c_size_t()
    st = _lib.lib().dab_jit_compile_check_reduce(src, _lib.F16, getattr(_lib, op), 2, (C.c_int32 * 2)(_lib.F16, _lib.F16),
                                                 (C.c_int32 * 2)(1, 1), C.byref(sz))
    assert st == 0 and sz.value > 0


def test_result_dtypes_and_fold():
    from darray_b200 import _lib
    L = _lib.lib()
    out = C.c_int32()
    for op in (_lib.SUM, _lib.PROD, _lib.MAX, _lib.MIN):
        assert L.dab_reduce_result_dtype(_lib.F16, op, _lib.MAP_ID, C.byref(out)) == 0 and out.value == _lib.F16
    assert L.dab_reduce_result_dtype(_lib.F16, _lib.COUNT, _lib.MAP_NONZERO, C.byref(out)) == 0 and out.value == _lib.I64
    v = np.array([65504, 65504, -65504], F16)                               # Float16 left fold: Inf after the first add stays Inf
    o = np.zeros(1, F16)
    assert L.dab_combine_ordered(_lib.F16, _lib.SUM, C.c_void_p(v.ctypes.data), 3, C.c_void_p(o.ctypes.data)) == 0 and o[0] == np.inf
    v = np.array([1, 2 ** -11, 2 ** -11], F16)                              # each add rounds to Float16: 1 + 2^-11 ties to 1, twice
    assert L.dab_combine_ordered(_lib.F16, _lib.SUM, C.c_void_p(v.ctypes.data), 3, C.c_void_p(o.ctypes.data)) == 0 and o[0] == F16(1)
    v = np.array([-0.0, 0.0, np.nan], F16)
    assert L.dab_combine_ordered(_lib.F16, _lib.MAX, C.c_void_p(v.ctypes.data), 2, C.c_void_p(o.ctypes.data)) == 0
    assert o[0] == 0 and not np.signbit(o[0])
    assert L.dab_combine_ordered(_lib.F16, _lib.MIN, C.c_void_p(v.ctypes.data), 3, C.c_void_p(o.ctypes.data)) == 0 and np.isnan(o[0])


def test_host_float16_round_trip_matches_numpy():
    """dab_combine_ordered's host Float16 conversions: every bit pattern through a one-element fold, and random sums against NumPy."""
    from darray_b200 import _lib
    L = _lib.lib()
    allh = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(F16)
    o = np.zeros(1, F16)
    got = np.empty_like(allh)
    for i in range(0, allh.size, 1):
        if i % 257 and not (0x7c00 <= (i & 0x7fff) <= 0x7c00 + 3) and i > 0x10 and i < 0xffef:
            continue                                                        # a spread of patterns, all the edges
        L.dab_combine_ordered(_lib.F16, _lib.SUM, C.c_void_p(allh[i:i + 1].ctypes.data), 1, C.c_void_p(o.ctypes.data))
        got[i] = o[0]
        assert o.view(np.uint16)[0] == allh[i:i + 1].view(np.uint16)[0] or (np.isnan(o[0]) and np.isnan(allh[i]))
    rng = np.random.default_rng(1)
    pairs = rng.integers(0, 1 << 16, (20000, 2)).astype(np.uint16).view(F16)
    with np.errstate(all="ignore"):
        want = pairs[:, 0] + pairs[:, 1]
    for (a, b), w in zip(pairs, want):
        v = np.array([a, b], F16)
        L.dab_combine_ordered(_lib.F16, _lib.SUM, C.c_void_p(v.ctypes.data), 2, C.c_void_p(o.ctypes.data))
        assert (np.isnan(w) and np.isnan(o[0])) or o.view(np.uint16)[0] == np.asarray(w, F16).view(np.uint16)


def test_generated_sources_of_existing_expressions_unchanged():
    """The Float16 blocks are appended only to sources that use the type and the linear / partial kernels widen only for Float16: the
    sources of a corpus of Float32 / Float64 / integer / Bool / complex / Int128 expressions hash to what the parent commit generated
    (tests/golden/jit_sources.json, recorded with the same dab_jit_source accessor on the parent's dab_jit.cu)."""
    import hashlib
    import json
    from darray_b200 import _lib
    f = _lib.lib().dab_jit_source
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "jit_sources.json")))
    assert len(golden) >= 30
    for g in golden:
        n = len(g["args"])
        dts, ia = (C.c_int32 * max(n, 1))(*g["args"]), (C.c_int32 * max(n, 1))(*g["is_array"])
        ln = C.c_size_t()
        assert f(g["kind"], g["expr"].encode(), g["dtype"], g["op"], n, dts, ia, None, 0, C.byref(ln)) == 0
        buf = C.create_string_buffer(ln.value + 1)
        assert f(g["kind"], g["expr"].encode(), g["dtype"], g["op"], n, dts, ia, buf, ln.value, C.byref(ln)) == 0
        src = buf.raw[:ln.value]
        assert hashlib.sha256(src).hexdigest() == g["sha256"], g["expr"]
        assert b"jl_f16" not in src


# every exported elementwise function of the package applied to Float16 values: either it compiles for sm_90a or the tracer raises
# UnsupportedError naming Float16 (never a KeyError or an NVRTC failure)
def _exported_elementwise(dab):
    from darray_b200 import _broadcast as bc
    skip = {"broadcast", "broadcast_into", "copy", "deepcopy", "drandn", "map_", "map_bang", "map_inplace", "map_localparts", "Expr", "trace"}
    out = []
    for name in sorted(dir(dab)):
        obj = getattr(dab, name)
        if callable(obj) and getattr(obj, "__module__", "") == bc.__name__ and name not in skip and not isinstance(obj, type):
            out.append(name)
    return out


def _one_sweep_case(dab, name):
    import inspect
    f = getattr(dab, name)
    try:
        nparams = len([p for p in inspect.signature(f).parameters.values() if p.default is inspect.Parameter.empty])
    except (TypeError, ValueError):
        nparams = 1
    if name == "ifelse":
        return [(lambda c, x: dab.ifelse(c, x, 1j), ["bool", "f16"], "c128"), (lambda c, x: dab.ifelse(c, x, 2), ["bool", "f16"], "f16"),
                (lambda x: dab.ifelse(x, 1, 2), ["f16"], "i64")]
    if nparams >= 2:
        return [(lambda x, y: f(x, y), ["f16", "f16"], None), (lambda x, y: f(x, y), ["f16", "f64"], None), (lambda x, y: f(x, y), ["i32", "f16"], None)]
    return [(lambda x: f(x), ["f16"], None)]


def test_sweep_exported_functions_compile_or_refuse(dab):
    from darray_b200 import _lib
    from darray_b200._broadcast import _NPT, codegen, convert, trace
    names = _exported_elementwise(dab)
    assert {"cis", "angle", "complex", "real", "imag", "conj", "iszero", "Float16", "Int128", "widen", "sqrt", "erf", "jl_max", "mod",
            "deg2rad", "ifelse", "sec"} <= set(names)
    extra = [(lambda x: x == 1j, ["f16"], None), (lambda x: x * 1j, ["f16"], None), (lambda x: x, ["f16"], "c64"), (lambda x: x, ["f16"], "c128"),
             (lambda x, z: x + z, ["f16", "c64"], None), (lambda x: x // 2, ["f16"], None), (lambda x: x ** 2.5, ["f16"], None)]
    for name, (fn, tags, out) in [(n, c) for n in names for c in _one_sweep_case(dab, n)] + [("extra", c) for c in extra]:
        try:
            e = trace(fn, tags)
            o = out or e.jt
            src = codegen(convert(e, o)).encode()
        except dab.UnsupportedError as err:
            assert re.search("(?i)float16|f16", str(err)), (name, str(err))
            continue
        except (TypeError, dab.InexactError):                     # Julia's MethodError / InexactError for these operand types
            continue
        n = len(tags)
        dts = (C.c_int32 * n)(*[dab.dab_dtype(_NPT[t]) for t in tags])
        sz = C.c_size_t()
        st = _lib.lib().dab_jit_compile_check(src, dab.dab_dtype(_NPT[o]), n, dts, (C.c_int32 * n)(*([1] * n)), C.byref(sz))
        assert st == 0, (name, tags, src)


# ---- the Float16 host flow through the host-memory emulation of the C ABI -----------------------------------------------------------
import f16_hostmem  # noqa: E402

f16_hostmem.install()


@pytest.mark.parametrize("nw", [1, 3, 8])
def test_host_flow(hostmem, dab, nw):
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(nw)
    x = (rng.standard_normal((37, 29)) * 4).astype(F16)
    d = dab.distribute(x)
    assert d.dtype == F16 and np.array_equal(dab.to_array(d).view(np.uint16), x.view(np.uint16))
    assert np.array_equal(dab.to_array(dab.dzeros((5, 6), dtype=F16)), np.zeros((5, 6), F16))
    assert np.array_equal(dab.to_array(dab.dones((5, 6), dtype=F16)), np.ones((5, 6), F16))
    f = dab.dfill(F16(1.5), (11,))
    dab.fill_(f, F16(-2))
    assert f.dtype == F16 and np.all(dab.to_array(f) == F16(-2))
    r = dab.to_array(dab.drand((40, 3), dtype=F16, seed=7))
    from oracle import darray_oracle as orc
    k = orc.hash_u32(7, np.arange(120, dtype=np.uint64)) >> np.uint32(22)
    assert np.array_equal(r.reshape(-1, order="F"), (k.astype(np.float64) * 2.0 ** -10).astype(F16))
    g = dab.drandn((20, 5), dtype=F16, seed=3)
    assert g.dtype == F16 and np.array_equal(dab.to_array(g), dab.to_array(dab.drandn((20, 5), dtype=np.float64, seed=3)).astype(F16))
    # movers
    assert np.array_equal(np.asarray(d[2:9, ::3]).view(np.uint16), x[2:9, ::3].view(np.uint16))
    assert np.array_equal(np.asarray(d[[4, 0, 2], :]).view(np.uint16), x[[4, 0, 2], :].view(np.uint16))
    t = dab.copy_transposed(dab.transpose(d))
    assert np.array_equal(dab.to_array(t), x.T)
    c = dab.copy(d)
    c[0:3, :] = np.ones((3, 29), F16)
    xc = x.copy()
    xc[0:3, :] = 1
    assert np.array_equal(dab.to_array(c), xc)
    # broadcast: routed to the NVRTC kernel (never a hand-written real kernel), Julia's promotion
    a, b = F16(0.5), F16(0.25)
    y = dab.broadcast(lambda v: a * v + b, d)
    assert y.dtype == F16 and rt.last_kernel == "dab_broadcast_expr" and np.array_equal(dab.to_array(y), a * x + b)
    assert dab.broadcast(lambda v: v * 2.0, d).dtype == np.float64 and dab.broadcast(lambda v: v * 2, d).dtype == F16
    z = dab.similar(d, dtype=np.complex64)
    dab.broadcast_into(z, lambda v: v, d)
    assert np.array_equal(dab.to_array(z), x.astype(np.complex64))
    # reductions without and with dims
    ints = rng.integers(-3, 4, (37, 29)).astype(F16)
    di = dab.distribute(ints)
    assert dab.sum(di) == F16(ints.astype(np.float64).sum()) and isinstance(dab.sum(di), F16)
    assert dab.maximum(di) == ints.max() and dab.minimum(di) == ints.min() and dab.extrema(di) == (ints.min(), ints.max())
    assert dab.count(di, lambda v: v > 0) == int(np.count_nonzero(ints > 0))
    s1 = dab.sum(di, dims=1)
    assert s1.dtype == F16 and np.array_equal(dab.to_array(s1), ints.astype(np.float64).sum(axis=0, keepdims=True).astype(F16))
    m2 = dab.mean(di, dims=2)
    assert m2.dtype == F16 and np.array_equal(dab.to_array(m2), dab.to_array(dab.sum(di, dims=2)) / F16(29))
    exact = (ints.astype(np.float64) ** 2).sum()                          # chunk results are Float16 and fold in Float16: 1/2 ulp each
    assert abs(float(dab.dot(di, di)) - exact) <= nw * float(np.spacing(F16(exact))) and dab.isequal(di, ints)


def test_host_refusals_launch_nothing(hostmem, dab):
    rt = dab.init(workers_per_rank=2, use_dist=False)
    A = dab.distribute(np.ones((8, 8), F16))
    v = dab.distribute(np.ones(8, F16))
    I = dab.distribute(np.arange(1, 9, dtype=np.int64))
    m = dab.distribute(np.ones(8, np.bool_))
    l0 = hostmem.launches
    for call in [lambda: A @ np.ones(8, F16), lambda: A @ A, lambda: dab.lmul_diag(np.ones(8, F16), A), lambda: dab.sort(v),
                 lambda: dab.sortperm(v), lambda: dab.cumsum(v), lambda: dab.findmax(v), lambda: v[I], lambda: v[m],
                 lambda: dab.filter(lambda a: a > 0, v), lambda: dab.findall(lambda a: a > 0, v), lambda: v.__setitem__(I, F16(1)),
                 lambda: dab.mapslices(dab.sort, A, dims=1), lambda: dab.broadcast(dab.cis, v), lambda: dab.broadcast(dab.complex, v)]:
        with pytest.raises(dab.UnsupportedError, match="(?i)float16"):
            call()
    assert hostmem.launches == l0
    assert rt is not None
