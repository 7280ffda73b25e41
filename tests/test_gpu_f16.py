"""Float16 DArrays on the GPU: conversions, elementwise arithmetic with Julia's "widen to Float32, operate, round to Float16" methods,
reductions on every dispatch path, data movement, and the refusals.

Exactness: NumPy's float16 operations are correctly rounded, and so is Julia's Float16 arithmetic for + - * / sqrt (24 >= 2*11 + 2), so
those are compared bit for bit (NaN as NaN).  Transcendental functions are Float16(f(Float32(x))) with CUDA's single-precision libdevice
kernels, within one Float16 ulp of float16(float32 f(x)).  Sums of small integers are exact.  Other sums follow the exact multi-worker
model: each chunk's sum rounded once to Float16, then a left fold of the chunk results in Float16 (whole-array reductions) or one fp64
fold of the chunk slabs rounded once (with dims)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F16 = np.float16
RTS = ["rt1", "rt2", "rt8"]
ALL16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(F16)     # every Float16 bit pattern


def bits(a):
    return np.ascontiguousarray(a).view(np.uint16 if np.asarray(a).dtype == F16 else (np.uint32 if np.asarray(a).dtype == np.float32 else np.uint64))


def same_or_nan(got, want):
    """Bit-identical, except that any NaN matches any NaN (arithmetic canonicalises payloads)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    bad = (gn != wn) | (~gn & (bits(got) != bits(want)))
    return int(bad.sum())


def ulps16(got, want):
    """Distance in Float16 ulps on the ordered integer line (NaN must match NaN)."""
    g = bits(np.asarray(got, F16)).astype(np.int32)
    w = bits(np.asarray(want, F16)).astype(np.int32)
    g = np.where(g & 0x8000, 0x8000 - g, g)
    w = np.where(w & 0x8000, 0x8000 - w, w)
    d = np.abs(g - w)
    nan = np.isnan(np.asarray(got, F16)) | np.isnan(np.asarray(want, F16))
    d = np.where(nan, np.where(np.isnan(np.asarray(got, F16)) == np.isnan(np.asarray(want, F16)), 0, 1 << 20), d)
    return d


SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 0.5, 65504.0, -65504.0, 6.1035156e-05, 5.9604645e-08, -5.9604645e-08, np.inf, -np.inf,
                    np.nan, 3.0, 1 / 3, 2048.0, 2049.0, 0.1, 1e-7, 32768.0], dtype=F16)


def test_every_float16_widens_exactly(dab, rt1):
    d = dab.distribute(ALL16)
    for T in (np.float32, np.float64):
        out = dab.similar(d, dtype=T)
        dab.broadcast_into(out, lambda x: x, d)
        assert np.array_equal(bits(dab.to_array(out)), bits(ALL16.astype(T)))     # NaN payloads widen bit for bit too


def test_float64_to_float16_rounds_once(dab, rt2):
    # just above a Float16 rounding midpoint by less than half a Float32 ulp: through Float32 the value lands ON the midpoint and
    # rounds to even; the single rounding of Float64 -> Float16 goes up
    h = ALL16[np.isfinite(ALL16) & (ALL16 > 0) & (ALL16 < F16(60000))].astype(np.float64)
    nxt = np.nextafter(h.astype(F16), F16(np.inf)).astype(np.float64)
    mid = (h + nxt) / 2
    tricky = np.concatenate([mid * (1 + 2.0 ** -40), mid * (1 - 2.0 ** -40), -mid * (1 + 2.0 ** -40), mid])
    assert np.count_nonzero(tricky.astype(np.float32).astype(F16) != tricky.astype(F16)) > 1000    # the set does tell the two apart
    rng = np.random.default_rng(3)
    rand = rng.standard_normal(1 << 24) * np.exp2(rng.integers(-30, 20, 1 << 24))
    for x in (tricky, rand):
        d = dab.distribute(x)
        out = dab.similar(d, dtype=F16)
        dab.broadcast_into(out, lambda v: v, d)
        assert same_or_nan(dab.to_array(out), x.astype(F16)) == 0
        f = dab.broadcast(lambda v: dab.Float16(v), d)
        assert f.dtype == F16 and same_or_nan(dab.to_array(f), x.astype(F16)) == 0


def test_integers_to_float16(dab, rt2):
    i32 = np.array([0, 1, -1, 2047, 2049, 4097, 65504, 65519, 65520, 65535, 70000, -70000, 2 ** 31 - 1, -2 ** 31], dtype=np.int32)
    i64 = np.concatenate([i32.astype(np.int64), np.array([2 ** 62, -2 ** 63, 2 ** 24 + 1, 65519], dtype=np.int64)])
    rng = np.random.default_rng(4)
    i32 = np.concatenate([i32, rng.integers(-70000, 70000, 100000).astype(np.int32)])
    for x in (i32, i64):
        d = dab.distribute(x)
        out = dab.similar(d, dtype=F16)
        dab.broadcast_into(out, lambda v: v, d)
        assert same_or_nan(dab.to_array(out), x.astype(np.float64).astype(F16)) == 0      # exact in Float64, one rounding, +-Inf past 65520
        g = dab.broadcast(lambda v, h: v * h, d, dab.dones(x.shape, dtype=F16))              # Int * Float16 promotes to Float16
        assert g.dtype == F16 and same_or_nan(dab.to_array(g), x.astype(np.float64).astype(F16)) == 0


@pytest.mark.parametrize("op", ["add", "sub", "mul", "div"])
def test_arithmetic_bit_exact(dab, rt2, op):
    f = {"add": lambda a, b: a + b, "sub": lambda a, b: a - b, "mul": lambda a, b: a * b, "div": lambda a, b: a / b}[op]
    a_s, b_s = np.meshgrid(SPECIAL, SPECIAL)
    rng = np.random.default_rng(5)
    ra = rng.integers(0, 1 << 16, 1 << 24).astype(np.uint16).view(F16)
    rb = rng.integers(0, 1 << 16, 1 << 24).astype(np.uint16).view(F16)
    with np.errstate(all="ignore"):
        for a, b in ((a_s.ravel(), b_s.ravel()), (ra, rb)):
            got = dab.broadcast(f, dab.distribute(a), dab.distribute(b))
            assert got.dtype == F16
            assert same_or_nan(dab.to_array(got), f(a, b)) == 0


def test_no_fused_multiply_add(dab, rt1):
    x = np.array([1 + 2 ** -10, 3.0, 1 / 3], dtype=F16)
    a, b = F16(1 - 2 ** -11), F16(-1.0)
    got = dab.to_array(dab.broadcast(lambda v: a * v + b, dab.distribute(x)))
    assert np.array_equal(bits(got), bits((a * x) + b))                       # two roundings, as Julia
    got3 = dab.to_array(dab.broadcast(lambda v: v ** 3, dab.distribute(x)))
    assert np.array_equal(bits(got3), bits(x * x * x))                         # literal_pow: x*x*x, rounded after each multiply


@pytest.mark.parametrize("name", ["sqrt", "abs", "neg", "floor", "ceil", "trunc", "round_"])
def test_unary_exhaustive_bit_exact(dab, rt2, name):
    f = {"neg": lambda v: -v, "abs": abs}.get(name) or getattr(dab, name)
    ref = {"sqrt": np.sqrt, "abs": np.abs, "neg": np.negative, "floor": np.floor, "ceil": np.ceil, "trunc": np.trunc, "round_": np.rint}[name]
    got = dab.broadcast(f, dab.distribute(ALL16))
    assert got.dtype == F16
    with np.errstate(all="ignore"):
        want = ref(ALL16)
    if name in ("abs", "neg"):
        assert np.array_equal(bits(dab.to_array(got)), bits(want))             # sign-bit operations keep NaN payloads
    else:
        assert same_or_nan(dab.to_array(got), want) == 0


@pytest.mark.parametrize("name", ["sin", "cos", "exp", "log", "tanh", "atan", "exp2", "log2", "expm1", "log1p", "cbrt", "erf"])
def test_transcendentals_within_one_ulp(dab, rt1, name):
    import scipy.special as sp
    ref = {"erf": sp.erf, "exp2": np.exp2, "log2": np.log2, "expm1": np.expm1, "log1p": np.log1p, "cbrt": np.cbrt}.get(name) or getattr(np, name)
    got = dab.broadcast(getattr(dab, name), dab.distribute(ALL16))
    assert got.dtype == F16
    with np.errstate(all="ignore"):
        want = ref(ALL16.astype(np.float32)).astype(np.float32).astype(F16)
    assert int(ulps16(dab.to_array(got), want).max()) <= 1


def test_max_min_comparisons(dab, rt1):
    a_s, b_s = np.meshgrid(SPECIAL, SPECIAL)
    a, b = a_s.ravel(), b_s.ravel()
    da, db = dab.distribute(a), dab.distribute(b)
    mx = dab.to_array(dab.broadcast(dab.jl_max, da, db))
    mn = dab.to_array(dab.broadcast(dab.jl_min, da, db))
    nan = np.isnan(a) | np.isnan(b)
    assert np.all(np.isnan(mx[nan])) and np.all(np.isnan(mn[nan]))
    assert np.array_equal(mx[~nan], np.maximum(a, b)[~nan]) and np.array_equal(mn[~nan], np.minimum(a, b)[~nan])
    z = (a == 0) & (b == 0) & (np.signbit(a) != np.signbit(b))                  # max(-0.0, 0.0) == 0.0, min == -0.0
    assert not np.any(np.signbit(mx[z])) and np.all(np.signbit(mn[z]))
    for f, ref in ((lambda x, y: x < y, np.less), (lambda x, y: x <= y, np.less_equal), (lambda x, y: x == y, np.equal),
                   (lambda x, y: x != y, np.not_equal), (lambda x, y: x > y, np.greater)):
        got = dab.broadcast(f, da, db)
        assert got.dtype == np.bool_ and np.array_equal(dab.to_array(got), ref(a, b))
    assert np.array_equal(dab.to_array(dab.broadcast(dab.isnan, da)), np.isnan(a))
    assert np.array_equal(dab.to_array(dab.broadcast(dab.isinf, da)), np.isinf(a))


def test_promotion_and_scalars(dab, rt2):
    x = np.linspace(-3, 3, 101).astype(F16)
    d = dab.distribute(x)
    assert dab.broadcast(lambda v: v * 2, d).dtype == F16                       # Int64 literal: Float16
    assert dab.broadcast(lambda v: v * 2.0, d).dtype == np.float64              # Python float: Float64 literal
    assert dab.broadcast(lambda v: v * np.float32(2), d).dtype == np.float32
    f32 = dab.distribute(x.astype(np.float32))
    r = dab.broadcast(lambda v: F16(1.5) * v, f32)                              # np.float16 scalar: a Float16 constant, Float32 result
    assert r.dtype == np.float32 and np.array_equal(dab.to_array(r), np.float32(1.5) * x.astype(np.float32))
    h = dab.broadcast(lambda v: F16(0.1) * v, d)
    assert h.dtype == F16 and np.array_equal(bits(dab.to_array(h)), bits(F16(0.1) * x))
    dab.rmul_(d, 3)
    assert np.array_equal(bits(dab.to_array(d)), bits(x * F16(3)))
    y = dab.distribute(np.ones(101, F16))
    dab.axpy_(2, dab.distribute(x), y)
    assert np.array_equal(bits(dab.to_array(y)), bits(F16(2) * x + F16(1)))


def exact16(x, axis=None):
    return np.sum(x.astype(np.float64), axis=axis)


@pytest.mark.parametrize("rtname", RTS)
@pytest.mark.parametrize("n", [0, 1, 7, 2047, 2048 * 8 + 5, 1 << 20, (1 << 22) + 3])
def test_sum_prod_max_min_paths(dab, request, rtname, n):
    request.getfixturevalue(rtname)
    rng = np.random.default_rng(n)
    ints = rng.integers(-3, 4, n).astype(F16)
    if n == 0:                                       # a DArray of length 0 has no processors: length 0 through the C ABI
        import ctypes as C
        from darray_b200 import _lib
        x = dab.B200Array.empty(dab.runtime(), (4,), F16)
        for op, want in ((_lib.SUM, 0), (_lib.PROD, 1)):
            slot = np.full(2, 0xFF, dtype=np.uint64)
            _lib.call("dab_reduce_host", dab.runtime().ctx, _lib.F16, op, _lib.MAP_ID, None, C.c_void_p(x.ptr), 0, C.c_void_p(slot.ctypes.data))
            assert slot.view(F16)[0] == F16(want)
        with pytest.raises(dab.DabError):
            _lib.call("dab_reduce_host", dab.runtime().ctx, _lib.F16, _lib.MAX, _lib.MAP_ID, None, C.c_void_p(x.ptr), 0, C.c_void_p(slot.ctypes.data))
        return
    d = dab.distribute(ints)
    sl = chunk_slices(dab, d)
    whole = lambda v: fold16([F16(v[c].astype(np.float64).sum()) for c in sl], "+")   # chunk sums rounded once, folded in Float16
    if n * 3 <= 2048:
        assert dab.sum(d) == F16(exact16(ints))                                 # small integers: exact
    s = dab.sum(d)
    assert isinstance(s, F16) and bits(s) == bits(whole(ints))
    if n == 0:
        return
    assert bits(dab.maximum(d)) == bits(ints.max()) and bits(dab.minimum(d)) == bits(ints.min())
    lo, hi = dab.extrema(d)
    assert lo == ints.min() and hi == ints.max() and isinstance(lo, F16)
    x = (rng.standard_normal(n) * 10).astype(F16)
    dx = dab.distribute(x)
    assert bits(dab.sum(dx)) == bits(whole(x))
    assert bits(dab.sum(dx, abs)) == bits(whole(np.abs(x)))
    with np.errstate(over="ignore"):
        assert bits(dab.sum(dx, lambda v: v * v)) == bits(whole(x * x))            # abs2 rounds x*x to Float16 first, as Julia
    assert int(ulps16(dab.mapreduce(lambda v: -v, "max", dx), (-x).max())) == 0
    assert dab.count(dx, lambda v: v > 0) == int(np.count_nonzero(x > 0))
    p = np.where(rng.random(n) < 0.5, F16(1), F16(-1)) * np.where(rng.random(n) < 0.01, F16(2), F16(1))
    pp = np.prod(p.astype(np.float64))
    if abs(pp) < 60000:
        assert dab.prod(dab.distribute(p)) == F16(pp)


def chunk_slices(dab, d):
    """Each chunk's part of the host array, in procs(d) order."""
    return [tuple(slice(lo - 1, hi) for lo, hi in d.layout.localindices(p)) for p in dab.procs(d)]


def fold16(parts, op):
    """dab_combine_ordered for Float16: a left fold in procs(d) order in Float16 arithmetic (NumPy's float16 + and * round the Float32
    result once, as Julia's Float16 methods do)."""
    r = parts[0]
    for p in parts[1:]:
        r = F16(r + p) if op == "+" else F16(r * p)
    return r


@pytest.mark.parametrize("rtname", RTS)
@pytest.mark.parametrize("n", [2047, 2048 * 8 + 5, (1 << 20) + 1, (1 << 22) + 3])
def test_whole_array_reductions_exact_across_workers(dab, request, rtname, n):
    """sum / prod / dot / norm(x, 1) of Float16 data whose chunk sums round: each chunk's S_k is rounded once to Float16, then the chunk
    results fold left to right in Float16, bit for bit."""
    request.getfixturevalue(rtname)
    rng = np.random.default_rng(n + 1)
    x = (rng.standard_normal(n) * 10).astype(F16)
    y = (rng.standard_normal(n) * 3).astype(F16)
    z = (rng.standard_normal(n) * 2.0 ** -8).astype(F16)                       # small: sums of |z| and z*z (subnormal) stay finite
    dx, dy, dz = dab.distribute(x), dab.distribute(y), dab.distribute(z)
    sl = chunk_slices(dab, dx)
    assert len(sl) == {"rt1": 1, "rt2": 2, "rt8": 8}[rtname]
    chunk = lambda v: [F16(v[s].astype(np.float64).sum()) for s in sl]
    for got, want in ((dab.sum(dx), fold16(chunk(x), "+")), (dab.sum(dz, abs), fold16(chunk(np.abs(z)), "+")),
                      (dab.norm(dz, 1), fold16(chunk(np.abs(z)), "+")), (dab.dot(dx, dz), fold16(chunk(x * z), "+")),
                      (dab.sum(dz, lambda v: v * v), fold16(chunk(z * z), "+"))):
        assert isinstance(got, F16) and np.isfinite(want) and bits(got) == bits(want), (got, want)
    assert bits(dab.mean(dx)) == bits(fold16(chunk(x), "+") / n)                 # sum / length in Float16 (Int promotes to Float16)
    # views at odd 2-byte offsets: dot and a general mapreduce take the view's values as a DArray of their own (fresh, aligned chunks)
    for lo in (1, 3, 7):
        v, w = dx[lo:].to_darray(), dz[lo:].to_darray()
        vs = chunk_slices(dab, v)
        part = lambda a: fold16([F16(a[s].astype(np.float64).sum()) for s in vs], "+")
        assert bits(dab.dot(v, w)) == bits(part(x[lo:] * z[lo:])), lo
        assert bits(dab.mapreduce(lambda a, b: a * b - b, "+", v, w)) == bits(part(x[lo:] * z[lo:] - z[lo:])), lo
    p = np.where(rng.random(n) < 0.5, F16(1), F16(-1))
    p[rng.choice(n, 12, replace=False)] *= F16(1.5)
    parts = [F16(np.prod(p[s].astype(np.float64))) for s in sl]                   # 1.5^k rounds to Float16 in each chunk, then again
    assert bits(dab.prod(dab.distribute(p))) == bits(fold16(parts, "*"))


@pytest.mark.parametrize("rtname", ["rt2", "rt8"])
def test_sum_dims_exact_across_workers(dab, request, rtname):
    """sum(d; dims) over a dimension split across chunks: each chunk's slab is rounded once to Float16, and phase 2 folds the slabs (and
    init) in fp64 and rounds once: R = Float16(init + sum_k Float16(S_k))."""
    request.getfixturevalue(rtname)
    rng = np.random.default_rng(31)
    A = np.asfortranarray((rng.standard_normal((20000, 7)) * 10).astype(F16))
    d = dab.distribute(A, dist=[{"rt2": 2, "rt8": 8}[rtname], 1])
    sl = chunk_slices(dab, d)
    assert len(sl) > 1 and all(s[1] == slice(0, 7) for s in sl), sl
    slabs = np.stack([A[s].astype(np.float64).sum(axis=0).astype(F16) for s in sl]).astype(np.float64)
    got = dab.to_array(dab.sum(d, dims=1))
    assert np.array_equal(bits(got), bits(slabs.sum(axis=0).astype(F16).reshape(1, 7)))
    got = dab.to_array(dab.reduce("+", d, dims=1, init=F16(0.5)))
    assert np.array_equal(bits(got), bits((0.5 + slabs.sum(axis=0)).astype(F16).reshape(1, 7)))


def test_sum_overflow_and_nan(dab, rt2):
    x = np.full(4, F16(40000))
    assert dab.sum(dab.distribute(x)) == F16(np.inf)
    assert dab.sum(dab.distribute(x), dims=1).dtype == F16
    assert np.isinf(dab.to_array(dab.sum(dab.distribute(x.reshape(2, 2)), dims=1))).all()
    y = np.array([1, np.nan, 3], F16)
    assert np.isnan(dab.sum(dab.distribute(y))) and np.isnan(dab.maximum(dab.distribute(y)))


def test_misaligned_view_and_long_chunk(dab, rt1):
    x = np.random.default_rng(9).integers(-2, 3, 100003).astype(F16)
    d = dab.distribute(x)
    for lo in (1, 3, 5, 7):                                                     # views at odd 2-byte offsets: head peel of the flat grid
        s = dab.sum(d[lo:])
        assert s == F16(exact16(x[lo:]))
        assert dab.maximum(d[lo:]) == x[lo:].max()


def test_more_than_2_31_elements(dab, rt1):
    n = (1 << 31) + 5
    d = dab.dfill(F16(2.0 ** -20), (n,))
    assert int(ulps16(dab.sum(d), F16(n * 2.0 ** -20))) <= 1
    assert dab.maximum(d) == F16(2.0 ** -20)
    d.close()


def slab_model(dab, d, v, ax):
    """sum(d; dims) of Float16 data: each chunk's slab (its part of v summed over ax) rounded once to Float16, then the slabs that share an
    output position summed in fp64 and rounded once (phase 2)."""
    acc = np.zeros(tuple(1 if k in ax else v.shape[k] for k in range(v.ndim)))
    for c in chunk_slices(dab, d):
        part = v[c].astype(np.float64).sum(axis=ax, keepdims=True).astype(F16)
        acc[tuple(slice(0, 1) if k in ax else c[k] for k in range(v.ndim))] += part
    return acc.astype(F16)


@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
@pytest.mark.parametrize("shape,dims", [((37, 29), 1), ((37, 29), 2), ((37, 29), (1, 2)), ((5, 6, 7), 2), ((5, 6, 7), (1, 3)),
                                        ((4, 3, 5, 6), (2, 4)), ((4, 3, 5, 6), 4), ((70000,), 1), ((3, 40000), 2)])
def test_reducedim(dab, request, rtname, shape, dims):
    request.getfixturevalue(rtname)
    rng = np.random.default_rng(11)
    ints = rng.integers(-3, 4, shape).astype(F16)
    d = dab.distribute(ints)
    ax = tuple(k - 1 for k in (dims if isinstance(dims, tuple) else (dims,)))
    s = dab.sum(d, dims=dims)
    assert s.dtype == F16
    want = exact16(ints, ax).reshape(s.dims)
    # dims that collapse into one reduced extent are reduced in one pass per chunk: exact model.  Other dims (e.g. (1, 3)) take one
    # pass per dimension, each rounded to Float16: within the ulps the slabs of the chunks add.
    one_pass = ax == tuple(range(ax[0], ax[-1] + 1))
    tol = max(1, len(dab.procs(d)) - 1)

    def check(got, v):
        if one_pass:
            assert np.array_equal(bits(got), bits(slab_model(dab, d, v, ax).reshape(got.shape)))
        else:
            assert int(ulps16(got, exact16(v, ax).reshape(got.shape).astype(F16)).max()) <= tol

    check(dab.to_array(s), ints)
    if max(np.prod([shape[a] for a in ax]), 1) * 3 < 2048:
        assert np.array_equal(dab.to_array(s), want.astype(F16))
    for op, ref in (("max", np.max), ("min", np.min)):
        r = dab.mapreduce(None, op, d, dims=dims)
        assert r.dtype == F16 and np.array_equal(dab.to_array(r), ref(ints, axis=ax, keepdims=True).reshape(r.dims))
    x = (rng.standard_normal(shape) * 4).astype(F16)
    dx = dab.distribute(x)
    check(dab.to_array(dab.sum(dx, abs, dims=dims)), np.abs(x))
    m = dab.to_array(dab.mean(dx, dims=dims))
    cnt = int(np.prod([shape[a] for a in ax]))
    assert m.dtype == F16 and np.array_equal(m, dab.to_array(dab.sum(dx, dims=dims)) / F16(cnt))    # sum ./ n in Float16
    c = dab.count(dx, lambda v: v > 0, dims=dims)
    assert np.array_equal(dab.to_array(c).ravel(), np.count_nonzero(x > 0, axis=ax).ravel())


def test_compositions(dab, rt8):
    rng = np.random.default_rng(12)
    x = rng.integers(-4, 5, (33, 17)).astype(F16)
    y = rng.integers(-4, 5, (33, 17)).astype(F16)
    dx, dy = dab.distribute(x), dab.distribute(y)
    assert dab.dot(dx, dy) == F16(np.sum(x.astype(np.float64) * y))
    assert int(ulps16(dab.norm(dx), F16(np.sqrt(np.sum(x.astype(np.float64) ** 2))))) <= 2
    assert dab.norm(dx, 1) == F16(np.abs(x.astype(np.float64)).sum())
    assert dab.norm(dx, np.inf) == np.abs(x).max()
    assert int(ulps16(dab.mean(dx), F16(x.astype(np.float64).mean()))) <= 2
    assert dab.isequal(dx, x) and not dab.isequal(dx, y) and dab.isequal(dab.copy(dx), dx)
    assert dab.extrema(dx) == (x.min(), x.max())
    assert dab.count(dx, lambda v: v == 0) == int(np.count_nonzero(x == 0))
    assert dab.all(dx, lambda v: v < 5) and not dab.any(dx, lambda v: v > 4)
    assert dab.sum(dab.broadcast(lambda a, b: a * b, dx, dy)) == F16(np.sum(x.astype(np.float64) * y))


def payload_data(shape, seed):
    """Random bit patterns, NaN payloads and signed zeros included."""
    return np.random.default_rng(seed).integers(0, 1 << 16, shape).astype(np.uint16).view(F16)


@pytest.mark.parametrize("rtname", RTS)
def test_movers_byte_exact(dab, request, rtname):
    request.getfixturevalue(rtname)
    x = payload_data((37, 29), 13)
    d = dab.distribute(x)
    assert np.array_equal(bits(dab.to_array(d)), bits(x))
    assert np.array_equal(bits(np.asarray(d[2:9, ::3])), bits(x[2:9, ::3]))
    assert np.array_equal(bits(np.asarray(d[[4, 0, 2], :])), bits(x[[4, 0, 2], :]))
    assert bits(d[5, 7]) == bits(x[5, 7])
    assert np.array_equal(bits(dab.to_array(dab.copy(d))), bits(x)) and np.array_equal(bits(dab.to_array(dab.deepcopy(d))), bits(x))
    t = dab.copy_transposed(dab.transpose(d))
    assert t.dtype == F16 and np.array_equal(bits(dab.to_array(t)), bits(np.ascontiguousarray(x.T)))
    r = dab.reshape(dab.distribute(x.ravel(order="F")), (29, 37))
    assert np.array_equal(bits(dab.to_array(r)), bits(x.reshape((29, 37), order="F")))
    v = d[1:30, 3:20]                                                            # a view at odd 2-byte offsets, crossing chunks
    assert np.array_equal(bits(dab.to_array(v.to_darray())), bits(x[1:30, 3:20]))
    w = payload_data((10, 29), 14)
    e = dab.distribute(x.copy())
    e[0:10, :] = w
    xe = x.copy()
    xe[0:10, :] = w
    assert np.array_equal(bits(dab.to_array(e)), bits(xe))
    e[3, 4] = F16(-0.0)
    xe[3, 4] = F16(-0.0)
    e[[1, 5], 2:4] = F16(7)
    xe[[1, 5], 2:4] = F16(7)
    assert np.array_equal(bits(dab.to_array(e)), bits(xe))
    f = dab.similar(d)
    dab.copyto(f, x)
    assert f.dtype == F16 and np.array_equal(bits(dab.to_array(f)), bits(x))
    g = dab.distribute(x, procs=[1], dist=[1, 1]) if rtname == "rt1" else dab.distribute(x, dist=[1, len(dab.procs(d))])
    h = dab.similar(g)
    dab.broadcast_into(h, lambda a: a, d)                                        # halo reads across layouts: the identity keeps payloads
    assert np.array_equal(bits(dab.to_array(h)), bits(x))


def test_constructors(dab, rt8):
    assert np.array_equal(bits(dab.to_array(dab.dzeros((13, 7), dtype=F16))), bits(np.zeros((13, 7), F16)))
    assert np.array_equal(bits(dab.to_array(dab.dones((13, 7), dtype=F16))), bits(np.ones((13, 7), F16)))
    f = dab.dfill(F16(1.5), (29,))
    assert f.dtype == F16 and np.all(dab.to_array(f) == F16(1.5))
    dab.fill_(f, F16(-0.0))
    assert np.all(bits(dab.to_array(f)) == 0x8000)
    r = dab.drand((50, 11), dtype=F16, seed=5)
    h = dab.to_array(r)
    from oracle import darray_oracle as orc
    u32 = (orc.rand_u01(5, 0, h.size) * 2.0 ** 24).astype(np.uint64)               # hash32 >> 8; Float16 takes hash32 >> 22
    assert np.array_equal(h.reshape(-1, order="F"), ((u32 >> 14).astype(np.float64) * 2.0 ** -10).astype(F16))
    assert np.array_equal(bits(dab.to_array(dab.drand((50, 11), dtype=F16, seed=5, procs=[1, 2, 3]))), bits(h))
    g = dab.drandn((300, 300), dtype=F16, seed=8)
    g64 = dab.to_array(dab.drandn((300, 300), dtype=np.float64, seed=8))
    assert g.dtype == F16 and np.array_equal(bits(dab.to_array(g)), bits(g64.astype(F16)))    # Float16(randn(Float64))


def test_refusals_launch_nothing(dab, rt2):
    A = dab.drand((64, 64), dtype=F16)
    v = dab.drand((64,), dtype=F16)
    A3 = dab.drand((4, 4, 3), dtype=F16)
    I = dab.distribute(np.arange(1, 65, dtype=np.int64))
    m = dab.broadcast(lambda a: a > 0.5, v)
    f32 = dab.drand((64, 64), dtype=np.float32)
    y = dab.dzeros((64,), dtype=F16)
    rt2.sync()
    before = rt2.launches()
    for call in [lambda: A @ np.ones(64, F16), lambda: A @ A, lambda: f32 @ np.ones(64, F16), lambda: dab.lmul_diag(np.ones(64, F16), A),
                 lambda: dab.rmul_diag(A, np.ones(64, F16)), lambda: dab.mul_(y, A, v),
                 lambda: dab.sort(v), lambda: dab.sortperm(v), lambda: dab.cumsum(v), lambda: dab.cumprod(A, dims=1),
                 lambda: dab.findmax(v), lambda: dab.argmin(A, dims=1), lambda: v[I], lambda: v[m], lambda: dab.filter(lambda a: a > 0, v),
                 lambda: v.__setitem__(I, F16(1)), lambda: v.__setitem__(m, F16(1)),
                 lambda: dab.mapslices(dab.sort, A, dims=1), lambda: dab.ppeval(dab.eigvals, A3),
                 lambda: dab.broadcast(lambda a: dab.complex(a), v)]:
        with pytest.raises(dab.UnsupportedError, match="(?i)float16|f16"):
            call()
    rt2.sync()
    assert rt2.launches() == before


def test_sweep_every_exported_elementwise_function(dab, rt2):
    """Every exported elementwise function of the package on a Float16 DArray (and with a Float64, an Int32 or a complex partner): the
    result matches a NumPy model of the traced expression, or the call raises UnsupportedError naming Float16 without a launch."""
    import sys
    sys.path.insert(0, __import__("os").path.dirname(__file__))
    import hostmem_abi as hm
    from test_cpu_f16 import _exported_elementwise, _one_sweep_case
    from darray_b200._broadcast import _NPT, trace
    rng = np.random.default_rng(21)
    host = {"f16": (rng.random(300) * 0.8 + 0.1).astype(F16), "f64": rng.random(300) + 0.5, "i32": rng.integers(1, 5, 300).astype(np.int32),
            "bool": rng.random(300) < 0.5}
    dev = {t: dab.distribute(v) for t, v in host.items()}
    extra = [(lambda x: x == 1j, ["f16"], None), (lambda x: x * 1j, ["f16"], None), (lambda x: x, ["f16"], "c64"), (lambda x: x, ["f16"], "c128")]
    served = refused = 0
    for name, (fn, tags, out) in [(n, c) for n in _exported_elementwise(dab) for c in _one_sweep_case(dab, n)] + [("extra", c) for c in extra]:
        rt2.sync()
        before = rt2.launches()
        try:
            e = trace(fn, tags)
            odt = _NPT[out or e.jt]
            if out is None:
                got = dab.broadcast(fn, *[dev[t] for t in tags])
            else:
                got = dab.similar(dev[tags[0]], dtype=odt)
                dab.broadcast_into(got, fn, *[dev[t] for t in tags])
        except dab.UnsupportedError as err:
            assert "float16" in str(err).lower() or "f16" in str(err), (name, str(err))
            rt2.sync()
            assert rt2.launches() == before, name
            refused += 1
            continue
        except (TypeError, dab.InexactError):                     # Julia's MethodError / InexactError for these operand types
            continue
        assert got.dtype == odt, (name, got.dtype, odt)
        with np.errstate(all="ignore"):
            args = [host[t] for t in tags]
            if e.op == "angle":                                   # angle(x::Real) = atan(zero(x), x)
                v = np.asarray(hm.eval_expr(e.args[0], args))
                want = np.arctan2(np.zeros_like(v), v).astype(odt)
            else:
                want = np.broadcast_to(np.asarray(hm.eval_expr(e, args)), (300,)).astype(odt)
        g = dab.to_array(got)
        if odt == np.bool_:
            assert np.array_equal(g, want), name
        else:
            # 8 Float16 ulps relative: the model evaluates on NumPy's float16 loops, whose transcendental functions are themselves off by
            # up to 3 ulps (arcsin); the bit-exact and one-ulp checks of each operation are the tests above
            assert np.allclose(g.astype(np.complex128), want.astype(np.complex128), rtol=8 * 2.0 ** -11, atol=1e-6, equal_nan=True), name
        served += 1
    assert served > 60 and refused >= 2
