"""ComplexF32 / ComplexF64 DArrays on the GPU: storage, elementwise arithmetic with Julia's complex methods, sums / products and the
other reductions, the conjugating transpose, and the refusals.  Layouts come from the 1-, 2- and 8-worker runtimes, sizes are uneven.

Exactness: + - * conj abs2 are compared bit for bit with a componentwise restatement written as real operations in T (never NumPy's
complex ufuncs); / inv abs against mpmath at 50 digits (each component within 4 eps(T) |exact|); sums against the exact sum of the
drand components (multiples of 2^-24, so integer accumulation is exact)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

mpmath = pytest.importorskip("mpmath")
mpmath.mp.dps = 50

CT = [np.complex64, np.complex128]
RTS = ["rt1", "rt2", "rt8"]


def comp(ct):
    return np.float32 if np.dtype(ct) == np.complex64 else np.float64


def eps(ct):
    return float(np.finfo(comp(ct)).eps)


def rnd(shape, ct, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    T = comp(ct)
    z = np.empty(shape, dtype=ct)
    z.real = (rng.standard_normal(shape) * scale).astype(T)
    z.imag = (rng.standard_normal(shape) * scale).astype(T)
    return z


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    u = np.uint32 if a.dtype == np.complex64 else np.uint64                       # bit patterns: signed zeros and NaN payloads count
    return np.array_equal(np.ascontiguousarray(a).view(u), np.ascontiguousarray(b).view(u))


# componentwise restatement of Julia's methods, every operation a real operation in T
def cmul(a, b):
    return _mk(a.real * b.real - a.imag * b.imag, a.real * b.imag + a.imag * b.real)


def _mk(re, im):
    out = np.empty(np.broadcast(re, im).shape, dtype=np.complex64 if np.asarray(re).dtype == np.float32 else np.complex128)
    out.real, out.imag = re, im
    return out


def mp_exact(z):
    return mpmath.mpc(float(z.real), float(z.imag))


def floor_of(ct):
    """The format's absolute resolution: below the normal range a correctly rounded result is off by up to half the subnormal spacing,
    which a relative bound cannot express."""
    return float(np.finfo(comp(ct)).smallest_subnormal)


def within(got, exact, ct, k=4):
    e = eps(ct)
    for part, ex in ((got.real, exact.real), (got.imag, exact.imag)):
        if abs(float(part) - float(ex)) > k * e * abs(exact) + floor_of(ct):
            return False
    return True


# ------------------------------------------------------------------------------------------------------------- reference replays
@pytest.mark.parametrize("rtname", RTS)
def test_reference_transpose_adjoint(dab, request, rtname):
    request.getfixturevalue(rtname)
    A = dab.drand((200, 100), dtype=np.complex128)
    h = dab.to_array(A)
    assert np.all(h.imag != 0) and np.all(h.real != h.imag)
    T = dab.transpose(A).copy()
    assert T.dtype == np.complex128 and same_bits(dab.to_array(T), np.asfortranarray(h.T))
    B = dab.drand((100, 200), dtype=np.complex128)
    hb = dab.to_array(B)
    H = dab.adjoint(B).copy()
    want = np.asfortranarray(hb.T)
    want.imag = -want.imag
    assert same_bits(dab.to_array(H), want)
    C32 = dab.distribute(rnd((37, 53), np.complex64, 3))
    w32 = np.asfortranarray(dab.to_array(C32).T)
    w32.imag = -w32.imag
    assert same_bits(dab.to_array(dab.adjoint(C32).copy()), w32)
    R = dab.drand((30, 20))
    assert np.array_equal(dab.to_array(dab.adjoint(R).copy()), dab.to_array(R).T)       # a real adjoint stays the transpose


def test_reference_scalar_math_subset(dab, rt2):
    a = dab.drand((20, 20))
    h = dab.to_array(a)
    z = dab.to_array(dab.broadcast(lambda x: dab.complex(x), a))
    assert z.dtype == np.complex128 and np.array_equal(z.real, h) and np.all(z.imag == 0)
    z2 = dab.to_array(dab.broadcast(lambda x, y: dab.complex(x, y), a, a))
    assert np.array_equal(z2.real, h) and np.array_equal(z2.imag, h)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.conj, a)), h)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.real, a)), h)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.imag, a)), np.zeros_like(h))
    c = dab.to_array(dab.broadcast(dab.cis, a))
    ulp = np.spacing(1.0)
    assert c.dtype == np.complex128
    assert np.all(np.abs(c.real - np.cos(h)) <= 2 * ulp) and np.all(np.abs(c.imag - np.sin(h)) <= 2 * ulp)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.angle, a)), np.zeros_like(h))       # angle(x >= 0) = 0
    Z = dab.drand((20, 20), dtype=np.complex128)
    hz = dab.to_array(Z)
    an = dab.to_array(dab.broadcast(dab.angle, Z))
    assert np.all(np.abs(an - np.arctan2(hz.imag, hz.real)) <= 2 * np.spacing(np.abs(np.arctan2(hz.imag, hz.real))))
    zc = dab.to_array(dab.broadcast(dab.conj, Z))
    assert np.array_equal(zc.real, hz.real) and np.array_equal(zc.imag, -hz.imag)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.real, Z)), hz.real)
    assert np.array_equal(dab.to_array(dab.broadcast(dab.imag, Z)), hz.imag)


# ------------------------------------------------------------------------------------------------------------- arithmetic
@pytest.mark.parametrize("ct", CT)
@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_arithmetic_bit_exact(dab, request, rtname, ct):
    request.getfixturevalue(rtname)
    T = comp(ct)
    shape = (67, 45)
    x, y = rnd(shape, ct, 1), rnd(shape, ct, 2)
    r = (np.random.default_rng(3).standard_normal(shape)).astype(T)
    dx, dy, dr = dab.distribute(x), dab.distribute(y), dab.distribute(r)
    got = lambda f, *a: dab.to_array(dab.broadcast(f, *a))                                           # noqa: E731
    assert same_bits(got(lambda a, b: a + b, dx, dy), _mk(x.real + y.real, x.imag + y.imag))
    assert same_bits(got(lambda a, b: a - b, dx, dy), _mk(x.real - y.real, x.imag - y.imag))
    assert same_bits(got(lambda a, b: a * b, dx, dy), cmul(x, y))
    assert same_bits(got(lambda a: dab.conj(a), dx), _mk(x.real, -x.imag))
    assert same_bits(got(lambda a: -a, dx), _mk(-x.real, -x.imag))
    assert np.array_equal(got(dab.abs2, dx), x.real * x.real + x.imag * x.imag)
    # with a real DArray: the real operand is not promoted to complex first
    assert same_bits(got(lambda a, b: a * b, dr, dx), _mk(r * x.real, r * x.imag))
    assert same_bits(got(lambda a, b: a + b, dr, dx), _mk(r + x.real, x.imag))
    assert same_bits(got(lambda a, b: a - b, dr, dx), _mk(r - x.real, -x.imag))
    assert same_bits(got(lambda a, b: a - b, dx, dr), _mk(x.real - r, x.imag))
    assert same_bits(got(lambda a, b: a / b, dx, dr), _mk(x.real / r, x.imag / r))
    # with scalars: a real scalar in the component type, a complex scalar of the array's type, an Int literal
    s = T(1.75)
    assert same_bits(got(lambda a: s * a, dx), _mk(s * x.real, s * x.imag))
    w = ct(0.5 - 2.25j)
    ws = np.full(shape, w, dtype=ct)
    assert same_bits(got(lambda a: a * w, dx), cmul(x, ws))
    assert same_bits(got(lambda a: a + 3, dx), _mk(x.real + T(3), x.imag))
    # a Python complex literal is a ComplexF64 constant: ComplexF32 arrays promote
    assert got(lambda a: a + 1j, dx).dtype == np.complex128
    # extruded size-1 dimensions
    col = rnd((67, 1), ct, 4)
    row = rnd((1, 45), ct, 5)
    assert same_bits(got(lambda a, b: a * b, dx, dab.distribute(col)), cmul(x, np.broadcast_to(col, shape)))
    assert same_bits(got(lambda a, b, c: a + b * c, dx, row, col),
                     _mk(x.real + cmul(np.broadcast_to(row, shape), np.broadcast_to(col, shape)).real,
                         x.imag + cmul(np.broadcast_to(row, shape), np.broadcast_to(col, shape)).imag))
    # dest .= ... into an existing complex DArray, from a real expression
    dz = dab.similar(dx)
    dab.broadcast_into(dz, lambda b: b * 2, dr)
    assert same_bits(dab.to_array(dz), _mk(r * T(2), np.zeros_like(r)))


def test_mixed_methods_at_inf(dab, rt1):
    """2.0 * complex(Inf, 0.0) is Inf + 0im in Julia (x*z multiplies each component), full complex multiplication would give NaN."""
    z = dab.distribute(np.array([complex(np.inf, 0.0), complex(0.0, np.inf), complex(np.inf, np.inf)], dtype=np.complex128))
    got = dab.to_array(dab.broadcast(lambda a: 2.0 * a, z))
    assert got[0] == complex(np.inf, 0.0) and not np.isnan(got[0].imag)
    assert got[1] == complex(0.0, np.inf) and not np.isnan(got[1].real)
    full = dab.to_array(dab.broadcast(lambda a: complex(2.0, 0.0) * a, z))                  # complex * complex: 0 * Inf = NaN
    assert np.isnan(full[0].imag)
    add = dab.to_array(dab.broadcast(lambda a: 1.0 + a, z))
    assert add[1] == complex(1.0, np.inf)
    sub = dab.to_array(dab.broadcast(lambda a: 1.0 - a, z))
    assert sub[0].real == -np.inf and sub[0].imag == 0.0 and np.signbit(sub[0].imag)
    div = dab.to_array(dab.broadcast(lambda a: a / 2.0, z))
    assert div[2] == complex(np.inf, np.inf)


@pytest.mark.parametrize("ct", CT)
def test_division_inverse_abs_against_mpmath(dab, rt2, ct):
    T = comp(ct)
    n = 3001
    x, y = rnd((n,), ct, 11, 3.0), rnd((n,), ct, 12, 0.2)
    big = 1e300 if ct == np.complex128 else 1e37
    tiny = 1e-300 if ct == np.complex128 else 1e-37
    # operands near the overflow / underflow thresholds whose quotient is representable: naive (ac + bd) / (c^2 + d^2) overflows or underflows
    x[:6] = [complex(big, big), complex(big, -big / 3), complex(tiny, tiny), complex(1.0, 2.0), complex(big, 1.0), complex(3.0, tiny)]
    y[:6] = [complex(big, big / 2), complex(-big / 7, big), complex(tiny, -tiny / 3), complex(big / 4, big / 8), complex(big / 2, tiny), complex(tiny, 1.0)]
    # subnormal components (the scaling by 2/eps^2 below 2 floatmin/eps): subnormal / subnormal, subnormal / small normal
    sub = 3e-310 if ct == np.complex128 else 3e-40
    x[6:10] = [complex(sub, -sub / 3), complex(sub / 5, sub), complex(sub, sub / 7), complex(1.0, -sub)]
    y[6:10] = [complex(sub / 2, sub), complex(-sub, sub / 9), complex(tiny, -tiny / 2), complex(3.0, sub / 11)]
    x, y = x.astype(ct), y.astype(ct)
    dx, dy = dab.distribute(x), dab.distribute(y)
    q = dab.to_array(dab.broadcast(lambda a, b: a / b, dx, dy))
    iv = dab.to_array(dab.broadcast(dab.inv, dy))
    ab = dab.to_array(dab.broadcast(abs, dx))
    assert q.dtype == ct and iv.dtype == ct and ab.dtype == T
    bad = []
    for i in range(n):
        ex = mp_exact(x[i]) / mp_exact(y[i])
        if not within(q[i], ex, ct):
            bad.append(("div", i, x[i], y[i], q[i]))
        if abs(1 / mp_exact(y[i])) < float(np.finfo(T).max) and not within(iv[i], 1 / mp_exact(y[i]), ct):   # 1/subnormal overflows
            bad.append(("inv", i, y[i], iv[i]))
        ea = mpmath.fabs(mp_exact(x[i]))
        if abs(float(ab[i]) - float(ea)) > 4 * eps(ct) * float(ea) + floor_of(ct):
            bad.append(("abs", i, x[i], ab[i]))
    assert not bad, bad[:5]


@pytest.mark.parametrize("ct", CT)
def test_abs_is_inf_when_a_component_is_inf(dab, rt1, ct):
    """Julia's hypot(x, y) is Inf when either argument is infinite, even when the other is NaN: abs in broadcasts and in the reduce maps."""
    inf, nan = np.inf, np.nan
    z = np.array([complex(inf, nan), complex(nan, -inf), complex(nan, 1.0), complex(-inf, 2.0), complex(3.0, 4.0)], dtype=ct)
    d = dab.distribute(z)
    a = dab.to_array(dab.broadcast(abs, d))
    assert np.isinf(a[0]) and np.isinf(a[1]) and np.isnan(a[2]) and np.isinf(a[3]) and a[4] == 5
    assert np.isnan(dab.sum(d, abs)) and np.isnan(dab.maximum(d, abs))                    # the NaN of element 3 propagates
    dz = dab.distribute(np.array([complex(inf, nan), complex(1.0, 0.0)], dtype=ct))
    assert np.isinf(dab.sum(dz, abs)) and np.isinf(dab.maximum(dz, abs)) and dab.minimum(dz, abs) == 1


# ------------------------------------------------------------------------------------------------------------- reductions
def exact_sum(h):
    """Sum of drand components (multiples of 2^-24) exactly, as Python floats of integer sums."""
    k = 2.0 ** 24
    re = int(np.sum(np.round(h.real.astype(np.float64) * k).astype(np.int64)))
    im = int(np.sum(np.round(h.imag.astype(np.float64) * k).astype(np.int64)))
    return complex(re / k, im / k)


@pytest.mark.parametrize("ct", CT)
def test_empty_sum_and_prod(dab, rt1, ct):
    """Length 0 through the C ABI (a DArray of length 0 has no processors): sum is 0, prod is 1 + 0im, in [0, 2 sizeof(T)) of the slot."""
    import ctypes as C
    from darray_b200 import _lib
    x = dab.B200Array.empty(rt1, (4,), ct)
    code = dab.dab_dtype(ct)
    for op, want in ((_lib.SUM, 0), (_lib.PROD, 1)):
        slot = np.full(2, 0xFF, dtype=np.uint64)
        _lib.call("dab_reduce_host", rt1.ctx, code, op, _lib.MAP_ID, None, C.c_void_p(x.ptr), 0, C.c_void_p(slot.ctypes.data))
        got = slot.view(np.uint8)[:np.dtype(ct).itemsize].view(ct)[0]
        assert got == want and not np.signbit(got.imag)
        assert not slot.view(np.uint8)[np.dtype(ct).itemsize:].any()
    x.free()


@pytest.mark.parametrize("ct", CT)
@pytest.mark.parametrize("n", [1, 31, (1 << 20) + 3])
@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_sum_exact(dab, request, rtname, ct, n):
    request.getfixturevalue(rtname)
    tol = 1e-6 if ct == np.complex64 else 1e-13
    d = dab.drand((n,), dtype=ct)
    h = dab.to_array(d)
    assert h.dtype == ct
    s = dab.sum(d)
    assert np.asarray(s).dtype == ct
    ex = exact_sum(h)
    for g, e in ((s.real, ex.real), (s.imag, ex.imag)):
        assert abs(float(g) - e) <= tol * max(abs(e), 1.0), (s, ex)
    if n > 64:                                               # a misaligned view: sum(view) goes through DArray(view)
        v = d[3:n - 5]
        sv = dab.sum(v)
        ev = exact_sum(h[3:n - 5])
        assert abs(float(sv.real) - ev.real) <= tol * abs(ev.real) and abs(float(sv.imag) - ev.imag) <= tol * abs(ev.imag)
        m = dab.mean(d)
        assert abs(complex(m) - ex / n) <= 2 * tol * abs(ex / n)


@pytest.mark.parametrize("ct", CT)
@pytest.mark.parametrize("n", [1, 31, 4099])
def test_prod_of_unit_modulus(dab, rt8, ct, n):
    th = np.random.default_rng(n).uniform(-np.pi, np.pi, n)
    z = np.empty(n, dtype=ct)
    z.real, z.imag = np.cos(th), np.sin(th)
    p = dab.prod(dab.distribute(z))
    ex = mpmath.mpc(1)
    for v in z:
        ex *= mp_exact(v)
    tol = 8 * eps(ct) + (n * 2.0 ** -52 if ct == np.complex128 else 0)
    assert abs(float(p.real) - float(ex.real)) <= tol and abs(float(p.imag) - float(ex.imag)) <= tol, (p, ex)


@pytest.mark.parametrize("ct", CT)
@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_map_reductions_dims_dot_norm(dab, request, rtname, ct):
    request.getfixturevalue(rtname)                        # rt1: one chunk per GPU, dab_mapreduce_all (sum(abs, z) in the fused kernel)
    T = comp(ct)
    x = rnd((203, 37), ct, 21)
    x[5, 3] = complex(np.nan, 1.0)
    x[100, 30] = complex(2.0, np.nan)
    x[7, 7] = 0
    d = dab.distribute(x)
    good = np.isfinite(x.real) & np.isfinite(x.imag)
    xg = np.where(good, x, 0).astype(ct)
    dg = dab.distribute(xg)
    a2 = (xg.real.astype(np.float64) ** 2 + xg.imag.astype(np.float64) ** 2)
    rtol = 1e-5 if ct == np.complex64 else 1e-12
    s2 = dab.sum(dg, dab.abs2)
    assert np.asarray(s2).dtype == T and abs(float(s2) - a2.sum()) <= rtol * a2.sum()
    s1 = dab.sum(dg, abs)
    assert abs(float(s1) - np.sqrt(a2).sum()) <= rtol * np.sqrt(a2).sum()
    assert abs(float(dab.maximum(dg, abs)) - np.sqrt(a2).max()) <= 4 * eps(ct) * np.sqrt(a2).max()
    assert dab.count(d, dab.isnan) == 2 and dab.any(d, dab.isnan) and not dab.all(d, dab.isnan)
    assert dab.count(d, lambda z: z != 0) == x.size - 1 and dab.count(d, dab.iszero) == 1
    for dims in (1, 2, (1, 2)):
        ax = tuple(k - 1 for k in ((dims,) if isinstance(dims, int) else dims))
        S = dab.to_array(dab.sum(dg, dims=dims))
        want = xg.astype(np.complex128).sum(axis=ax, keepdims=True)
        assert S.dtype == ct and np.allclose(S, want, rtol=rtol, atol=rtol)
        M = dab.to_array(dab.mean(dg, dims=dims))
        assert M.dtype == ct and np.allclose(M, want / np.prod([x.shape[k] for k in ax]), rtol=rtol, atol=rtol)
    y = rnd((203, 37), ct, 22)
    dy = dab.distribute(y)
    dt = complex(dab.dot(dg, dy))
    want = np.sum(np.conj(xg.astype(np.complex128)) * y.astype(np.complex128))
    assert abs(dt - want) <= rtol * np.sum(np.abs(xg) * np.abs(y))
    xx = complex(dab.dot(dg, dg))
    assert xx.imag == 0 and xx.real >= 0 and abs(xx.real - a2.sum()) <= rtol * a2.sum()
    assert abs(float(dab.norm(dg)) - np.sqrt(a2.sum())) <= rtol * np.sqrt(a2.sum())
    assert abs(float(dab.norm(dg, 1)) - np.sqrt(a2).sum()) <= rtol * np.sqrt(a2).sum()
    assert abs(float(dab.norm(dg, np.inf)) - np.sqrt(a2).max()) <= 4 * eps(ct) * np.sqrt(a2).max()
    assert abs(float(dab.norm(dg, -np.inf)) - np.sqrt(a2).min()) <= 4 * eps(ct) * max(np.sqrt(a2).min(), 1e-30)
    assert float(dab.norm(dg, 0)) == np.count_nonzero(xg)


@pytest.mark.parametrize("ct", CT)
def test_reduce_kernel_head_peel_and_reducedim_entry(dab, rt1, ct):
    """dab_reduce on a chunk that starts 8 bytes past a 16-byte boundary (a ComplexF32 head peel; ComplexF64 needs 16-byte alignment and
    refuses), and dab_reducedim called with the complex codes directly: SUM runs on the real view, other ops are refused with nothing
    launched."""
    import ctypes as C
    from darray_b200 import _lib
    code = dab.dab_dtype(ct)
    n = 5000
    h = rnd((n + 1,), ct, 51)
    buf = dab.B200Array.from_numpy(rt1, h)
    slot = np.zeros(2, dtype=np.uint64)
    isz = np.dtype(ct).itemsize
    if ct == np.complex64:
        _lib.call("dab_reduce_host", rt1.ctx, code, _lib.SUM, _lib.MAP_ID, None, C.c_void_p(buf.ptr + isz), n, C.c_void_p(slot.ctypes.data))
        got = slot.view(np.uint8)[:isz].view(ct)[0]
        want = h[1:].astype(np.complex128).sum()
        assert abs(got - want) <= 1e-5 * np.abs(h[1:]).sum()
        _lib.call("dab_reduce_host", rt1.ctx, code, _lib.SUM, _lib.MAP_ABS2, None, C.c_void_p(buf.ptr + isz), n, C.c_void_p(slot.ctypes.data))
        a2 = slot.view(np.uint8)[:4].view(np.float32)[0]
        want2 = (h[1:].real.astype(np.float64) ** 2 + h[1:].imag.astype(np.float64) ** 2).sum()
        assert abs(a2 - want2) <= 1e-5 * want2
    else:
        with pytest.raises(dab.ArgumentError):
            _lib.call("dab_reduce_host", rt1.ctx, code, _lib.SUM, _lib.MAP_ID, None, C.c_void_p(buf.ptr + 8), n, C.c_void_p(slot.ctypes.data))
    # dab_reducedim with the complex code: columns of a 40 x 125 matrix summed (inner 40, reduce 125, outer 1)
    out = dab.B200Array.empty(rt1, (40,), ct)
    _lib.call("dab_reducedim", rt1.ctx, code, _lib.SUM, _lib.MAP_ID, C.c_void_p(buf.ptr), 40, 125, 1, C.c_void_p(out.ptr), 0)
    want = h[:n].reshape((40, 125), order="F").astype(np.complex128).sum(axis=1)
    assert np.allclose(out.to_numpy(), want, rtol=1e-5 if ct == np.complex64 else 1e-13)
    rt1.sync()
    before = rt1.launches()
    for op, m in ((_lib.PROD, _lib.MAP_ID), (_lib.MAX, _lib.MAP_ID), (_lib.SUM, _lib.MAP_ABS)):
        for red in (0, 125, 1 << 16):                                             # empty, plain and "full reduction in disguise" shapes
            with pytest.raises(dab.UnsupportedError):
                _lib.call("dab_reducedim", rt1.ctx, code, op, m, C.c_void_p(buf.ptr), 1 if red == 1 << 16 else 40, red, 1, C.c_void_p(out.ptr), 0)
    rt1.sync()
    assert rt1.launches() == before
    out.free()
    buf.free()


@pytest.mark.parametrize("ct", CT)
def test_complex_scalar_arguments(dab, rt2, ct):
    """A complex scalar passed as an ARGUMENT (not a constant of f): ComplexF32 in its 8-byte slot, ComplexF64 as two Float64 slots."""
    x = rnd((300,), ct, 61)
    d = dab.distribute(x)
    s = ct(0.75 - 1.5j)
    sv = np.full(300, s, dtype=ct)
    assert same_bits(dab.to_array(dab.broadcast(lambda a, b: a * b, d, s)), cmul(x, sv))
    assert same_bits(dab.to_array(dab.broadcast(lambda b, a: b - a, s, d)), _mk(sv.real - x.real, sv.imag - x.imag))
    t = np.complex128(2.0 + 0.5j)                                                    # a ComplexF64 argument with a ComplexF32 array
    tv = np.full(300, t)
    assert same_bits(dab.to_array(dab.broadcast(lambda a, b: a * b, d, t)), cmul(x.astype(np.complex128), tv))
    m = complex(dab.mapreduce(lambda a, b: a * b, "+", d, t))
    want = cmul(x.astype(np.complex128), tv).sum()
    assert abs(m - want) <= 1e-12 * np.abs(cmul(x.astype(np.complex128), tv)).sum()


@pytest.mark.parametrize("ct", CT)
def test_rmul_axpy_keep_real_scalars_real(dab, rt1, ct):
    """rmul!(z, 2.0) multiplies each component (Julia's Complex * Real): Inf components stay Inf + 0im, no NaN from 0 * Inf."""
    T = comp(ct)
    z = np.array([complex(np.inf, 0.0), complex(0.0, -np.inf), complex(1.5, -2.5)], dtype=ct)
    d = dab.distribute(z)
    dab.rmul_(d, 2.0)
    got = dab.to_array(d)
    assert same_bits(got, _mk(z.real * T(2), z.imag * T(2)))
    y = dab.distribute(np.array([1 + 1j, 2, 3j], dtype=ct))
    dab.axpy_(2.0, d, y)
    assert same_bits(dab.to_array(y), _mk(T(2) * got.real + np.array([1, 2, 0], T), T(2) * got.imag + np.array([1, 0, 3], T)))


@pytest.mark.parametrize("ct", CT)
def test_equality(dab, rt2, ct):
    x = rnd((41, 9), ct, 31)
    d = dab.distribute(x)
    assert dab.isequal(d, x) and dab.isequal(d, dab.distribute(x.copy()))
    y = x.copy()
    y[3, 4] = complex(y[3, 4].real, np.nextafter(y[3, 4].imag, np.inf))
    assert not dab.isequal(d, y)
    n1 = x.copy()
    n1[0, 0] = complex(np.nan, 0.0)
    assert not dab.isequal(dab.distribute(n1), n1)                                                 # NaN != NaN, real part
    n2 = x.copy()
    n2[1, 1] = complex(0.0, np.nan)
    assert not dab.isequal(dab.distribute(n2), n2)                                                 # ... and imaginary part
    z0 = x.copy()
    z0[2, 2] = complex(-0.0, 0.0)
    z1 = x.copy()
    z1[2, 2] = complex(0.0, -0.0)
    assert dab.isequal(dab.distribute(z0), z1)                                                     # -0.0 == 0.0
    r = dab.distribute(x.real.copy())
    eq = dab.to_array(dab.broadcast(lambda z, a: z == a, d, r))
    assert np.array_equal(eq, x.imag == 0)


def test_full_size_sum_complex128(dab, rt1):
    n = 1 << 28                                                                                   # 4 GiB of ComplexF64
    d = dab.drand((n,), dtype=np.complex128, seed=77)
    s = dab.sum(d)
    from oracle import darray_oracle as orc
    ex_re = ex_im = 0
    step = 1 << 24
    for g in range(0, n, step):
        c = orc.rand_u01(77, 2 * g, 2 * min(step, n - g)).astype(np.float64)
        k = np.round(c * 2.0 ** 24).astype(np.int64)
        ex_re += int(k[0::2].sum())
        ex_im += int(k[1::2].sum())
    ex = complex(ex_re / 2.0 ** 24, ex_im / 2.0 ** 24)
    assert abs(s.real - ex.real) <= 1e-13 * ex.real and abs(s.imag - ex.imag) <= 1e-13 * ex.imag
    d.close()


# ------------------------------------------------------------------------------------------------------------- constructors / movers
@pytest.mark.parametrize("ct", CT)
def test_constructors_and_movers(dab, rt8, ct):
    T = comp(ct)
    assert np.array_equal(dab.to_array(dab.dzeros((13, 7), dtype=ct)), np.zeros((13, 7), ct))
    assert np.array_equal(dab.to_array(dab.dones((13, 7), dtype=ct)), np.ones((13, 7), ct))
    v = ct(1.5 - 0.25j)
    f = dab.dfill(v, (29,))
    assert f.dtype == ct and np.all(dab.to_array(f) == v)
    dab.fill_(f, ct(-2 + 3j))
    assert np.all(dab.to_array(f) == ct(-2 + 3j))
    r = dab.drand((50, 11), dtype=ct, seed=5)
    h = dab.to_array(r)
    from oracle import darray_oracle as orc
    u = orc.rand_u01(5, 0, 2 * h.size).astype(T)                   # element g = complex(u(2g), u(2g + 1)), layout-independent
    assert np.array_equal(h.reshape(-1, order="F").real, u[0::2]) and np.array_equal(h.reshape(-1, order="F").imag, u[1::2])
    r1 = dab.drand((50, 11), dtype=ct, seed=5, procs=[1, 2, 3])
    assert same_bits(dab.to_array(r1), h)
    g = dab.to_array(dab.drandn((300, 300), dtype=ct))
    assert g.dtype == ct and abs(g.mean()) < 0.02 and abs(np.mean(g.real ** 2) - 0.5) < 0.02 and abs(np.mean(g.imag ** 2) - 0.5) < 0.02
    x = rnd((23, 19), ct, 41)
    d = dab.distribute(x)
    assert same_bits(dab.to_array(d), x)
    c = dab.copy(d)
    assert same_bits(dab.to_array(c), x) and same_bits(dab.to_array(dab.deepcopy(d)), x)
    e = dab.similar(d)
    dab.copyto(e, x[::-1].copy())
    assert same_bits(dab.to_array(e), x[::-1])
    dab.copyto(e, d)
    assert same_bits(dab.to_array(e), x)
    assert same_bits(np.asarray(d[3:20:4, [5, 1, 18]]), x[3:20:4][:, [5, 1, 18]])
    assert same_bits(np.asarray(d[2:9, 4:15]), x[2:9, 4:15])
    assert d[4, 7] == x[4, 7] and type(d[4, 7]) is np.dtype(ct).type
    sub = d[1:22, 3:9].to_darray()
    assert same_bits(dab.to_array(sub), x[1:22, 3:9])
    vec = dab.distribute(x.reshape(-1, order="F").copy())
    rs = dab.reshape(vec, (19, 23))
    assert same_bits(dab.to_array(rs), x.reshape(-1, order="F").reshape((19, 23), order="F"))
    # a complex scalar into a real array is an InexactError; into a complex one it is served
    y = dab.distribute(rnd((40,), ct, 42))
    xr = dab.distribute(np.ones(40, dtype=T))
    with pytest.raises(dab.InexactError):
        dab.rmul_(xr, 1 + 2j)
    yh = dab.to_array(y)
    dab.rmul_(y, ct(0.5 + 1j))
    assert same_bits(dab.to_array(y), cmul(yh, np.full(40, ct(0.5 + 1j), dtype=ct)))
    yh = dab.to_array(y)
    xc = dab.distribute(rnd((40,), ct, 43))
    a = ct(2 - 1j)
    dab.axpy_(a, xc, y)
    ax = cmul(np.full(40, a, dtype=ct), dab.to_array(xc))
    assert same_bits(dab.to_array(y), _mk(ax.real + yh.real, ax.imag + yh.imag))


# ------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_launch_nothing(dab, rt2):
    z = dab.drand((64, 64), dtype=np.complex128)
    v = dab.drand((64,), dtype=np.complex64)
    z3 = dab.drand((4, 4, 3), dtype=np.complex128)
    rt2.sync()
    before = rt2.launches()
    for call, exc in [(lambda: dab.maximum(z), TypeError), (lambda: dab.minimum(z), TypeError), (lambda: dab.extrema(z), TypeError),
                      (lambda: dab.sort(v), TypeError), (lambda: dab.broadcast(lambda a: a < 1, z), TypeError),
                      (lambda: dab.broadcast(lambda a, b: dab.jl_max(a, b), z, z), TypeError),
                      (lambda: dab.broadcast(dab.exp, z), dab.UnsupportedError), (lambda: dab.broadcast(dab.sqrt, z), dab.UnsupportedError),
                      (lambda: dab.broadcast(dab.sin, z), dab.UnsupportedError), (lambda: dab.broadcast(lambda a: a ** 2, z), dab.UnsupportedError),
                      (lambda: dab.broadcast(lambda a: dab.mod(a, 2.0), z), dab.UnsupportedError),
                      (lambda: dab.broadcast(dab.floor, z), dab.UnsupportedError),
                      (lambda: dab.prod(z, dims=1), dab.UnsupportedError), (lambda: z @ np.ones(64, np.complex128), dab.UnsupportedError),
                      (lambda: z @ z, dab.UnsupportedError), (lambda: dab.lmul_diag(np.ones(64), z), dab.UnsupportedError),
                      (lambda: dab.rmul_diag(z, np.ones(64)), dab.UnsupportedError),
                      (lambda: dab.mapslices(dab.sort, z, dims=1), dab.UnsupportedError),
                      (lambda: dab.ppeval(dab.eigvals, z3), dab.UnsupportedError)]:
        with pytest.raises(exc):
            call()
    rt2.sync()
    assert rt2.launches() == before
