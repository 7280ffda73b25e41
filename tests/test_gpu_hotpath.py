"""GPU parity tests of the hot path, called through the C ABI (ctypes) and checked against the CPU oracle.

Bit-exact for elementwise / integer / index work; float reductions within 1e-6 relative of BOTH the exact (integer or fp64)
value and the Julia-like pairwise-fp32 oracle (BASELINE.json tolerance).
"""
import ctypes as C

import numpy as np
import pytest

from oracle import core as ocore
from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

F32 = np.float32
TOL = 1e-6


def dev(dab, rt, a):
    return dab.B200Array.from_numpy(rt, np.asfortranarray(a))


def same_bits(got, want):
    """Bit-identical, except that NaN payloads are not compared: GPU arithmetic returns the canonical quiet NaN (0x7fffffff)
    where x86 propagates the input payload; Julia's `==`-based tests cannot see the difference either (NaN != NaN)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    if not np.array_equal(np.isnan(got), nan):
        return False
    u = {4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    return np.array_equal(got.view(u)[~nan], want.view(u)[~nan])


# ---------------------------------------------------------------------------------------------- synthetic input generator
@pytest.mark.parametrize("n,off", [(1, 0), (7, 3), (4096, 0), (100003, 12345), (1 << 20, (1 << 40) + 5)])
def test_rand_u01_bit_exact(dab, rt1, n, off):
    from darray_b200 import _lib

    x = dab.B200Array.empty(rt1, (n,), F32)
    _lib.call("dab_rand_u01", rt1.ctx, _lib.F32, C.c_void_p(x.ptr), n, 1234, off)
    assert np.array_equal(x.to_numpy(), orc.rand_u01(1234, off, n))
    x64 = dab.B200Array.empty(rt1, (n,), np.float64)
    _lib.call("dab_rand_u01", rt1.ctx, _lib.F64, C.c_void_p(x64.ptr), n, 99, off)
    assert np.array_equal(x64.to_numpy(), orc.rand_u01(99, off, n, np.float64))


# ---------------------------------------------------------------------------------------------- K1-K3 elementwise
@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 1023, 1024, 4097, 1 << 20, (1 << 22) + 13])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_affine_bit_exact(dab, rt1, n, dtype):
    from darray_b200 import _lib

    rng = np.random.default_rng(n + 1)
    if np.dtype(dtype).kind == "f":
        x = rng.standard_normal(n).astype(dtype)
        a, b = dtype(1.5), dtype(0.25)
        if n > 4:
            x[:4] = [np.inf, -np.inf, np.nan, -0.0]
    else:
        x = rng.integers(-1000, 1000, n).astype(dtype)
        a, b = dtype(3), dtype(-7)
    dx = dev(dab, rt1, x)
    dy = dab.B200Array.empty(rt1, (n,), dtype)
    code = dab.dab_dtype(dtype)
    av, bv = np.asarray(a), np.asarray(b)
    _lib.call("dab_affine", rt1.ctx, code, C.c_void_p(dy.ptr), C.c_void_p(dx.ptr), C.c_void_p(av.ctypes.data), C.c_void_p(bv.ctypes.data), n)
    want = orc.affine_unfused(a, x, b)
    got = dy.to_numpy()
    assert same_bits(got, want)
    # in place (map!(f, d, d)) and on unaligned views (head/tail peel, mismatched alignment -> scalar kernel)
    _lib.call("dab_affine", rt1.ctx, code, C.c_void_p(dx.ptr), C.c_void_p(dx.ptr), C.c_void_p(av.ctypes.data), C.c_void_p(bv.ctypes.data), n)
    assert same_bits(dx.to_numpy(), want)
    if n > 16:
        es = np.dtype(dtype).itemsize
        x2 = dev(dab, rt1, x)
        _lib.call("dab_affine", rt1.ctx, code, C.c_void_p(dy.ptr + es), C.c_void_p(x2.ptr + es), C.c_void_p(av.ctypes.data),
                  C.c_void_p(bv.ctypes.data), n - 3)
        assert same_bits(dy.to_numpy()[1:n - 2], want[1:n - 2])
        _lib.call("dab_affine", rt1.ctx, code, C.c_void_p(dy.ptr), C.c_void_p(x2.ptr + es), C.c_void_p(av.ctypes.data),
                  C.c_void_p(bv.ctypes.data), n - 3)
        assert same_bits(dy.to_numpy()[:n - 3], want[1:n - 2])


@pytest.mark.parametrize("n", [8192, 8192 * 3 + 5, (1 << 22) + 12345])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int64])
def test_affine_tma_variant(dab, rt1, n, dtype):
    """The opt-in TMA-staged kernel (cp.async.bulk + mbarrier ring; dab_set_option "ew_tma") gives bit-identical results to the
    default kernel and to the oracle, including the ragged tail and in place."""
    rng = np.random.default_rng(n)
    x = (rng.standard_normal(n) * 100).astype(dtype)
    a, b = dtype(3), dtype(-7)
    want = orc.affine_unfused(a, x, b) if np.dtype(dtype).kind == "f" else (a * x + b)
    d = dab.distribute(x)
    y = dab.similar(d)
    rt1.set_option("ew_tma", 1)
    try:
        dab.broadcast_into(y, lambda v: a * v + b, d)
        assert rt1.last_kernel == "dab_affine" and same_bits(dab.to_array(y), want)
        dab.map_inplace(lambda v: a * v + b, d, d)
        assert same_bits(dab.to_array(d), want)
        assert same_bits(dab.to_array(dab.map_(lambda v: abs(v), y)), np.abs(want))
    finally:
        rt1.set_option("ew_tma", 0)


@pytest.mark.parametrize("key,value", [("gemm_rawhi", 0), ("gemm_simt", 0), ("gemm_kc", 64), ("gemv_phase", 1), ("gemv_t_cols", 8),
                                       ("gemv_t_waves", 4), ("spmv_group", 0)])
def test_set_option_refuses_kernel_choices(dab, rt1, key, value):
    """dab_set_option knows "ew_tma" and "combine_timeout_ms" only.  The GEMM, GEMV and SpMV kernels are chosen from the operands,
    so naming one of those choices, even with the value they are chosen with, is an unknown key."""
    with pytest.raises(dab.ArgumentError):
        rt1.set_option(key, value)


def test_affine_is_not_fma(dab, rt1):
    """a*x+b must be two roundings (Julia never contracts): pick values where fma(a,x,b) != (a*x)+b."""
    n = 1 << 16
    x = orc.rand_u01(7, 0, n) + F32(1)
    d = dab.distribute(x)
    dab.map_inplace(lambda v: F32(1.0000001) * v + F32(-1.0000001), d, d)
    want = F32(1.0000001) * x + F32(-1.0000001)
    fused = (x.astype(np.float64) * np.float64(F32(1.0000001)) + np.float64(F32(-1.0000001))).astype(F32)
    assert (want != fused).any(), "test vector does not discriminate FMA"
    assert np.array_equal(dab.to_array(d), want)


UNARY = [("abs", abs, np.abs), ("neg", lambda x: -x, np.negative), ("abs2", None, lambda x: x * x), ("sqrt", None, np.sqrt),
         ("floor", None, np.floor), ("ceil", None, np.ceil), ("sign", None, np.sign), ("inv", None, None)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int64])
def test_unary_binary_bit_exact(dab, rt2, dtype):
    rng = np.random.default_rng(5)
    shape = (37, 41)
    if np.dtype(dtype).kind == "f":
        a = (rng.standard_normal(shape) * 10).astype(dtype)
        b = (rng.standard_normal(shape) * 3 + 0.5).astype(dtype)
    else:
        a = rng.integers(-50, 50, shape).astype(dtype)
        b = rng.integers(1, 9, shape).astype(dtype)
    da, db = dab.distribute(a), dab.distribute(b)
    eq = lambda d, want: same_bits(dab.to_array(d), np.asfortranarray(want.astype(d.dtype)))
    assert eq(dab.map_(lambda x: abs(x), da), np.abs(a))
    assert eq(dab.map_(lambda x: -x, da), -a)
    assert eq(dab.map_(dab.abs2, da), a * a)
    assert eq(dab.broadcast(lambda x, y: x + y, da, db), a + b)
    assert eq(dab.broadcast(lambda x, y: x - y, da, db), a - b)
    assert eq(dab.broadcast(lambda x, y: x * y, da, db), a * b)
    assert eq(dab.broadcast(lambda x, y: x % y, da, db), np.fmod(a, b))          # Julia % == rem == C fmod
    assert eq(dab.broadcast(lambda x, y: dab.mod(x, y), da, db), np.mod(a, b))    # Julia mod == floored
    if np.dtype(dtype).kind == "f":
        assert eq(dab.map_(dab.sqrt, dab.map_(lambda x: abs(x), da)), np.sqrt(np.abs(a)))
        assert eq(dab.map_(dab.floor, da), np.floor(a))
        assert eq(dab.map_(dab.ceil, da), np.ceil(a))
        assert eq(dab.broadcast(lambda x, y: x / y, da, db), a / b)
        x = dtype(0.37)
        assert eq(dab.broadcast(lambda u, s: u + s, da, x), a + x)
        assert eq(dab.broadcast(lambda s, u: s - u, x, da), x - a)
        assert eq(dab.broadcast(lambda u, s: u * s, da, x), a * x)
        assert eq(dab.broadcast(lambda u, s: u / s, da, x), a / x)
        assert eq(dab.broadcast(lambda s, u: s / u, x, db), x / b)
        assert eq(dab.broadcast(lambda u, s: u % s, da, x), np.fmod(a, x))
    else:
        assert eq(dab.broadcast(lambda x, y: x // y, da, db), np.trunc(a / b).astype(dtype))  # Julia div truncates
        assert eq(dab.broadcast(lambda x, y: x & y, da, db), a & b)
        assert eq(dab.broadcast(lambda x, y: x | y, da, db), a | b)
        assert eq(dab.broadcast(lambda x, y: x ^ y, da, db), a ^ b)


# ---------------------------------------------------------------------------------------------- K4 whole-chunk reductions
@pytest.mark.parametrize("n", [1, 2, 15, 16, 17, 1000, 4096, 65537, (1 << 22) + 3])
def test_sum_f32_tolerance_and_exact(dab, rt1, n):
    x = orc.rand_u01(1234, 10, n)
    d = dab.distribute(x)
    got = dab.sum(d)
    assert got.dtype == np.float32  # Float32 sums return Float32 (add_sum does not widen floats)
    exact = orc.rand_u01_ksum(1234, 10, n) * 2.0 ** -24
    julia_like = float(ocore.sum_f32(x))
    assert abs(float(got) - exact) <= TOL * exact
    assert abs(float(got) - julia_like) <= TOL * exact
    # the kernel's fp64 carrier is the exactly rounded fp64 of the true sum to ~1e-9
    p = dab.prod(dab.distribute(np.full(min(n, 100), F32(1.01))))
    assert abs(float(p) - 1.01 ** min(n, 100)) <= 1e-5 * 1.01 ** min(n, 100)


@pytest.mark.parametrize("wpr", [1, 2, 8])
def test_sum_matches_left_fold_of_chunk_partials(dab, wpr):
    """reduce(op, results): the distributed sum must equal the LEFT fold, in procs order, in Float32, of the per-chunk results."""
    rt = dab.init(workers_per_rank=wpr, use_dist=False)
    try:
        n = 300007
        x = orc.rand_u01(5, 0, n)
        d = dab.distribute(x)
        res, parts = dab.mapreduce(None, "+", d, _partials=True)
        assert len(parts) == len(d.layout.pids) == min(wpr, n)
        fold = parts[0]
        for p in parts[1:]:
            fold = F32(fold + p)
        assert res == fold
        od = orc.distribute(x, nworkers=wpr)
        for p, ch in zip(parts, od.chunks):
            e = float(np.sum(ch.astype(np.float64)))
            assert abs(float(p) - e) <= TOL * e
    finally:
        dab.d_closeall()


def test_max_min_julia_semantics(dab, rt2):
    mx = lambda a: dab.maximum(dab.distribute(np.asarray(a, dtype=F32)))
    mn = lambda a: dab.minimum(dab.distribute(np.asarray(a, dtype=F32)))
    assert np.isnan(mx([1, np.nan, 3, 4])) and np.isnan(mn([1, 2, 3, np.nan]))
    z = mx([0.0, -0.0, -0.0, 0.0])
    assert z == 0 and not np.signbit(z)
    z = mx([-0.0, 0.0])
    assert z == 0 and not np.signbit(z)
    z = mn([0.0, -0.0, 0.0, 0.0])
    assert z == 0 and np.signbit(z)
    assert mx([-np.inf, -np.inf]) == -np.inf and mn([np.inf, np.inf]) == np.inf
    assert mx([-3, -1, -2]) == -1 and mn([5]) == 5
    x = (orc.rand_u01(3, 0, 1 << 20) - F32(0.5))
    x[777777] = F32(0.75)
    d = dab.distribute(x)
    assert dab.maximum(d) == x.max() and dab.minimum(d) == x.min()
    assert dab.maximum(d, abs) == np.abs(x).max() and dab.minimum(d, abs) == np.abs(x).min()
    assert dab.extrema(d) == (x.min(), x.max())
    x[5] = np.nan
    assert np.isnan(dab.maximum(dab.distribute(x)))
    x64 = x.astype(np.float64)
    assert np.isnan(dab.minimum(dab.distribute(x64)))
    # empty collection: the reference's distribute() itself throws "no processors given" (workers()[1:0], src/darray.jl:169-171);
    # an explicitly constructed empty DArray reduces like Base: sum -> 0, maximum -> ArgumentError
    with pytest.raises(ValueError):
        dab.distribute(np.zeros(0, dtype=F32))
    e = dab.dzeros((0,), procs=[1], dtype=F32)
    assert dab.sum(e) == 0 and dab.prod(e) == 1
    with pytest.raises(dab.ArgumentError):
        dab.maximum(e)


def test_reference_int_reductions(dab, rt8):
    """reference test/darray.jl:439-452 ("test max / min / sum"), exact on Int."""
    rng = np.random.default_rng(1234)
    a = (np.round(rng.random((100, 1000)) * 100) - 50).astype(np.int64)
    d = dab.distribute(a)
    assert dab.sum(d) == a.sum()
    assert dab.maximum(d) == a.max() and dab.minimum(d) == a.min()
    assert dab.maximum(d, abs) == np.abs(a).max() and dab.minimum(d, abs) == np.abs(a).min()
    assert dab.sum(d, abs) == np.abs(a).sum()
    assert dab.sum(d, dab.abs2) == (a * a).sum()
    assert dab.extrema(d) == (a.min(), a.max())
    a32 = a.astype(np.int32)
    s = dab.sum(dab.distribute(a32))
    assert s.dtype == np.int64 and s == a.sum()  # add_sum widens Int32


def test_reference_all_any_count_prod(dab, rt8):
    """reference test/darray.jl:456-518."""
    a = np.ones(100, dtype=bool)
    d = dab.distribute(a)
    assert dab.all(d) and dab.any(d)
    a[49] = False
    d = dab.distribute(a)
    assert not dab.all(d) and dab.any(d)
    d = dab.distribute(np.zeros(100, dtype=bool))
    assert not dab.all(d) and not dab.any(d)
    d = dab.dones((10, 10))
    assert not dab.all(d, lambda x: x > 1.0) and dab.all(d, lambda x: x > 0.0)
    a = np.ones((10, 10))
    a[9, 0] = 2.0
    d = dab.distribute(a)
    assert dab.any(d, lambda x: x == 1.0) and dab.any(d, lambda x: x == 2.0) and not dab.any(d, lambda x: x == 3.0)
    assert dab.count(d, lambda x: x == 2.0) == 1 and dab.count(d, lambda x: x == 1.0) == 99 and dab.count(d, lambda x: x == 0.0) == 0
    assert dab.prod(dab.distribute(np.full(10, 2, dtype=np.int64))) == 2 ** 10


def test_reference_reduce_map(dab, rt2):
    """reference test/darray.jl:238-257: D = fill(myid()) on (10,10) over 2 procs."""
    D = dab.darray(lambda I: np.full(dab.layout.shape_of(I), 0, dtype=np.int64), (10, 10), [1, 2])
    for pid, ch in D.chunks.items():
        ch.copy_from_host(np.full(ch.shape, pid, dtype=np.int64))
    assert dab.reduce("+", D) == 50 * 1 + 50 * 2
    D2 = dab.map_(lambda x: 1, D)
    assert isinstance(D2, dab.DArray) and dab.reduce("+", D2) == 100
    dab.map_inplace(lambda x: 1, D, D)
    assert dab.reduce("+", D) == 100


def test_reference_mapreduce_int_exact(dab, rt8):
    """reference test/darray.jl:286-294: mapreduce(f, opt, DA) exact for integer-valued f (Int128 there, Int64 here)."""
    rng = np.random.default_rng(7)
    fs = [(lambda x: 2 * x, lambda a: 2 * a), (lambda x: x ** 2, lambda a: a * a), (lambda x: x ** 2 + 2 * x - 1, lambda a: a * a + 2 * a - 1)]
    for _ in range(6):
        for f, fnp in fs:
            for op, red in (("+", np.sum), ("*", np.prod)):
                A = rng.integers(1, 6, rng.integers(2, 20)).astype(np.int64)
                DA = dab.distribute(A)
                assert dab.mapreduce(f, op, DA) - red(fnp(A)) == 0
                DA.close()


# ---------------------------------------------------------------------------------------------- K5/K6 mapreducedim
def test_reference_mapreducedim_int(dab, rt2):
    """reference test/darray.jl:298-304: 73x73 over 2 procs (uneven 37/36)."""
    D2 = dab.dones((73, 73), [1, 2], dtype=np.int64)
    A = np.ones((73, 73), dtype=np.int64)
    sq = lambda t: t * t
    for dims, ax in ((1, 0), (2, 1), ((1, 2), (0, 1))):
        R = dab.mapreduce(sq, "+", D2, dims=dims)
        assert isinstance(R, dab.DArray)
        assert np.array_equal(dab.to_array(R), (A * A).sum(axis=ax, keepdims=True))


def test_reference_irregular_chunks_sum_dims2(dab, rt2):
    """reference test/darray.jl:306-310: 3+7-row chunks, sum(D, dims=2) (dense here; the reference uses sprandn)."""
    rng = np.random.default_rng(3)
    r1, r2 = rng.standard_normal((3, 10)), rng.standard_normal((7, 10))
    D = dab.darray_from_chunks([r1, r2], (2, 1))
    assert D.dims == (10, 10) and D.indices == [((1, 3), (1, 10)), ((4, 10), (1, 10))]
    got = dab.to_array(dab.sum(D, dims=2))
    A = np.vstack([r1, r2])
    assert np.allclose(got, A.sum(axis=1, keepdims=True), rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("dms", [1, 2, 3, (1, 2), (1, 3), (2, 3), (1, 2, 3)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reference_mapreducedim_all_subsets(dab, rt8, dms, dtype):
    """reference test/darray.jl:319-332 (20^3 randn, all 7 dim subsets, with/without init) + Float32."""
    rng = np.random.default_rng(11)
    A = rng.standard_normal((20, 20, 20)).astype(dtype)
    DA = dab.distribute(A)
    od = orc.distribute(A, nworkers=8)
    assert DA.layout.grid == tuple(od.grid) and DA.indices == od.indices
    ax = tuple(d - 1 for d in ((dms,) if isinstance(dms, int) else dms))
    rtol = 1.5e-8 ** 0.5 if dtype == np.float64 else 1e-5
    sq = lambda t: t * t
    A64 = A.astype(np.float64)
    R = dab.mapreduce(sq, "+", DA, dims=dms)
    oR = orc.darray_mapreducedim(lambda a: a * a, "+", od, ax and [a + 1 for a in ax])
    assert R.layout.grid == tuple(oR.grid) and R.indices == oR.indices and R.layout.pids == oR.pids
    assert np.allclose(dab.to_array(R), (A64 * A64).sum(axis=ax, keepdims=True), rtol=1e-6 if dtype == np.float32 else 1e-13)
    assert np.allclose(dab.to_array(R), orc.to_array(oR), rtol=1e-6 if dtype == np.float32 else 1e-13)
    R = dab.mapreduce(sq, "+", DA, dims=dms, init=1.0)
    assert np.allclose(dab.to_array(R), (A64 * A64).sum(axis=ax, keepdims=True) + 1.0, rtol=1e-6 if dtype == np.float32 else 1e-13)
    R = dab.reduce("*", DA, dims=dms)
    assert np.allclose(dab.to_array(R), A64.prod(axis=ax, keepdims=True), rtol=rtol)
    R = dab.reduce("*", DA, dims=dms, init=2.0)
    assert np.allclose(dab.to_array(R), 2.0 * A64.prod(axis=ax, keepdims=True), rtol=rtol)
    R = dab.maximum(DA, dims=dms)
    assert np.array_equal(dab.to_array(R), A.max(axis=ax, keepdims=True))


def test_reference_sum_dims_errors(dab, rt8):
    """reference test/darray.jl:357-401."""
    rng = np.random.default_rng(2)
    A = rng.standard_normal((100, 100))
    DA = dab.distribute(A)
    with pytest.raises(dab.ArgumentError):
        dab.sum(DA, dims=-1)
    with pytest.raises(dab.ArgumentError):
        dab.sum(DA, dims=0)
    assert np.isclose(dab.sum(DA), A.sum(), rtol=1e-12)
    assert np.allclose(dab.to_array(dab.sum(DA, dims=1)), A.sum(axis=0, keepdims=True), rtol=1e-12)
    assert np.allclose(dab.to_array(dab.sum(DA, dims=2)), A.sum(axis=1, keepdims=True), rtol=1e-12)
    assert np.allclose(dab.to_array(dab.sum(DA, dims=3)), A, rtol=0)


@pytest.mark.parametrize("shape,dims", [((4096, 300), 1), ((300, 4096), 2), ((5, 7, 9), 2), ((100003, 3), 1), ((3, 100003), 2), ((33, 1), 1),
                                        ((1 << 21,), 1),
                                        # sub-warp-group kernel: G = 32/16/8/4/2 lanes per run, vector and scalar variants, ragged tails
                                        ((1000, 5000), 1), ((1001, 3000), 1), ((64, 200000), 1), ((36, 100001), 1), ((20, 100001), 1),
                                        ((7, 50000), 1), ((2, 40000), 1), ((3000, 2400), 1),
                                        # strided kernel with small inner / split r
                                        ((64, 128, 700), 2), ((3, 100000, 2), 2), ((1030, 5000), 2),
                                        # vectorised strided kernel (16-byte loads along inner), without and with the r-split
                                        ((65536, 600), 2), ((32768, 4100), 2)])
def test_reducedim_shapes_f32(dab, rt2, shape, dims):
    n = int(np.prod(shape))
    A = orc.rand_u01(21, 0, n).reshape(shape, order="F")
    DA = dab.distribute(A)
    got = dab.to_array(dab.sum(DA, dims=dims))
    want = A.astype(np.float64).sum(axis=dims - 1, keepdims=True)
    assert got.dtype == np.float32 and np.allclose(got, want, rtol=TOL, atol=0)
    mx = dab.to_array(dab.maximum(DA, dims=dims))
    assert np.array_equal(mx, A.max(axis=dims - 1, keepdims=True))
    Ai = (A * 1000).astype(np.int32)
    si = dab.to_array(dab.sum(dab.distribute(Ai), dims=dims))
    assert si.dtype == np.int64 and np.array_equal(si, Ai.astype(np.int64).sum(axis=dims - 1, keepdims=True))


def test_randomized_layouts_slices_and_reductions(dab, rt8):
    """Seeded random sweep: random shapes (1-3 dims), random explicit grids, random unit-range slices, every dims subset -- halo
    reads bit-exact, integer reductions exact, layouts identical to the oracle's."""
    rng = np.random.default_rng(2024)
    for case in range(40):
        nd = int(rng.integers(1, 4))
        shape = tuple(int(x) for x in rng.integers(1, 33, nd))
        # a random grid with <= 8 chunks, each dim split at most into its extent
        grid = []
        left = 8
        for s in shape:
            g = int(rng.integers(1, min(s, left) + 1))
            grid.append(g)
            left = max(1, left // g)
        A = rng.integers(-20, 20, shape).astype(np.int64)
        procs = list(range(1, int(np.prod(grid)) + 1))
        d = dab.distribute(A, procs=procs, dist=grid)
        od = orc.distribute(A, procs=procs, dist=grid)
        assert d.indices == od.indices and d.cuts == od.cuts, (shape, grid)
        sl = []
        for s in shape:
            lo = int(rng.integers(0, s))
            sl.append(slice(lo, int(rng.integers(lo + 1, s + 1))))
        assert np.array_equal(np.asarray(d[tuple(sl)]), A[tuple(sl)]), (shape, grid, sl)
        assert dab.sum(d) == A.sum() and dab.maximum(d) == A.max() and dab.extrema(d) == (A.min(), A.max())
        for k in range(1, nd + 1):
            dims = tuple(sorted(int(x) + 1 for x in rng.choice(nd, size=k, replace=False)))
            ax = tuple(x - 1 for x in dims)
            R = dab.sum(d, dims=dims)
            oR = orc.darray_mapreducedim(None, "+", od, dims)
            assert R.indices == oR.indices and R.layout.pids == oR.pids, (shape, grid, dims)
            assert np.array_equal(dab.to_array(R), A.sum(axis=ax, keepdims=True)), (shape, grid, dims)
        B = rng.integers(1, 5, shape).astype(np.int64)
        e = dab.distribute(B)                                        # default layout: usually differs from `grid`
        assert np.array_equal(dab.to_array(dab.broadcast(lambda x, y: x * y - 1, d, e)), A * B - 1)
        assert np.array_equal(dab.to_array(d + e), A + B)
        d.close()
        e.close()
    dab.d_closeall()
    assert dab.registry_size() == 0


def test_full_size_c4_c5(dab, rt8):
    """BASELINE configs 4 and 5 at full size on one GPU (8 workers, grid (2,4), 2 GiB chunks): sum(A, dims=1) of 65536 x 65536
    Float32 -- 64 sampled columns against the exact integer column sums, all columns through the identity sum(R) == sum(A) --
    and a 256 MiB slab read from non-owned chunks, bit-exact on sampled windows."""
    if rt8.device_info()["free_bytes"] < 24 * (1 << 30):
        pytest.skip("not enough free HBM")
    n = 65536
    A = dab.drand((n, n), dtype=F32, seed=11)
    assert A.layout.grid == (2, 4) and dab.layout.shape_of(A.indices[0]) == (32768, 16384)
    R = dab.sum(A, dims=1)
    assert R.dims == (1, n) and R.layout.grid == (1, 4) and R.layout.pids == [1, 3, 5, 7]   # owners: grid row 1 (src/mapreduce.jl:44)
    r = dab.to_array(R)[0]
    for c in list(range(0, n, 2048)) + [n - 1, 16383, 16384, 49151]:
        exact = ocore.rand_ksum(11, c * n, n) * 2.0 ** -24
        assert abs(float(r[c]) - exact) <= TOL * exact, c
    tot = float(dab.sum(A))
    assert abs(float(r.astype(np.float64).sum()) - tot) <= 2e-6 * tot
    mx = dab.to_array(dab.maximum(A, dims=1))[0]
    assert mx.max() == dab.maximum(A) and (mx <= 1).all() and (mx > 0.99).all()
    # C5: 2^26 elements = 256 MiB, rows 100..100+4096 x columns 20000..20000+16384: spans the chunks of workers 3 and 5
    # (grid row 1, grid columns 2 and 3), neither of which is the reading worker's own chunk
    sub = A[100:100 + 4096, 20000:20000 + 16384]
    dev = sub.to_device()
    from darray_b200 import _lib
    host = np.empty(4096, dtype=F32)
    for col in (0, 1, 7777, 16383):
        _lib.call("dab_d2h", rt8.ctx, C.c_void_p(host.ctypes.data), C.c_void_p(dev.ptr + 4 * 4096 * col), 4 * 4096)
        rt8.sync()
        assert np.array_equal(host, orc.rand_u01(11, (20000 + col) * n + 100, 4096))
    dev.free()


def test_full_size_8gib_chunk(dab, rt1):
    """north_star: "an 8 GiB-per-chunk Float32 DArray" = 2^31 elements: 64-bit indexing, in-place map!, sum, maximum."""
    n = 1 << 31
    if rt1.device_info()["free_bytes"] < 18 * (1 << 30):
        pytest.skip("not enough free HBM")
    from darray_b200 import _lib

    x = dab.drand((n,), dtype=F32, seed=77)
    s0 = float(dab.sum(x))
    assert abs(s0 / n - 0.5) < 1e-4
    dab.map_inplace(lambda v: 2 * v + 1, x, x)                      # config-1 function at the north-star chunk size
    ch = x.chunks[1]
    w = 4096
    host = np.empty(w, dtype=F32)
    for off in (0, (1 << 30) - 7, (1 << 31) - w, 3 * (1 << 29) + 12345):
        _lib.call("dab_d2h", rt1.ctx, C.c_void_p(host.ctypes.data), C.c_void_p(ch.ptr + 4 * off), 4 * w)
        rt1.sync()
        assert np.array_equal(host, F32(2) * orc.rand_u01(77, off, w) + F32(1))
    s1 = float(dab.sum(x))
    assert abs(s1 - (2 * s0 + n)) <= 2e-6 * s1
    assert 1 <= dab.minimum(x) and dab.maximum(x) <= 3   # 2*(1-2^-24)+1 rounds to 3.0f0
    # exact check of the last 2^24 elements (offset near 2^31: exercises the upper index range of the reduce kernel)
    out = np.zeros(2, dtype=np.uint64)
    off = n - (1 << 24)
    _lib.call("dab_reduce_host", rt1.ctx, _lib.F32, _lib.SUM, _lib.MAP_ID, None, C.c_void_p(ch.ptr + 4 * off), 1 << 24, C.c_void_p(out.ctypes.data))
    exact = 2 * ocore.rand_ksum(77, off, 1 << 24) * 2.0 ** -24 + (1 << 24)
    assert abs(out.view(np.float64)[1] - exact) <= 1e-9 * exact


# ---------------------------------------------------------------------------------------------- K8 halo getindex / makelocal
def test_reference_subdarray_to_array(dab, rt2):
    """reference test/darray.jl:182-218: 200x200 over 2 procs."""
    rng = np.random.default_rng(9)
    A = rng.random((200, 200))
    D = dab.distribute(A, procs=[1, 2])
    assert D.layout.grid == (1, 2)
    assert np.array_equal(np.asarray(D[0:150, 0:150]), A[0:150, 0:150])
    assert dab.localpart(D, 1).to_numpy()[0, 0] == D[0, 0]
    assert dab.localpart(D, 2).to_numpy()[0, 0] == D[0, 100]          # D[1,101] is worker 2's [1,1]
    assert np.array_equal(np.asarray(D[3, 22:176]), A[3, 22:176])
    assert np.array_equal(np.asarray(D[22:176, 196]), A[22:176, 196])
    assert np.array_equal(np.asarray(D[2:4, 98:100]), A[2:4, 98:100])  # spans both chunks
    assert np.array_equal(np.asarray(D[0, 0:4]), A[0, 0:4])
    dab.allowscalar(False)
    with pytest.raises(RuntimeError):
        D[0, 0]
    dab.allowscalar(True)


def test_reference_makelocal(dab, rt8):
    """reference test/darray.jl:740-757."""
    rng = np.random.default_rng(4)
    n = 5 * 9
    A = rng.standard_normal((n, n))
    dA = dab.distribute(A)
    for i in range(0, n, 7):
        a = dab.makelocal(dA, ((1, n), (i + 1, i + 1)))
        assert np.array_equal(a.to_numpy()[:, 0], A[:, i])
        a = dab.makelocal(dA, ((i + 1, i + 1), (1, n)))
        assert np.array_equal(a.to_numpy()[0, :], A[i, :])
    a = dab.makelocal(dA, ((1, 5), (1, 5)))
    assert np.array_equal(a.to_numpy(), A[:5, :5])
    # zero-copy branch: asking for exactly my chunk returns the chunk itself
    pid = dA.layout.pids[3]
    assert dab.makelocal(dA, dA.layout.localindices(pid), pid) is dA.chunks[pid]


def test_layout_matches_oracle_and_roundtrip(dab, rt8):
    for shape in [(50,), (3,), (1024, 1024), (73, 73), (20, 20, 20), (7, 1), (1, 9), (2, 3, 5, 4)]:
        A = np.arange(int(np.prod(shape)), dtype=np.float64).reshape(shape, order="F")
        d = dab.distribute(A)
        od = orc.distribute(A, nworkers=8)
        assert d.layout.grid == tuple(od.grid) and d.indices == od.indices and d.cuts == od.cuts and d.layout.pids == od.pids
        assert np.array_equal(dab.to_array(d), A)
        for pid in d.layout.pids:
            assert np.array_equal(dab.localpart(d, pid).to_numpy(), od.chunks[od.pids.index(pid)])
        d.close()
    assert dab.registry_size() == 0  # leak check (reference test/darray.jl:1079-1086)


# ---------------------------------------------------------------------------------------------- general broadcast (NVRTC)
def test_reference_broadcast_ops(dab, rt8):
    """reference test/darray.jl:880-905: extruded 1xn operand, scalar*array, nested, in-place from a plain Array."""
    nw = 8
    nrows, ncols = 20 * nw, 10 * nw
    rng = np.random.default_rng(8)
    A = rng.random((nrows, ncols))
    a = dab.distribute(A, procs=list(range(1, nw + 1)), dist=(1, nw))
    M = A.mean(axis=0, keepdims=True)
    m = dab.distribute(M)
    c = dab.broadcast(lambda x, y: x - y, a, m)
    assert isinstance(c, dab.DArray) and np.array_equal(dab.to_array(c), A - M)
    f = dab.broadcast(lambda s, e: s * e, 2, a)
    assert np.array_equal(dab.to_array(f), 2 * A)
    g = dab.broadcast(lambda x, y, z: x - y * dab.sin(z), a, m, c)
    assert np.allclose(dab.to_array(g), A - M * np.sin(A - M), rtol=1e-14, atol=1e-15)  # sin: libdevice vs libm, <= 2 ulp
    dab.broadcast_into(a, lambda o: o, np.ones((nrows, ncols)))
    assert dab.all(a, lambda x: x == 1.0)
    Z = np.zeros((nrows, ncols + 5))[:, 5:]
    dab.broadcast_into(a, lambda z: 3 + dab.abs2(z), Z)
    assert dab.all(a, lambda x: x == 3)
    with pytest.raises(dab.DimensionMismatch):
        dab.broadcast_into(a, lambda z: z, np.zeros((nrows + 1, ncols)))


def test_broadcast_mixed_types_and_layouts(dab, rt8):
    rng = np.random.default_rng(6)
    A = rng.standard_normal((64, 48)).astype(F32)
    B = rng.standard_normal((64, 48)).astype(np.float64)
    a = dab.distribute(A, dist=(8, 1))          # different layouts: args are halo-fetched into the dest chunks
    b = dab.distribute(B, dist=(2, 4))
    r = dab.broadcast(lambda x, y: x * y + 1, a, b)
    assert r.dtype == np.float64
    assert np.array_equal(dab.to_array(r), A.astype(np.float64) * B + 1)
    r = dab.broadcast(lambda x: x > 0, a)
    assert r.dtype == np.bool_ and np.array_equal(dab.to_array(r), A > 0)
    r = dab.broadcast(lambda x: 1.5 * x, a)   # Float64 literal * Float32 -> Float64 (Julia promotion)
    assert r.dtype == np.float64 and np.array_equal(dab.to_array(r), 1.5 * A.astype(np.float64))
    r = dab.broadcast(lambda x: F32(1.5) * x, a)
    assert r.dtype == np.float32 and np.array_equal(dab.to_array(r), F32(1.5) * A)
    # in-place broadcast of SMALLER operands into dest (materialize! instantiates with axes(dest)): row, column, scalar
    row = dab.distribute(B[:1, :])
    col = B[:, :1].copy()
    dab.broadcast_into(b, lambda v: v, row)
    assert np.array_equal(dab.to_array(b), np.broadcast_to(B[:1, :], B.shape))
    dab.broadcast_into(b, lambda u, v: u + v, row, col)
    assert np.array_equal(dab.to_array(b), B[:1, :] + B[:, :1])
    dab.broadcast_into(b, lambda: 7.0)
    assert (dab.to_array(b) == 7.0).all()
    with pytest.raises(dab.DimensionMismatch):
        dab.broadcast_into(b, lambda v: v, dab.distribute(B[:2, :]))


# ---------------------------------------------------------------------------------------------- full-size properties (BASELINE sizes)
def test_full_size_c2_affine_and_sum(dab, rt1):
    """C2: 2^30 Float32.  y .= a.*x .+ b checked bit-exact on 64 windows against the regenerated input; sum(x) against the
    exact integer sum (size-independent property of the counter-based input: sum = ksum * 2^-24)."""
    n = 1 << 30
    info = rt1.device_info()
    if info["free_bytes"] < 10 * (1 << 30):
        pytest.skip("not enough free HBM")
    x = dab.drand((n,), dtype=F32, seed=1234)
    exact = ocore.rand_ksum(1234, 0, 1 << 24)  # first 2^24 exactly; full-array exact sum via per-block GPU/CPU identity below
    s = dab.sum(x)
    mean = float(s) / n
    assert abs(mean - 0.5) < 1e-4
    # exact check on a prefix view (same kernel, n = 2^24)
    from darray_b200 import _lib
    out = np.zeros(2, dtype=np.uint64)
    ch = x.chunks[1]
    _lib.call("dab_reduce_host", rt1.ctx, _lib.F32, _lib.SUM, _lib.MAP_ID, None, C.c_void_p(ch.ptr), 1 << 24, C.c_void_p(out.ctypes.data))
    wide = out.view(np.float64)[1]
    assert abs(wide - exact * 2.0 ** -24) <= 1e-9 * exact * 2.0 ** -24
    y = dab.similar(x)
    a, b = F32(1.5), F32(0.25)
    dab.broadcast_into(y, lambda v: a * v + b, x)
    ych = y.chunks[1]
    w = 4096
    host = np.empty(w, dtype=F32)
    for k in range(64):
        off = (k * 16777259 + 12345) % (n - w)
        _lib.call("dab_d2h", rt1.ctx, C.c_void_p(host.ctypes.data), C.c_void_p(ych.ptr + 4 * off), 4 * w)
        rt1.sync()
        assert np.array_equal(host, a * orc.rand_u01(1234, off, w) + b)
    # linearity / sum identity at full size: sum(a*x+b) ~= a*sum(x) + b*n
    sy = float(dab.sum(y))
    assert abs(sy - (1.5 * float(s) + 0.25 * n)) <= 2e-6 * sy
    assert dab.maximum(y) <= a * F32(1) + b and dab.minimum(y) >= b


@pytest.mark.parametrize("log2n", [30, 31])
def test_full_size_reduce_exact_1e6(dab, rt1, log2n):
    """The headline reduce_kernel (dab_reduce / dab_mapreduce_all, hand-written path) at the BASELINE sizes -- 2^30 (4 GiB chunk) and
    2^31 (the north star's 8 GiB chunk) -- against the EXACT value at 1e-6 rel: the inputs are multiples of 2^-24 (x) / 2^-25 (y), so
    the oracle's uint64 accumulation over every element is a rounding-free ground truth.  Also maximum bit-exact."""
    n = 1 << log2n
    if rt1.device_info()["free_bytes"] < (9 << 30) * (n >> 30):
        pytest.skip("not enough free HBM")
    x = dab.drand((n,), dtype=F32, seed=4321)
    st = ocore.rand_stats(4321, 0, n, 1.5, 0.25)
    sx = dab.sum(x)
    exact_x = st["ksum"] * 2.0 ** -24
    assert abs(float(sx) - exact_x) <= TOL * exact_x, (sx, exact_x)
    assert dab.maximum(x) == st["xmax"]
    y = dab.similar(x)
    a, b = F32(1.5), F32(0.25)
    dab.broadcast_into(y, lambda v: a * v + b, x)
    assert st["inexact"] == 0
    exact_y = st["ysum"] * 2.0 ** -25
    sy = dab.sum(y)
    assert abs(float(sy) - exact_y) <= TOL * exact_y, (sy, exact_y)
    assert dab.maximum(y) == st["ymax"]
    # the fp64 carrier of the chunk result is far tighter than the Float32 result
    from darray_b200 import _lib
    out = np.zeros(2, dtype=np.uint64)
    ch = y.chunks[1]
    _lib.call("dab_reduce_host", rt1.ctx, _lib.F32, _lib.SUM, _lib.MAP_ID, None, C.c_void_p(ch.ptr), n, C.c_void_p(out.ctypes.data))
    assert abs(out.view(np.float64)[1] - exact_y) <= 1e-9 * exact_y
    assert out.view(np.float32)[0] == sy
    x.close()
    y.close()


# ---------------------------------------------------------------------------------------------- f1: fill! / copyto! / dfill / dzeros / dones
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64, np.bool_])
def test_fill_copyto_dfill(dab, rt8, dtype):
    """``fill!(A, x)`` (src/darray.jl:822-827), ``copyto!(dest::DArray, src::Array)`` (:679-687), ``dfill/dzeros/dones`` (:468-494)
    on a multi-chunk, uneven layout; every result gathered and compared bit-exactly."""
    dims = (37, 53)
    v = np.asarray(3 if dtype != np.bool_ else True, dtype=dtype)
    d = dab.dfill(v[()], dims, dtype=dtype)
    assert d.dtype == np.dtype(dtype) and d.dims == dims
    assert np.array_equal(dab.to_array(d), np.full(dims, v, dtype=dtype))
    z, o = dab.dzeros(dims, dtype=dtype), dab.dones(dims, dtype=dtype)
    assert np.array_equal(dab.to_array(z), np.zeros(dims, dtype)) and np.array_equal(dab.to_array(o), np.ones(dims, dtype))
    rng = np.random.default_rng(5)
    H = (rng.integers(-100, 100, dims) if dtype != np.bool_ else rng.integers(0, 2, dims)).astype(dtype)
    r = dab.copyto(d, H)
    assert r is d and same_bits(dab.to_array(d), H)
    # non-contiguous host source (a transposed view) and a second layout
    e = dab.dzeros(dims, dist=(4, 2), dtype=dtype)
    Ht = np.ascontiguousarray(H.T).T
    dab.copyto(e, Ht)
    assert same_bits(dab.to_array(e), H)
    with pytest.raises(dab.DimensionMismatch):
        dab.copyto(e, H[:, :-1])
    w = np.asarray(7 if dtype != np.bool_ else False, dtype=dtype)
    assert dab.fill_(e, w[()]) is e
    assert np.array_equal(dab.to_array(e), np.full(dims, w, dtype=dtype))
    assert np.array_equal(dab.to_array(d), H)               # fill! of e did not touch d


def test_copyto_pinned_large_and_pageable(dab, rt1):
    """The e2e leg of bench.py: copyto!(x::DArray, host) from pinned and from pageable memory, 2^26 Float32, bit-exact."""
    n = 1 << 26
    x = dab.dzeros((n,), dtype=F32)
    hp = dab.pinned_empty(rt1, (n,), F32)
    hp[:] = orc.rand_u01(77, 0, n)
    dab.copyto(x, hp)
    assert np.array_equal(dab.to_array(x), hp)
    pg = orc.rand_u01(78, 0, n)
    dab.copyto(x, pg)
    assert np.array_equal(dab.to_array(x), pg)
    st = ocore.rand_stats(78, 0, n, 1.0, 0.0)
    assert abs(float(dab.sum(x)) - st["ksum"] * 2.0 ** -24) <= TOL * st["ksum"] * 2.0 ** -24


def test_finalizer_releases_hbm(dab, rt1):
    """DArrays register a WeakRef + finalizer like the reference (src/darray.jl:46-49): dropping the last reference returns the
    localparts, so an iterative ``x = f(x)`` loop does not grow HBM."""
    import gc
    gc.collect()
    base = dab.registry_size()
    x = dab.dones((1 << 20,), dtype=F32)
    for _ in range(50):
        x = dab.map_(lambda v: v + 1, x)                   # each iteration drops the previous array
    gc.collect()
    assert dab.registry_size() == base + 1
    assert float(dab.sum(x)) == 51.0 * (1 << 20)
    x.close()
    assert dab.registry_size() == base


def test_uint8_is_not_bool(dab, rt1):
    with pytest.raises(dab.UnsupportedError):
        dab.distribute(np.array([2, 3, 4], dtype=np.uint8))
