"""GPU tests of findmax / findmin / argmax / argmin (K20, ``dab_findminmax.cu``) against the model of Julia's loops
(tests/findmax_oracle.py): exact equality of values (NaN payloads included) and indices, through the C entries on offset pointers and
through the public API on 1- and 8-worker layouts, with and without dims; the refusals launch nothing."""
import ctypes as C
import os

import numpy as np
import pytest

import findmax_oracle as fo

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets the K20 entry points too
    fo.install()

DTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_]
WHICH = {"findmax": fo.FINDMAX, "findmin": fo.FINDMIN}


def _nan(dtype, payload, neg=False):
    if np.dtype(dtype) == np.float32:
        return np.array([(0xFF800000 if neg else 0x7F800000) | payload], dtype=np.uint32).view(np.float32)[0]
    return np.array([(0xFFF0000000000000 if neg else 0x7FF0000000000000) | payload], dtype=np.uint64).view(np.float64)[0]


def _values(rng, dtype, n, special=True):
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return rng.random(n) < 0.3
    if dt.kind == "f":
        v = (rng.integers(-50, 50, n) / 4).astype(dt)            # many ties
        if special and n:
            k = max(1, n // 50)
            v[rng.integers(0, n, k)] = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf], dtype=dt), k)
        return v
    info = np.iinfo(dt)
    v = rng.integers(-100, 100, n).astype(dt)
    if special and n:
        v[rng.integers(0, n, max(1, n // 50))] = rng.choice(np.array([info.min, info.max, info.min + 1], dtype=dt), max(1, n // 50))
    return v


def _same(got, want, f):
    """Bit for bit; a NaN made by arithmetic (abs2, a general f) is only required to be a NaN -- the GPU's FP units return the canonical
    NaN, as the elementwise kernels do.  The identity and abs (a sign-bit operation in Julia) keep the payload."""
    if f is None or f is abs:
        return fo.same_bits(got, want)
    got, want = np.asarray(got), np.asarray(want)
    nan = np.isnan(want) if want.dtype.kind == "f" else np.zeros(want.shape, dtype=bool)
    return got.dtype == want.dtype and np.array_equal(np.isnan(got) if got.dtype.kind == "f" else nan, nan) and \
        fo.same_bits(got[~nan], want[~nan])


def _check_whole(dab, d, A, which, f=None):
    fn = dab.findmax if which == fo.FINDMAX else dab.findmin
    v, i = fn(f, d) if f is not None else fn(d)
    wv, wi = fo.find(which, A, f)
    assert _same(np.asarray([v]), np.asarray([wv]), f), (v, wv)
    assert i == fo.julia_index(A.shape, wi), (i, fo.julia_index(A.shape, wi))
    return v, i


def _c_entry(dab, rt, x, which, mapc=0, offset=0):
    """dab_findminmax on x[offset:] of a device copy of x (any 16-byte phase): (value, 0-based index)."""
    from darray_b200 import _lib
    buf = dab.B200Array.from_numpy(rt, x)
    slot = dab.B200Array.empty(rt, (16,), np.uint8)
    try:
        code = dab.dab_dtype(x.dtype)
        _lib.call("dab_findminmax", rt.ctx, code, which, mapc, None, C.c_void_p(buf.ptr + offset * x.dtype.itemsize), x.size - offset,
                  C.c_void_p(slot.ptr))
        s = slot.to_numpy()
    finally:
        buf.free()
        slot.free()
    return s[:x.dtype.itemsize].view(x.dtype)[0], int(s[8:16].view(np.int64)[0])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("which", ["findmax", "findmin"])
def test_every_dtype_and_map(dab, rt8, dtype, which):
    """Every dtype x {id, abs, abs2, a general traced f} on an 8-worker grid."""
    rng = np.random.default_rng(1)
    A = _values(rng, dtype, 40 * 37).reshape((40, 37), order="F")
    d = dab.distribute(A, dist=(2, 4))
    w = WHICH[which]
    _check_whole(dab, d, A, w)
    if np.dtype(dtype) != np.bool_:
        _check_whole(dab, d, A, w, abs)
        _check_whole(dab, d, A, w, lambda x: x * x)
        _check_whole(dab, d, A, w, lambda x: x - x * x)            # general f: the elementwise temporary
    d.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["findmax", "findmin"])
def test_special_float_values(dab, rt8, dtype, which):
    w, dt = WHICH[which], np.dtype(dtype)
    cases = [
        np.array([1, 3, 3, 2, 3], dtype=dt),                                             # ties keep the first
        np.array([1, _nan(dt, 5), 7, _nan(dt, 9), -np.inf], dtype=dt),                   # first NaN, payload kept
        np.array([np.inf, -np.inf, _nan(dt, 3, neg=True), np.inf], dtype=dt),             # NaN beside ±Inf
        np.array([_nan(dt, 11), _nan(dt, 1), _nan(dt, 2, neg=True)], dtype=dt),          # all NaN
        np.array([-0.0, 0.0, -0.0], dtype=dt),
        np.array([0.0, -0.0, 0.0], dtype=dt),
        np.array([-np.inf, -np.inf, -np.inf], dtype=dt),
        np.array([np.inf] * 3, dtype=dt),
    ]
    for A in cases:
        big = np.concatenate([np.full(5000, 0.5, dtype=dt), A, np.full(7000, 0.25, dtype=dt)])
        for arr in (A, big):
            d = dab.distribute(arr, procs=[1, 2, 3], dist=[3]) if arr.size >= 3 else dab.distribute(arr)
            _check_whole(dab, d, arr, w)
            _check_whole(dab, d, arr, w, abs)
            d.close()


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
def test_integer_extremes_and_wrapping_maps(dab, rt8, dtype):
    info = np.iinfo(dtype)
    A = np.array([3, info.min, info.max, info.min, -5, info.max], dtype=dtype)
    d = dab.distribute(A, procs=[1, 2], dist=[2])
    for w in (fo.FINDMAX, fo.FINDMIN):
        _check_whole(dab, d, A, w)
        _check_whole(dab, d, A, w, abs)                                                  # abs(typemin) == typemin
        _check_whole(dab, d, A, w, lambda x: x * x)
    d.close()


def test_bool_all_false_and_single_true(dab, rt8):
    for A in (np.zeros(10001, dtype=np.bool_), np.ones(10001, dtype=np.bool_)):
        d = dab.distribute(A)
        for w in (fo.FINDMAX, fo.FINDMIN):
            _check_whole(dab, d, A, w)
        d.close()
    for pos in (0, 4095, 9999, 10000):
        A = np.zeros(10001, dtype=np.bool_)
        A[pos] = True
        d = dab.distribute(A)
        assert dab.findmax(d) == (True, pos + 1) and dab.argmax(d) == pos + 1
        assert dab.argmin(d) == (2 if pos == 0 else 1)
        d.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_winner_at_tile_boundaries_and_behind_misaligned_pointers(dab, rt1, dtype):
    """The winner at 8191 / 8192 / 8193 (vector and tile edges) and in head / tail elements behind an offset pointer at the C entry."""
    dt = np.dtype(dtype)
    n = 3 * 8192 + 77
    for pos in (0, 1, 2, 8191, 8192, 8193, n - 70, n - 2, n - 1):
        for off in (0, 1, 3):
            if pos < off:
                continue
            x = np.zeros(n, dtype=dt)
            x[pos] = True if dt == np.bool_ else 7
            x[(pos + 4099) % n] = False if dt == np.bool_ else -7
            for w in (fo.FINDMAX, fo.FINDMIN):
                v, i = _c_entry(dab, rt1, x, w, 0, off)
                wv, wi = fo.find(w, x[off:])
                assert fo.same_bits(np.asarray([v]), np.asarray([wv])) and i == wi, (pos, off, w, v, i, wv, wi)


@pytest.mark.skipif(HOSTMEM, reason="a 2^31 + 5 element chunk is a device-memory case")
def test_winner_beyond_2_31_in_a_bool_chunk(dab, rt1):
    n = 2 ** 31 + 5
    d = dab.dzeros((n,), dtype=np.bool_)
    from darray_b200 import _lib
    ch = d.chunks[1]
    one = np.ones(1, dtype=np.uint8)
    _lib.call("dab_h2d", rt1.ctx, C.c_void_p(ch.ptr + 2 ** 31 + 3), C.c_void_p(one.ctypes.data), 1)
    assert dab.findmax(d) == (True, 2 ** 31 + 4)
    assert dab.findmin(d) == (False, 1)
    d.close()


@pytest.mark.parametrize("grid", [(2, 4), (4, 2), (8, 1), (1, 8)])
def test_eight_worker_grids_with_uneven_cuts_and_an_empty_chunk(dab, rt8, grid):
    rng = np.random.default_rng(5)
    A = _values(rng, np.float32, 9 * 30).reshape((9, 30), order="F")
    d = dab.distribute(A, dist=grid)
    for w in (fo.FINDMAX, fo.FINDMIN):
        _check_whole(dab, d, A, w)
        for dims in (1, 2, (1, 2)):
            _check_dims(dab, d, A, w, dims)
    d.close()
    # an empty chunk: 3 rows cut over 4 workers along dim 1
    B = _values(rng, np.float64, 3 * 20).reshape((3, 20), order="F")
    e = dab.distribute(B, dist=(4, 2)) if grid == (4, 2) else None
    if e is not None:
        assert any(c.size == 0 for c in e.chunks.values())
        for w in (fo.FINDMAX, fo.FINDMIN):
            _check_whole(dab, e, B, w)
            for dims in (1, 2, (1, 2)):
                _check_dims(dab, e, B, w, dims)
        e.close()


def test_cross_chunk_tie_follows_global_linear_order(dab, rt8):
    """Element (M, 1) of chunk (2, 1) comes before element (1, 2) of chunk (1, 1) in column-major order: it must win the tie."""
    M = 8
    A = np.zeros((M, 4), dtype=np.float32)
    A[M - 1, 0] = 5                                          # chunk (2, 1): rows 5..8, column 1
    A[0, 1] = 5                                              # chunk (1, 1): rows 1..4, column 2
    d = dab.distribute(A, procs=[1, 2, 3, 4], dist=(2, 2))
    assert dab.findmax(d) == (np.float32(5), (M, 1))
    A[M - 1, 0] = A[0, 1] = -5
    d2 = dab.distribute(A, procs=[1, 2, 3, 4], dist=(2, 2))
    assert dab.findmin(d2) == (np.float32(-5), (M, 1))
    for dims in (2, (1, 2)):
        _check_dims(dab, d, np.where(A == -5, 5, A).astype(np.float32), fo.FINDMAX, dims)
    d.close()
    d2.close()


def _check_dims(dab, d, A, which, dims, f=None):
    fn = dab.findmax if which == fo.FINDMAX else dab.findmin
    V, I = fn(f, d, dims=dims) if f is not None else fn(d, dims=dims)
    wv, wi = fo.find_dims(which, A, dims, f)
    got_v, got_i = dab.to_array(V), dab.to_array(I)
    assert _same(got_v, wv, f), (dims, got_v, wv)
    assert got_i.dtype == np.int64 and np.array_equal(got_i, wi), (dims, got_i, wi)
    V.close()
    I.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_dims_every_subset_of_a_3d_array(dab, rt8, dtype):
    rng = np.random.default_rng(7)
    A = _values(rng, dtype, 10 * 12 * 9).reshape((10, 12, 9), order="F")
    if np.dtype(dtype).kind == "f":
        A[3, 4, 5] = _nan(dtype, 3)
        A[7, 1, 2] = _nan(dtype, 4)
    for dist in ((2, 2, 2), (1, 8, 1), (8, 1, 1)):
        d = dab.distribute(A, dist=dist)
        for dims in (1, 2, 3, (1, 2), (1, 3), (2, 3), (1, 2, 3), 4, (2, 5), (1, 3, 7)):
            for w in (fo.FINDMAX, fo.FINDMIN):
                _check_dims(dab, d, A, w, dims)
                if np.dtype(dtype) != np.bool_ and dims in (1, (1, 3)):
                    _check_dims(dab, d, A, w, dims, abs)
                    _check_dims(dab, d, A, w, dims, lambda x: x * x - x)
        d.close()
    d = dab.distribute(A, dist=(2, 2, 2))
    I = dab.argmax(d, dims=(1, 3))
    assert np.array_equal(dab.to_array(I), fo.find_dims(fo.FINDMAX, A, (1, 3))[1])
    I.close()
    d.close()


@pytest.mark.skipif(HOSTMEM, reason="sizes that reach the split kernels")
@pytest.mark.parametrize("shape,dims", [((1 << 18, 8), 1), ((64, 1 << 14), 2), ((3, 1 << 17), 2), ((1 << 17, 3), 1), ((1 << 20,), 1),
                                        ((40, 50, 60), (1, 3)), ((1 << 17, 4, 64), (1, 3)), ((8, 4096, 2, 64), (2, 4))])
def test_dims_split_paths_on_one_worker(dab, rt1, shape, dims):
    rng = np.random.default_rng(11)
    A = _values(rng, np.float32, int(np.prod(shape))).reshape(shape, order="F")
    d = dab.distribute(A)
    for w in (fo.FINDMAX, fo.FINDMIN):
        _check_dims(dab, d, A, w, dims)
    d.close()


@pytest.mark.skipif(HOSTMEM, reason="sizes that reach the 16-byte strided kernel")
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
@pytest.mark.parametrize("shape", [(1 << 13, 37, 20), (1 << 15, 512), (1 << 20, 8)])
def test_dims_16_byte_strided_kernel(dab, rt1, dtype, shape):
    """dims=2 with whole 16-byte vectors of outputs along the first dim: the 16-byte strided kernel, with and without a split of red."""
    rng = np.random.default_rng(13)
    A = _values(rng, dtype, int(np.prod(shape))).reshape(shape, order="F")
    d = dab.distribute(A)
    for w in (fo.FINDMAX, fo.FINDMIN):
        _check_dims(dab, d, A, w, 2)
        _check_dims(dab, d, A, w, 2, abs)
    d.close()


def test_strided_view(dab, rt8):
    rng = np.random.default_rng(3)
    A = _values(rng, np.float64, 50 * 40).reshape((50, 40), order="F")
    d = dab.distribute(A)
    sub = d[3:47:3, 1:39:2]
    S = A[3:47:3, 1:39:2]
    for w in (fo.FINDMAX, fo.FINDMIN):
        _check_whole(dab, sub, S, w)
        _check_dims(dab, sub, S, w, 1)
    d.close()


def test_errors_launch_nothing(dab, rt8):
    from darray_b200 import _lib
    from darray_b200._darray import registry_size
    import scipy.sparse as sp
    e = dab.distribute(np.zeros((0, 5), dtype=np.float32))
    z = dab.distribute(np.ones((4, 4), dtype=np.complex64))
    s = dab.distribute(sp.random(10, 10, density=0.3, format="csc"))
    n0, r0 = rt8.launches(), registry_size()
    with pytest.raises(dab.ArgumentError, match="empty collection"):
        dab.findmax(e)
    with pytest.raises(dab.ArgumentError, match="collection slices must be non-empty"):
        dab.findmin(e, dims=1)
    with pytest.raises(TypeError):
        dab.findmax(z)
    with pytest.raises(TypeError):
        dab.argmin(z, dims=1)
    with pytest.raises(dab.UnsupportedError, match="sparse"):
        dab.findmax(s)
    zv = z[0:3, 0:2]                                            # a view is checked before it is copied
    n1 = rt8.launches()
    with pytest.raises(TypeError):
        dab.findmax(zv)
    with pytest.raises(TypeError):
        dab.findmin(zv, dims=2)
    assert rt8.launches() == n1
    assert rt8.launches() == n0 and registry_size() == r0
    V, I = dab.findmax(e, dims=2)                               # a zero-length kept dimension: empty results
    assert dab.to_array(V).shape == (0, 1) and dab.to_array(I).shape == (0, 1)
    for bad in (dict(dtype=_lib.C64, which=0, mapc=0), dict(dtype=_lib.F32, which=2, mapc=0), dict(dtype=_lib.F32, which=0, mapc=_lib.MAP_NEG)):
        st = _lib.lib().dab_findminmax(None, bad["dtype"], bad["which"], bad["mapc"], None, None, 1, None)
        assert st in (_lib.ERR_UNSUPPORTED, _lib.ERR_ARG)
    for a in (V, I, e, z, s):
        a.close()
