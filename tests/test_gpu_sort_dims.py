"""GPU tests of ``sort(A; dims)`` and ``sortperm(A; dims)``: K26 (``dab_sortperm_slices``) on both of its paths against the per-fibre
stable ``isless`` permutation of oracle/darray_oracle.py mapped to global linear indices, and the distributed flow against the same model,
against ``mapslices(sort, A, dims)`` and against the DVector samplesort.  Everything here is integer / bit-pattern work: results must
equal the model exactly."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                      # the emulated C ABI gets K26 (and K21, K13) too
    import sort_dims_hostmem
    sort_dims_hostmem.install()

L = 4096                                                         # DAB_SORTPERM_SLICES_SMEM_LEN
DTYPES = [np.float32, np.float64, np.int32, np.int64]
LENS = (1, 2, 31, 32, 33, 1000, L, L + 1, 3 * L)


@pytest.fixture(autouse=True)
def _k13_on_the_emulation():
    if HOSTMEM:
        import sort_dims_hostmem
        from darray_b200 import _lib
        sort_dims_hostmem.install_slices(_lib._lib)
    yield


# ---- model ---------------------------------------------------------------------------------------------------------------------------


def _order_last_axis(k: np.ndarray) -> np.ndarray:
    """``jl_sortperm_stable`` of every row of a 2-D key array (one fibre per row), vectorised."""
    if k.dtype.kind != "f":
        return np.argsort(k, axis=-1, kind="stable")
    nan = np.isnan(k)
    return np.lexsort((~np.signbit(k) & ~nan, np.where(nan, 0, k), nan), axis=-1)


def model_perm(keys: np.ndarray, dim: int, lo=None, gdims=None) -> np.ndarray:
    """sortperm(keys; dims=dim) of a chunk at 0-based offset ``lo`` of an array of ``gdims``: 1-based global linear indices."""
    N = keys.ndim
    lo = [0] * N if lo is None else list(lo)
    gdims = list(keys.shape) if gdims is None else list(gdims)
    ax = dim - 1
    kk = np.moveaxis(keys, ax, -1)
    rows = kk.reshape(-1, keys.shape[ax])
    order = _order_last_axis(rows).reshape(kk.shape)
    G = np.cumprod([1] + gdims[:-1]).astype(np.int64)
    gidx = np.ones(keys.shape, dtype=np.int64)
    for k in range(N):
        sh = [1] * N
        sh[k] = keys.shape[k]
        gidx = gidx + ((lo[k] + np.arange(keys.shape[k], dtype=np.int64)) * G[k]).reshape(sh)
    return np.moveaxis(np.take_along_axis(np.moveaxis(gidx, ax, -1), order, axis=-1), -1, ax)


def test_model_is_the_oracle_per_fibre():
    """The vectorised model equals ``jl_sortperm_stable`` fibre by fibre (NaNs of both signs, signed zeros, ties)."""
    rng = np.random.default_rng(3)
    for T in DTYPES:
        a = _data(T, 37 * 11, rng, "specials" if np.dtype(T).kind == "f" else "repeated").reshape((37, 11), order="F")
        got = model_perm(a, 1)
        for j in range(11):
            assert np.array_equal(got[:, j], orc.jl_sortperm_stable(a[:, j]) + 1 + 37 * j)


# ---- data ----------------------------------------------------------------------------------------------------------------------------


def _data(T, n, rng, kind="full"):
    T = np.dtype(T)
    if kind == "full":
        if T.kind == "i":
            return rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T, endpoint=True)
        return (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(T)
    if kind == "specials":
        if T.kind == "i":
            a = _data(T, n, rng)
            a[rng.integers(0, n, max(1, n // 10))] = np.iinfo(T).min
            a[rng.integers(0, n, max(1, n // 10))] = np.iinfo(T).max
            return a
        a = np.round(rng.standard_normal(n), 1).astype(T)           # ties among the finite values too
        U = np.uint32 if T.itemsize == 4 else np.uint64
        sp = (np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800123, 0xFFFFFFFF], dtype=U)
              if T.itemsize == 4 else
              np.array([0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000123,
                        0xFFFFFFFFFFFFFFFF], dtype=U))
        idx = rng.integers(0, n, max(1, n // 3))
        a.view(U)[idx] = sp[rng.integers(0, len(sp), idx.size)]
        return a
    if kind == "equal":
        return np.full(n, 7, dtype=T)
    if kind == "repeated":                                       # 50 values repeated
        return rng.choice(_data(T, 50, rng, "specials"), n)
    raise ValueError(kind)


KINDS = ("full", "specials", "equal", "repeated")


# ---- the C entry ---------------------------------------------------------------------------------------------------------------------


def _k26(dab, rt, keys: np.ndarray, dim: int, lo=None, gdims=None, vals: np.ndarray = None):
    """dab_sortperm_slices on one device chunk: (perm, vals_out) on the host.  Keys and vals must come back unchanged."""
    from darray_b200 import _lib
    N = keys.ndim
    lo = [0] * N if lo is None else list(lo)
    gdims = list(keys.shape) if gdims is None else list(gdims)
    flat = keys.reshape(-1, order="F")
    dk = dab.B200Array.from_numpy(rt, flat)
    P = dab.B200Array.empty(rt, (flat.size,), np.int64)
    dv = vo = None
    if vals is not None:
        vflat = vals.reshape(-1, order="F")
        dv = dab.B200Array.from_numpy(rt, vflat)
        vo = dab.B200Array.empty(rt, (flat.size,), vals.dtype)
    SZ = C.c_size_t * N
    _lib.call("dab_sortperm_slices", rt.ctx, dab.dab_dtype(keys.dtype), C.c_void_p(dk.ptr), N, SZ(*keys.shape), SZ(*lo), SZ(*gdims), dim,
              C.c_void_p(P.ptr), vals.dtype.itemsize if vals is not None else 0, C.c_void_p(dv.ptr if dv else None),
              C.c_void_p(vo.ptr if vo else None))
    perm = P.to_numpy().reshape(keys.shape, order="F")
    assert np.array_equal(dk.to_numpy().view(np.uint8), flat.view(np.uint8))         # keys are never written
    out = None
    if vals is not None:
        assert np.array_equal(dv.to_numpy().view(np.uint8), vflat.view(np.uint8))    # nor are vals
        out = vo.to_numpy().reshape(keys.shape, order="F")
        dv.free()
        vo.free()
    dk.free()
    P.free()
    return perm, out


@pytest.mark.parametrize("T", DTYPES)
def test_k26_lengths_and_group_shapes(dab, rt1, T):
    """Every fibre length across both paths, inner == 1 (contiguous fibres) and inner > 1 (rows), outer > 1, every kind of input."""
    rng = np.random.default_rng(11)
    for ln in LENS:
        for shape, dim in (((ln, 3), 1), ((5, ln, 2), 2), ((ln,), 1)):
            kinds = KINDS if ln in (33, L, L + 1) else ("specials",)
            for kind in kinds:
                n = int(np.prod(shape))
                a = _data(T, n, rng, kind).reshape(shape, order="F")
                got, _ = _k26(dab, rt1, a, dim)
                assert np.array_equal(got, model_perm(a, dim)), (ln, shape, kind)


@pytest.mark.parametrize("T", DTYPES)
def test_k26_dims_and_chunk_offsets(dab, rt1, T):
    """``dim`` first, middle and last of 2-D to 8-D chunks, placed at nonzero offsets of a larger array in every other dim."""
    rng = np.random.default_rng(12)
    for N in range(2, 9):
        for dim in sorted({1, (N + 1) // 2, N}):
            for long_fibre in (False, True):
                shape = [int(x) for x in rng.integers(1, 4, N)]
                shape[dim - 1] = L + 7 if long_fibre else int(rng.integers(2, 40))
                if long_fibre:                                   # keep the chunk small
                    shape = [1 if k != dim - 1 and k % 2 else s for k, s in enumerate(shape)]
                lo = [0 if k == dim - 1 else int(rng.integers(1, 5)) for k in range(N)]
                gdims = [s if k == dim - 1 else s + lo[k] + int(rng.integers(0, 3)) for k, s in enumerate(shape)]
                a = _data(T, int(np.prod(shape)), rng, "specials").reshape(shape, order="F")
                got, _ = _k26(dab, rt1, a, dim, lo, gdims)
                assert np.array_equal(got, model_perm(a, dim, lo, gdims)), (N, dim, shape)


@pytest.mark.parametrize("VT", [np.float32, np.float64, np.int32, np.int64])
def test_k26_moves_values_bit_for_bit(dab, rt1, VT):
    """``vals_out`` of 4 and 8 bytes on both paths: the values in the order of the keys, NaN payloads kept."""
    rng = np.random.default_rng(13)
    for KT in DTYPES:
        for shape, dim in (((40, 6), 1), ((3, 40, 2), 2), ((2, 3 * L + 1), 2), ((L + 1, 2), 1)):
            n = int(np.prod(shape))
            k = _data(KT, n, rng, "repeated").reshape(shape, order="F")
            v = _data(VT, n, rng, "specials").reshape(shape, order="F")
            perm, got = _k26(dab, rt1, k, dim, vals=v)
            want = model_perm(k, dim)
            assert np.array_equal(perm, want)
            assert np.array_equal(_bits(got), _bits(v.reshape(-1, order="F")[want - 1]))


def test_k26_errors(dab, rt1):
    from darray_b200 import _lib
    a = np.zeros((4, 3), dtype=np.float32)
    with pytest.raises(dab.ArgumentError):
        _k26(dab, rt1, a, 1, gdims=[5, 3])                      # dim not whole
    with pytest.raises(dab.ArgumentError):
        _k26(dab, rt1, a, 3)
    with pytest.raises(dab.ArgumentError):
        _k26(dab, rt1, a, 2, lo=[2, 0], gdims=[5, 3])           # outside the array
    with pytest.raises(dab.UnsupportedError):
        _k26(dab, rt1, a.astype(np.float16), 1)
    with pytest.raises(dab.ArgumentError):                      # vals without vals_out
        _lib.call("dab_sortperm_slices", rt1.ctx, _lib.F32, C.c_void_p(16), 1, (C.c_size_t * 1)(4), (C.c_size_t * 1)(0),
                  (C.c_size_t * 1)(4), 1, C.c_void_p(16), 4, C.c_void_p(16), C.c_void_p(None))
    l0 = rt1.launches()
    _lib.call("dab_sortperm_slices", rt1.ctx, _lib.F32, C.c_void_p(None), 2, (C.c_size_t * 2)(0, 3), (C.c_size_t * 2)(0, 0),
              (C.c_size_t * 2)(0, 3), 1, C.c_void_p(None), 0, C.c_void_p(None), C.c_void_p(None))
    assert rt1.launches() == l0                                  # an empty chunk launches nothing


@pytest.mark.parametrize("inner", [1, 4])
def test_long_fibre_launches_do_not_grow_with_the_fibre_count(dab, rt1, inner):
    rng = np.random.default_rng(14)
    counts = []
    for nfib in (2, 64):
        shape, dim = ((L + 100, nfib), 1) if inner == 1 else ((inner, L + 100, nfib // inner if nfib > inner else 1), 2)
        if inner > 1 and nfib == 2:
            shape = (2, L + 100)
        a = _data(np.float64, int(np.prod(shape)), rng).reshape(shape, order="F")
        l0 = rt1.launches()
        got, _ = _k26(dab, rt1, a, dim)
        counts.append(rt1.launches() - l0)
        assert np.array_equal(got, model_perm(a, dim))
    assert counts[0] == counts[1], counts


# ---- public API ----------------------------------------------------------------------------------------------------------------------


def _bits(x):
    x = np.asarray(x)
    return x.view(np.dtype(f"u{x.itemsize}")) if x.dtype.kind in "fi" else x


def _nan_equal(x, y):
    x, y = np.asarray(x), np.asarray(y)
    if x.dtype.kind == "f":
        return x.shape == y.shape and bool(np.all((x == y) | (np.isnan(x) & np.isnan(y))))
    return np.array_equal(x, y)


def _same_layout(p, q):
    return list(p.layout.pids) == list(q.layout.pids) and list(p.layout.indices) == list(q.layout.indices) and p.layout.grid == q.layout.grid


CASES = [((64, 37), None), ((64, 37), [1, 8]), ((64, 37), [8, 1]), ((33, 8, 6), [2, 2, 2]), ((L + 3, 6), [3, 1]), ((5, L + 3), [1, 3]),
         ((7, 5, 9), None)]


@pytest.mark.parametrize("T", DTYPES)
@pytest.mark.parametrize("nw", [1, 8])
def test_public_sortperm_and_sort(dab, request, T, nw):
    """sortperm(A; dims) against the model, sort(A; dims) against mapslices(sort), A[sortperm] against sort, with and without ``by``."""
    request.getfixturevalue(f"rt{nw}")
    rng = np.random.default_rng(20 + nw)
    if True:
        for shape, dist in CASES:
            if dist is not None and int(np.prod(dist)) > nw:
                continue
            a = _data(T, int(np.prod(shape)), rng, "repeated").reshape(shape, order="F")
            A = dab.distribute(a) if dist is None else dab.distribute(a, procs=list(range(1, int(np.prod(dist)) + 1)), dist=dist)
            for dim in range(1, a.ndim + 1):
                P = dab.sortperm(A, dims=dim)
                assert P.dtype == np.int64 and P.dims == A.dims
                assert np.array_equal(dab.to_array(P), model_perm(a, dim)), (shape, dist, dim)
                S = dab.sort(A, dims=dim)
                M = dab.mapslices(dab.sort, A, dims=dim)
                assert _same_layout(S, M) and _same_layout(P, S)
                assert np.array_equal(_bits(dab.to_array(S)), _bits(dab.to_array(M)))
                AP = A[P]
                assert _nan_equal(dab.to_array(AP), dab.to_array(S))
                for by, f in ((abs, np.abs), (lambda x: -x, lambda x: -x), (lambda x: x > 0, lambda x: (x > 0).astype(np.int32))):
                    with np.errstate(over="ignore"):
                        k = f(a)
                    Pb = dab.sortperm(A, dims=dim, by=by)
                    assert np.array_equal(dab.to_array(Pb), model_perm(k, dim)) and _same_layout(Pb, S)
                    Sb = dab.sort(A, dims=dim, by=by)
                    want = a.reshape(-1, order="F")[model_perm(k, dim) - 1]
                    assert np.array_equal(_bits(dab.to_array(Sb)), _bits(want)) and _same_layout(Sb, S)
                    for x in (Pb, Sb):
                        x.close()
                for x in (P, S, M, AP):
                    x.close()
            A.close()
    dab.d_closeall()


@pytest.mark.parametrize("T", DTYPES)
def test_dvector_dims_1_is_the_samplesort(dab, rt8, T):
    rng = np.random.default_rng(30)
    a = _data(T, 5000, rng, "repeated")
    v = dab.distribute(a)
    for by in (None, abs):
        s0, s1 = dab.sort(v, by=by), dab.sort(v, dims=1, by=by)
        p0, p1 = dab.sortperm(v, by=by), dab.sortperm(v, dims=1, by=by)
        assert np.array_equal(_bits(dab.to_array(s0)), _bits(dab.to_array(s1))) and _same_layout(s0, s1)
        assert np.array_equal(dab.to_array(p0), dab.to_array(p1)) and _same_layout(p0, p1)
        assert len(p1.layout.pids) > 1                           # not funnelled onto one worker
    dab.d_closeall()


def test_refusals_launch_and_register_nothing(dab, rt8):
    """Every refusal of the dims forms is raised before anything is allocated or launched; the Float16 and complex errors name the type."""
    rng = np.random.default_rng(40)
    A = dab.distribute(rng.standard_normal((16, 8)))
    B = dab.distribute(rng.standard_normal((16, 8)) > 0)
    Z = dab.distribute(rng.standard_normal((16, 8)).astype(np.complex64))
    H = dab.distribute(rng.standard_normal((16, 8)).astype(np.float16))
    V = A[2:10, 1:5]
    assert isinstance(V, dab.SubDArray)
    cases = [(dab.ArgumentError, None, lambda: dab.sortperm(A, dims=0)), (dab.ArgumentError, None, lambda: dab.sortperm(A, dims=3)),
             (dab.ArgumentError, None, lambda: dab.sort(A, dims=True)), (dab.ArgumentError, None, lambda: dab.sortperm(A, dims=1.0)),
             (dab.ArgumentError, None, lambda: dab.sortperm(A, dims=(1,))), (dab.ArgumentError, None, lambda: dab.sort(A, dims=1, rev=True)),
             (dab.ArgumentError, None, lambda: dab.sortperm(A, dims=1, sample=True)),
             (dab.ArgumentError, None, lambda: dab.sort(A, dims=1, lt=abs)), (dab.ArgumentError, None, lambda: dab.sortperm(A, dims=2, order=1)),
             (TypeError, "complex", lambda: dab.sortperm(Z, dims=1)), (TypeError, "complex", lambda: dab.sort(Z, dims=2)),
             (dab.UnsupportedError, "complex", lambda: dab.sortperm(Z, dims=1, by=abs)),
             (dab.UnsupportedError, "complex", lambda: dab.sort(Z, dims=1, by=abs)),
             (dab.UnsupportedError, "Float16", lambda: dab.sortperm(H, dims=1)), (dab.UnsupportedError, "Float16", lambda: dab.sort(H, dims=2, by=abs)),
             (dab.UnsupportedError, None, lambda: dab.sortperm(B, dims=1)), (dab.UnsupportedError, None, lambda: dab.sort(B, dims=1, by=abs)),
             (dab.UnsupportedError, "DArray first", lambda: dab.sortperm(V, dims=1))]
    l0, r0 = rt8.launches(), dab.registry_size()
    for exc, text, f in cases:
        with pytest.raises(exc) as ei:
            f()
        assert (rt8.launches(), dab.registry_size()) == (l0, r0), (exc, text)
        if text is not None:
            assert text in str(ei.value), str(ei.value)
    dab.d_closeall()
