"""GPU tests of ``sortperm`` for DVectors: K21 (``dab_sort_pairs``, the pair path of the onesweep sort) against the stable ``isless``
permutation of oracle/darray_oracle.py, and the distributed flow against the model and against ``sort``'s layout.  Everything here is
integer / bit-pattern work: results must equal the model exactly."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets the pair sort too
    import sortperm_hostmem
    sortperm_hostmem.install()

DTYPES = [np.float32, np.float64, np.int32, np.int64]
SIZES = (0, 1, 2, 31, 1024, 1025, 4096, 4097, 100003, (1 << 20) + 17)


def _data(T, n, rng, kind="full"):
    T = np.dtype(T)
    if kind == "full":
        if T.kind == "i":
            return rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T)
        return (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(T)
    if kind == "small":                                         # most digit passes are constant and skipped
        return rng.integers(-1000, 1000, n).astype(T) if T.kind == "i" else (rng.integers(0, 3000, n) * 0.25).astype(T)
    if kind == "equal":
        return np.full(n, 7, dtype=T)
    if kind == "sorted":
        return np.sort(_data(T, n, rng))
    if kind == "reversed":
        return np.sort(_data(T, n, rng))[::-1].copy()
    if kind == "repeated":                                      # 50 values repeated
        return rng.choice(_data(T, 50, rng), n)
    raise ValueError(kind)


def _float_specials(T, n, rng):
    """±0, ±Inf and NaNs of both signs and several payloads, scattered through random data."""
    U = np.uint32 if np.dtype(T) == np.float32 else np.uint64
    a = _data(T, n, rng)
    nans = [np.nan, -np.nan]
    if U is np.uint32:
        nans += [np.array([0x7FC00001, 0xFFC00123, 0x7F800001, 0xFFBFFFFF], dtype=U).view(T)[i] for i in range(4)]
    else:
        nans += [np.array([0x7FF8000000000001, 0xFFF8000000000123, 0x7FF0000000000001], dtype=U).view(T)[i] for i in range(3)]
    for v, k in [(0.0, n // 20), (-0.0, n // 20), (np.inf, n // 50), (-np.inf, n // 50)] + [(x, n // 40) for x in nans]:
        a[rng.integers(0, n, k)] = v
    return a


def _pairs(dab, rt, keys, vals=None, base=1, inplace=False):
    """dab_sort_pairs on one device buffer: (keys_out, vals_out) on the host."""
    from darray_b200 import _lib
    n = keys.size
    dk = dab.B200Array.from_numpy(rt, keys) if n else dab.B200Array.empty(rt, (0,), keys.dtype)
    ko = dk if inplace else dab.B200Array.empty(rt, (n,), keys.dtype)
    dv = dab.B200Array.from_numpy(rt, vals) if vals is not None and n else None
    vo = dab.B200Array.empty(rt, (n,), np.int64)
    need = C.c_size_t()
    _lib.check(_lib.lib().dab_sort_pairs_scratch_bytes(dab.dab_dtype(keys.dtype), n, C.byref(need)))
    scratch = dab.B200Array.empty(rt, (max(need.value, 16),), np.uint8)
    _lib.call("dab_sort_pairs", rt.ctx, dab.dab_dtype(keys.dtype), C.c_void_p(dk.ptr), C.c_void_p(ko.ptr), C.c_void_p(dv.ptr if dv else None),
              base, C.c_void_p(vo.ptr), C.c_void_p(scratch.ptr), need.value, n)
    got_k, got_v = ko.to_numpy(), vo.to_numpy()
    if not inplace:
        assert np.array_equal(dk.to_numpy().view(np.uint8), keys.view(np.uint8))   # the input is never written
        ko.free()
    if dv is not None:
        assert np.array_equal(dv.to_numpy(), vals)
        dv.free()
    for b in (dk, vo, scratch):
        b.free()
    return got_k, got_v


def _check_pairs(keys, vals, base, got_k, got_v):
    p = orc.jl_sortperm_stable(keys)
    want_v = vals[p] if vals is not None else np.int64(base) + p.astype(np.int64)
    assert got_v.dtype == np.int64 and np.array_equal(got_v, want_v)
    want_k = orc.jl_sort(keys)
    if keys.dtype.kind == "f":
        k = int((~np.isnan(keys)).sum())
        U = np.uint32 if keys.dtype == np.float32 else np.uint64
        assert np.array_equal(got_k[:k].view(U), want_k[:k].view(U)) and np.all(np.isnan(got_k[k:]))   # incl. the sign of the zeros
    else:
        assert np.array_equal(got_k, want_k)


@pytest.mark.parametrize("T", DTYPES)
def test_sort_pairs_kernel_sizes_and_patterns(dab, rt1, T):
    """K21 for every size class (rank sort, one ragged tile, many tiles) and pattern, with generated indices at base 1 and at
    2^33 + 5 (64-bit index arithmetic) and with random distinct Int64 values."""
    rng = np.random.default_rng(71)
    for n in SIZES:
        for kind in ("full", "small", "equal", "sorted", "reversed", "repeated"):
            a = _data(T, n, rng, kind)
            for base in (1, (1 << 33) + 5):
                _check_pairs(a, None, base, *_pairs(dab, rt1, a, base=base))
            vals = rng.choice(np.int64(1) << 50, n, replace=False).astype(np.int64) - (1 << 49)
            _check_pairs(a, vals, 0, *_pairs(dab, rt1, a, vals=vals))


@pytest.mark.parametrize("T", DTYPES)
def test_sort_pairs_kernel_in_place(dab, rt1, T):
    """keys_out == keys: the sort runs in place (odd and even pass counts, the rank sort and the no-pass case)."""
    rng = np.random.default_rng(72)
    for n in (5, 1024, 1025, 100003):
        for kind in ("full", "small", "equal"):
            a = _data(T, n, rng, kind)
            _check_pairs(a, None, 1, *_pairs(dab, rt1, a, base=1, inplace=True))


@pytest.mark.parametrize("T", [np.float32, np.float64])
def test_sort_pairs_kernel_float_specials(dab, rt1, T):
    """-0.0 before +0.0, ±Inf in place, NaNs of both signs and several payloads all equal: last, in index order."""
    rng = np.random.default_rng(73)
    for n in (1000, 4097, 300001):
        a = _float_specials(T, n, rng)
        _check_pairs(a, None, 1, *_pairs(dab, rt1, a, base=1))
        vals = rng.permutation(n).astype(np.int64) * 3 - 7
        _check_pairs(a, vals, 0, *_pairs(dab, rt1, a, vals=vals))
    a = np.full(5000, np.nan, dtype=T)                          # every key a NaN: one tie, the identity
    a[::3] = -np.nan
    _check_pairs(a, None, 1, *_pairs(dab, rt1, a, base=1))


def _check_sortperm(dab, d, a, sample=True, by=None, keys=None):
    """The three properties of sortperm(d): the model's values, sort's layout, and a[p] sorted."""
    p = dab.sortperm(d, sample=sample, by=by)
    k = a if keys is None else keys
    got = dab.to_array(p)
    assert p.dtype == np.int64 and np.array_equal(got, orc.jl_sortperm_stable(k) + 1)
    ref_d = d if keys is None else dab.distribute(keys, procs=list(d.layout.pids), dist=list(d.layout.grid))
    s, _ = dab.sort_with_boundaries(ref_d, sample=sample)
    nan = np.isnan(dab.to_array(s)) if k.dtype.kind == "f" else np.zeros(len(s), dtype=bool)
    if not nan.any() or nan[np.argmax(nan):].all():         # sort's result is in isless order (NaNs last): the same layout
        assert list(p.layout.pids) == list(s.layout.pids) and list(p.layout.indices) == list(s.layout.indices)
        assert list(p.layout.cuts) == list(s.layout.cuts)
    s.close()
    if ref_d is not d:
        ref_d.close()
    ordered = k[got - 1]
    if k.dtype.kind == "f":
        ordered = ordered[~np.isnan(ordered)]
        want = np.sort(k[~np.isnan(k)])
    else:
        want = np.sort(k)
    assert np.array_equal(ordered, want)
    p.close()


@pytest.mark.parametrize("T", [np.int64, np.float64])
@pytest.mark.parametrize("i", range(0, 7))
def test_sortperm_reference_sweep(dab, rt8, T, i):
    """The reference sort test's sizes (test/darray.jl:1015-1025) with every kind of sample."""
    rng = np.random.default_rng(300 + i)
    n = 10 ** i
    a = _data(T, n, rng)
    d = dab.distribute(a)
    for sample in (True, False, (a.min(), a.max()), _data(T, min(n, 512), rng)):
        _check_sortperm(dab, d, a, sample)


def test_sortperm_other_types_layouts_and_runtimes(dab, rt8):
    rng = np.random.default_rng(81)
    for T in (np.float32, np.int32):
        for kind in ("full", "small"):
            a = _data(T, 77777, rng, kind)
            _check_sortperm(dab, dab.distribute(a), a)
            _check_sortperm(dab, dab.distribute(a, procs=[1, 2, 3], dist=[3]), a)


@pytest.mark.parametrize("T", DTYPES)
def test_sortperm_on_one_worker(dab, rt1, T):
    rng = np.random.default_rng(82)
    for n in (1, 1000, 300001):
        a = _data(T, n, rng, "repeated")
        _check_sortperm(dab, dab.distribute(a), a)


def test_sortperm_on_two_workers(dab, rt2):
    rng = np.random.default_rng(83)
    for T in DTYPES:
        a = _data(T, 200001, rng, "small")
        for sample in (True, False):
            _check_sortperm(dab, dab.distribute(a), a, sample)


def test_sortperm_ties_nans_and_skew(dab, rt8):
    """Ties spanning chunk boundaries (stability across workers), NaNs in several chunks, receivers that drop out."""
    rng = np.random.default_rng(84)
    for a in (np.zeros(100000), rng.integers(0, 3, 100000).astype(np.int64), rng.integers(0, 3, 100000).astype(np.float32)):
        for sample in (True, False):
            _check_sortperm(dab, dab.distribute(a), a, sample)
    for T in (np.float32, np.float64):
        a = _float_specials(T, 200000, rng)
        _check_sortperm(dab, dab.distribute(a), a)
    a = np.concatenate([np.zeros(5000, dtype=np.int64), np.arange(8, dtype=np.int64)])
    d = dab.distribute(a)
    p = dab.sortperm(d)
    assert len(p.layout.pids) < 8
    _check_sortperm(dab, d, a)


def test_sortperm_by(dab, rt8):
    """sortperm(d; by = f) is sortperm(f.(d)): abs, a Bool-valued key (false < true), an Int64 -> Float64 key."""
    rng = np.random.default_rng(85)
    a = _data(np.float64, 100003, rng, "small") - 300.0
    for sample in (True, False):
        _check_sortperm(dab, dab.distribute(a), a, sample, by=abs, keys=np.abs(a))
    _check_sortperm(dab, dab.distribute(a), a, True, by=lambda x: x > 0, keys=(a > 0).astype(np.int32))
    b = _data(np.int64, 100003, rng, "small")
    _check_sortperm(dab, dab.distribute(b), b, True, by=lambda x: x * 0.5, keys=b.astype(np.float64) * 0.5)


def test_sortperm_refusals_launch_nothing(dab, rt8):
    """The errors sort raises for the same arguments, all before any launch, with nothing left registered."""
    import scipy.sparse as sp
    rng = np.random.default_rng(86)
    v = dab.distribute(rng.standard_normal(1000))
    M = dab.distribute(rng.standard_normal((40, 30)))
    Z = dab.distribute(rng.standard_normal(1000).astype(np.complex128))
    B = dab.distribute(rng.standard_normal(1000) > 0)
    S = dab.distribute(sp.random(30, 20, density=0.2, format="csc", random_state=1))
    holes = dab.distribute(rng.standard_normal(7), procs=list(range(1, 9)), dist=[8])   # an empty localpart
    cases = [
        (dab.DimensionMismatch, lambda: dab.sortperm(M)),
        (TypeError, lambda: dab.sortperm(Z)),
        (dab.UnsupportedError, lambda: dab.sortperm(B)),
        (dab.UnsupportedError, lambda: dab.sortperm(S)),
        (dab.ArgumentError, lambda: dab.sortperm(v, rev=True)),
        (dab.ArgumentError, lambda: dab.sortperm(v, lt=lambda x, y: x < y)),
        (dab.ArgumentError, lambda: dab.sortperm(v, order="forward")),
        (dab.ArgumentError, lambda: dab.sortperm(v, sample="yes")),
        (dab.ArgumentError, lambda: dab.sortperm(v, sample=(1.0, 2.0, 3.0))),
        (dab.ArgumentError, lambda: dab.sortperm(v, sample=(-np.inf, 1.0))),
        (dab.ArgumentError, lambda: dab.sortperm(v, sample=(-np.inf, 1.0), by=abs)),
        (TypeError, lambda: dab.sortperm(v, by=lambda x: x if x > 0 else -x)),
        (ZeroDivisionError, lambda: dab.sortperm(holes)),
    ]
    for exc, f in cases:
        n0, l0 = dab.registry_size(), rt8.launches()
        with pytest.raises(exc):
            f()
        assert dab.registry_size() == n0 and rt8.launches() == l0, exc
    with pytest.raises(ZeroDivisionError):
        dab.sort(holes)                                         # the same error as sort


def test_sortperm_of_an_empty_vector(dab, rt8):
    e = dab.distribute(np.zeros(0), procs=[1])
    n0, l0 = dab.registry_size(), rt8.launches()
    for sample in (False, (0.0, 1.0)):
        with pytest.raises(dab.ArgumentError):
            dab.sortperm(e, sample=sample)
    assert dab.registry_size() == n0 and rt8.launches() == l0


def test_sortperm_large(dab, rt8):
    """2^28 Float32 keys with ~16 copies of every value: the result is the stable permutation, checked exactly by its definition
    (a permutation of 1:n, keys nondecreasing along it, indices ascending inside every run of equal keys)."""
    if HOSTMEM:
        pytest.skip("a GPU-sized case: 2^28 keys")
    n = 1 << 28
    a = np.random.default_rng(87).random(n, dtype=np.float32)
    p = dab.sortperm(dab.distribute(a))
    got = dab.to_array(p)
    p.close()
    assert got.dtype == np.int64 and got.size == n and got.min() == 1 and got.max() == n
    seen = np.zeros(n, dtype=bool)
    seen[got - 1] = True
    assert seen.all()
    del seen
    s = a[got - 1]
    up = s[1:] > s[:-1]
    tie = s[1:] == s[:-1]
    assert np.all(up | tie) and np.all(got[1:][tie] > got[:-1][tie])
