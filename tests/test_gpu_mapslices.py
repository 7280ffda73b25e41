"""GPU tests of ``mapslices`` (reference src/mapreduce.jl:191-208; reference testset test/darray.jl:804-841) and of its two kernels:
``dab_sort_slices`` (bit-identical to K11 per fibre) and ``dab_svdvals_batched`` (against numpy.linalg.svd in fp64)."""
import ctypes as C

import numpy as np
import pytest

import mapslices_oracle as mo

pytestmark = pytest.mark.gpu

SMEM_LEN = 8192                                                      # DAB_SORT_SLICES_SMEM_LEN
LENS = (1, 2, 5, 31, 32, 33, 1000, 4096, 4097, SMEM_LEN, SMEM_LEN + 1, (1 << 17) + 3)
INNERS = (1, 3, 8, 1000)


def _data(T, n, rng):
    """Floats with +-0.0, +-Inf and NaNs of both signs and several payloads; integers with the type's extremes."""
    T = np.dtype(T)
    if T.kind == "i":
        a = rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T, endpoint=True)
        k = max(1, n // 50)
        a[rng.integers(0, n, k)] = np.iinfo(T).min
        a[rng.integers(0, n, k)] = np.iinfo(T).max
        a[rng.integers(0, n, k)] = 0
        return a
    a = (rng.standard_normal(n) * 10.0 ** rng.integers(-5, 5, n)).astype(T)
    u = np.uint32 if T.itemsize == 4 else np.uint64
    specials = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800123, 0xFFFFFFFF] if T.itemsize == 4 else
                        [0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000123,
                         0xFFFFFFFFFFFFFFFF], dtype=u)
    v = a.view(u)
    idx = rng.integers(0, n, max(1, n // 8))
    v[idx] = specials[rng.integers(0, len(specials), idx.size)]
    return a


def _dev(dab, rt, a, offset):
    """A device copy of ``a`` starting ``offset`` elements into its allocation (offset 1: a misaligned base)."""
    buf = dab.B200Array.empty(rt, (a.size + offset,), a.dtype)
    view = dab.B200Array(rt, buf.ptr + offset * a.itemsize, (a.size,), a.dtype, own=False)
    view.copy_from_host(a)
    return buf, view


def _k11_fibre(dab, rt, f):
    from darray_b200 import _lib
    src = dab.B200Array.from_numpy(rt, np.ascontiguousarray(f))
    out = dab.B200Array.empty(rt, (f.size,), f.dtype)
    tmp = dab.B200Array.empty(rt, (max(f.size, 1),), f.dtype)
    _lib.call("dab_sort", rt.ctx, dab.dab_dtype(f.dtype), C.c_void_p(src.ptr), C.c_void_p(out.ptr), C.c_void_p(tmp.ptr), f.size)
    got = out.to_numpy()
    for b in (src, out, tmp):
        b.free()
    return got


@pytest.mark.parametrize("T", [np.float32, np.float64, np.int32, np.int64])
def test_sort_slices_equals_k11_per_fibre(dab, rt1, T):
    """Every output fibre is byte-identical to dab_sort of that fibre: in place and out of place, aligned and one element off, input
    untouched out of place.  The expected fibres come from K11 itself (a handful per case) and from the same radix-key order on the host
    (all of them; that order IS K11's, tests/test_gpu_sort.py)."""
    from darray_b200 import _lib
    import hostmem_abi as H
    rng = np.random.default_rng(7)
    code = dab.dab_dtype(np.dtype(T))
    for ln in LENS:
        for inner in INNERS:
            if ln * inner > (1 << 24):
                continue                                            # 131 M elements per case: covered by the smaller inners
            for outer in ((1, 3) if ln * inner < (1 << 18) else (2,)):
                n = inner * ln * outer
                a = _data(T, n, rng)
                u = a.view(np.uint32 if a.itemsize == 4 else np.uint64).reshape((inner, ln, outer), order="F")
                want = H.radix_dec(np.sort(H.radix_enc(u, code), axis=1), code).reshape(-1, order="F")
                for offset in (0, 1):
                    for inplace in (False, True):
                        buf, x = _dev(dab, rt1, a, offset)
                        obuf, y = (buf, x) if inplace else _dev(dab, rt1, np.zeros_like(a), offset)
                        _lib.call("dab_sort_slices", rt1.ctx, code, C.c_void_p(x.ptr), C.c_void_p(y.ptr), inner, ln, outer)
                        got = y.to_numpy()
                        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (T, ln, inner, outer, offset, inplace)
                        if not inplace:
                            assert np.array_equal(x.to_numpy().view(np.uint8), a.view(np.uint8))
                            obuf.free()
                        buf.free()
                g = want.view(a.dtype).reshape((inner, ln, outer), order="F")
                A3 = a.reshape((inner, ln, outer), order="F")
                for i, o in {(0, 0), (inner - 1, outer - 1), (inner // 2, outer // 2)}:
                    assert np.array_equal(_k11_fibre(dab, rt1, A3[i, :, o]).view(np.uint8), np.ascontiguousarray(g[i, :, o]).view(np.uint8))


def _svd_batch(dab, rt, A, T):
    from darray_b200 import _lib
    m, n, batch = A.shape
    k = min(m, n)
    src = dab.B200Array.from_numpy(rt, np.asfortranarray(A.astype(T)).reshape(-1, order="F"))
    S = dab.B200Array.empty(rt, (k * batch,), T)
    st = dab.B200Array.empty(rt, (1,), np.int32)
    try:
        _lib.call("dab_svdvals_batched", rt.ctx, dab.dab_dtype(np.dtype(T)), C.c_void_p(src.ptr), m, n, batch, C.c_void_p(S.ptr), C.c_void_p(st.ptr))
        return S.to_numpy().reshape((batch, k)), int(st.to_numpy()[0])
    finally:
        for b in (src, S, st):
            b.free()


@pytest.mark.parametrize("shape", [(1, 1), (5, 5), (10, 10), (32, 32), (3, 17), (17, 3), (32, 128), (128, 32)])
@pytest.mark.parametrize("T", [np.float64, np.float32])
def test_svdvals_batched_vs_numpy(dab, rt1, shape, T):
    m, n = shape
    k = min(m, n)
    rng = np.random.default_rng(m * 131 + n)
    mats = []
    for _ in range(3):
        mats.append(rng.standard_normal((m, n)))
    r = max(1, k // 2)
    mats.append(rng.standard_normal((m, r)) @ rng.standard_normal((r, n)))          # rank-deficient
    mats.append(np.zeros((m, n)))
    mats.append(np.eye(m, n))
    U, _ = np.linalg.qr(rng.standard_normal((m, m)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    mats.append((U[:, :k] * np.logspace(0, -12, k)) @ V[:, :k].T)                   # condition number 1e12
    A = np.stack(mats, axis=2).astype(T)
    got, status = _svd_batch(dab, rt1, A, T)
    assert status == 0 and got.dtype == np.dtype(T)
    tol = 1e-12 if T == np.float64 else 2e-6
    for b in range(A.shape[2]):
        want = np.linalg.svd(A[:, :, b].astype(np.float64), compute_uv=False)
        assert np.all(np.diff(got[b]) <= 0), (shape, b)
        assert np.max(np.abs(got[b].astype(np.float64) - want)) <= tol * max(want.max(), np.finfo(np.float64).tiny), (shape, T, b)


@pytest.mark.parametrize("shape", [(5, 5), (32, 32), (3, 17), (128, 32)])
def test_svdvals_batched_extreme_magnitudes(dab, rt1, shape):
    """Finite Float64 input far from 1: the kernel scales by a power of two, so nothing overflows or underflows (numpy's LAPACK scales too)."""
    m, n = shape
    base = np.random.default_rng(m + 7 * n).standard_normal((m, n))
    scales = [1e160, 1e-170, 1e-160, 1e300, 1e-300, 1e-310]
    A = np.stack([base * s for s in scales], axis=2)
    got, status = _svd_batch(dab, rt1, A, np.float64)
    assert status == 0
    for b, s in enumerate(scales):
        want = np.linalg.svd(A[:, :, b], compute_uv=False)
        assert np.all(np.isfinite(got[b])) and np.max(np.abs(got[b] - want)) <= 1e-12 * want.max(), (shape, s)
    F = np.stack([base * 1e30, base * 1e-30], axis=2).astype(np.float32)
    got, status = _svd_batch(dab, rt1, F, np.float32)
    for b in range(2):
        want = np.linalg.svd(F[:, :, b].astype(np.float64), compute_uv=False)
        assert status == 0 and np.max(np.abs(got[b].astype(np.float64) - want)) <= 2e-6 * want.max(), (shape, b)


def test_svdvals_batched_nonfinite_and_limits(dab, rt1):
    A = np.random.default_rng(3).standard_normal((6, 4, 5))
    A[1, 2, 3] = np.nan
    got, status = _svd_batch(dab, rt1, A, np.float64)
    assert status == 1 and np.all(np.isnan(got[3])) and np.all(np.isfinite(np.delete(got, 3, axis=0)))
    A[1, 2, 3] = -np.inf
    assert _svd_batch(dab, rt1, A, np.float32)[1] == 1
    A[1, 2, 3] = 0.0
    assert _svd_batch(dab, rt1, A, np.float64)[1] == 0                     # the flag is cleared by every call
    for shape in ((33, 33, 1), (40, 120, 1), (20, 300, 1)):
        with pytest.raises(dab.UnsupportedError, match="min\\(m,n\\) <= 32 and m\\*n <= 4096"):
            _svd_batch(dab, rt1, np.ones(shape), np.float64)
    D = dab.distribute(np.where(np.arange(48.0).reshape((4, 4, 3), order="F") == 17, np.nan, 1.0))
    with pytest.raises(dab.ArgumentError, match="Infs or NaNs"):
        dab.mapslices(dab.svdvals, D, dims=(1, 2))
    with pytest.raises(dab.UnsupportedError):
        dab.mapslices(dab.svdvals, dab.distribute(np.ones((40, 40, 2))), dims=(1, 2))


def test_reference_testset(dab, rt8):
    """test/darray.jl:804-841 on 8 workers: svdvals over (1,2) (1,3) (2,3), sort over 1 2 3 against the oracle's mapslices of the host array
    (layouts included), #3613, #5141, #5177."""
    mo.check_reference_testset(dab)


def test_layouts_local_and_redistributed(dab, rt8):
    """Result dims / pids / cuts equal the oracle's, for slice dimensions already local and for split ones (redistribution by halo reads)."""
    mo.check_layouts(dab)


def test_errors_raise_before_any_launch(dab, rt8):
    mo.check_errors_before_launch(dab, rt8)


def test_mapslices_sort_long_fibres_and_int_svdvals(dab, rt2):
    """Fibres past shared memory (K11 path) through the public API, both orientations, and Int64 svdvals computed in Float64."""
    rng = np.random.default_rng(11)
    A = rng.standard_normal((SMEM_LEN + 5, 3))
    D = dab.distribute(A)
    assert np.array_equal(dab.to_array(dab.mapslices(dab.sort, D, dims=1)), np.sort(A, axis=0))
    B = np.ascontiguousarray(A.T)
    assert np.array_equal(dab.to_array(dab.mapslices(dab.sort, dab.distribute(np.asfortranarray(B)), dims=2)), np.sort(B, axis=1))
    I = rng.integers(-50, 50, (6, 7, 4)).astype(np.int64)
    R = dab.mapslices(dab.svdvals, dab.distribute(I), dims=(1, 2))
    assert R.dtype == np.float64 and R.dims == (6, 1, 4)
    want = mo.jl_mapslices(mo.svdvals_np, I, (1, 2))
    assert np.max(np.abs(dab.to_array(R) - want)) <= 1e-12 * np.max(want)
