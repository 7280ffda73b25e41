"""GPU tests of ``ppeval`` (reference src/mapreduce.jl:210-323; reference testset test/darray.jl:973-986) and of its two kernels:
``dab_matmul_batched`` (exact for integers, within the fp64 rounding bound for floats) and ``dab_eigvals_sym_batched`` (against
numpy.linalg.eigvalsh)."""
import ctypes as C

import numpy as np
import pytest

import ppeval_oracle as po

pytestmark = pytest.mark.gpu

DIMS = (1, 7, 10, 33, 64, 65, 300)
# (m, k, n): every size of DIMS on every axis, k = 0, both sides of the staged / streamed / tiled switch
SHAPES = [(1, 1, 1), (7, 10, 1), (10, 10, 1), (10, 10, 10), (7, 0, 10), (64, 0, 1), (33, 7, 65), (64, 64, 64), (65, 33, 1),
          (64, 64, 1), (300, 300, 1), (1, 300, 300), (300, 1, 300), (65, 300, 7), (300, 65, 64), (10, 300, 1), (1, 7, 33)]


def _data(T, shape, rng):
    T = np.dtype(T)
    if T.kind == "i":
        return rng.integers(np.iinfo(T).min, np.iinfo(T).max, shape, dtype=T, endpoint=True)
    return (rng.standard_normal(shape) * 10.0 ** rng.integers(-3, 4, shape)).astype(T)


def _batched(dab, rt, A, B, T, bcast_a, bcast_b):
    """C[:, :, b] = A[:, :, b] @ B[:, :, b] on the GPU; a broadcast operand is passed as its one slice with stride 0."""
    from darray_b200 import _lib
    m, k, batch = A.shape
    n = B.shape[1]
    a = A[:, :, :1] if bcast_a else A
    b = B[:, :, :1] if bcast_b else B
    dA = dab.B200Array.from_numpy(rt, np.asfortranarray(a).reshape(-1, order="F")) if a.size else None
    dB = dab.B200Array.from_numpy(rt, np.asfortranarray(b).reshape(-1, order="F")) if b.size else None
    dC = dab.B200Array.empty(rt, (m * n * batch,), T)
    try:
        _lib.call("dab_matmul_batched", rt.ctx, dab.dab_dtype(np.dtype(T)), m, n, k, C.c_void_p(dA.ptr if dA else 0), 0 if bcast_a else m * k,
                  C.c_void_p(dB.ptr if dB else 0), 0 if bcast_b else k * n, C.c_void_p(dC.ptr), batch)
        return dC.to_numpy().reshape((m, n, batch), order="F")
    finally:
        for x in (dA, dB, dC):
            if x is not None:
                x.free()


def _check_product(got, A, B, T):
    T = np.dtype(T)
    k = A.shape[1]
    if T.kind == "i":                                             # exact, modulo 2^bits: unsigned 64-bit arithmetic is exactly that
        bits = T.itemsize * 8
        P = np.einsum("ikb,kjb->ijb", A.astype(np.int64).view(np.uint64), B.astype(np.int64).view(np.uint64))
        if bits == 32:
            P = P & np.uint64(0xFFFFFFFF)
            want = P.astype(np.uint32).view(np.int32)
        else:
            want = P.view(np.int64)
        assert np.array_equal(got, want)
        b0 = A.shape[2] // 2                                       # one slice in Python integers, as Julia's generic matmul wraps
        assert np.array_equal(got[:, :, b0], po.exact_matmul(A[:, :, b0], B[:, :, b0]))
        return
    ref = np.einsum("ikb,kjb->ijb", A.astype(np.longdouble), B.astype(np.longdouble))
    mag = np.einsum("ikb,kjb->ijb", np.abs(A).astype(np.float64), np.abs(B).astype(np.float64))
    bound = k * 2.0 ** -53 * mag
    if T == np.float32:
        r32 = ref.astype(np.float32)
        bound = bound + 0.5 * np.spacing(np.abs(r32)).astype(np.float64)
    err = np.abs(got.astype(np.longdouble) - ref).astype(np.float64)
    assert np.all(err <= bound * (1 + 1e-12)), float(np.max(err - bound))


@pytest.mark.parametrize("T", [np.float64, np.float32, np.int32, np.int64])
def test_matmul_batched_vs_numpy(dab, rt1, T):
    rng = np.random.default_rng(int(np.dtype(T).num))
    for m, k, n in SHAPES:
        for batch in (1, 3, 37):
            for bcast_a, bcast_b in ((False, False), (True, False), (False, True)):
                A, B = _data(T, (m, k, batch), rng), _data(T, (k, n, batch), rng)
                if bcast_a:
                    A = np.repeat(A[:, :, :1], batch, axis=2)
                if bcast_b:
                    B = np.repeat(B[:, :, :1], batch, axis=2)
                got = _batched(dab, rt1, A, B, T, bcast_a, bcast_b)
                assert got.dtype == np.dtype(T)
                if k == 0:
                    assert np.all(got == 0), (m, k, n)
                    continue
                _check_product(got, A, B, T)


@pytest.mark.parametrize("T", [np.float64, np.float32, np.int32, np.int64])
@pytest.mark.parametrize("mkn", [(10, 10, 1), (10, 10, 10), (7, 33, 1), (64, 64, 1), (33, 7, 65)])
def test_matmul_batched_large_batches(dab, rt1, T, mkn):
    """Batches up to 10^5 slices on both sides of the size switch."""
    m, k, n = mkn
    batch = 100_000 if m * k <= 1000 else 4_000
    rng = np.random.default_rng(m + 7 * k + 31 * n)
    A, B = _data(T, (m, k, batch), rng), _data(T, (k, n, batch), rng)
    _check_product(_batched(dab, rt1, A, B, T, False, False), A, B, T)


def _eig_batch(dab, rt, A, T):
    from darray_b200 import _lib
    n, _, batch = A.shape
    src = dab.B200Array.from_numpy(rt, np.asfortranarray(A.astype(T)).reshape(-1, order="F"))
    W = dab.B200Array.empty(rt, (n * batch,), T)
    st = dab.B200Array.empty(rt, (1,), np.int32)
    try:
        _lib.call("dab_eigvals_sym_batched", rt.ctx, dab.dab_dtype(np.dtype(T)), C.c_void_p(src.ptr), n, batch, C.c_void_p(W.ptr),
                  C.c_void_p(st.ptr))
        return W.to_numpy().reshape((batch, n)), int(st.to_numpy()[0]), src.to_numpy()
    finally:
        for b in (src, W, st):
            b.free()


@pytest.mark.parametrize("T", [np.float64, np.float32])
@pytest.mark.parametrize("n", [1, 2, 3, 8, 10, 16, 31, 32, 33, 47, 63, 64])
def test_eigvals_sym_batched_vs_eigvalsh(dab, rt1, T, n):
    rng = np.random.default_rng(n)
    mats = []
    for _ in range(4):
        X = rng.standard_normal((n, n))
        mats.append(X + X.T)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    mats.append((Q * np.resize([1.0, -2.0, 1.0], n)) @ Q.T)                          # repeated eigenvalues
    Y = rng.standard_normal((n, max(1, n // 2)))
    mats.append(Y @ Y.T)                                                             # rank-deficient
    mats += [np.zeros((n, n)), np.diag(rng.standard_normal(n))]
    if T == np.float64:
        mats += [mats[0] * 1e300, mats[0] * 1e-300, mats[0] * 1e-310]
    A = np.stack([(M + M.T) / 2 for M in mats], axis=2).astype(T)                    # exactly symmetric after the rounding to T
    got, status, _ = _eig_batch(dab, rt1, A, T)
    assert status == 0 and got.dtype == np.dtype(T)
    for b in range(A.shape[2]):
        want = np.linalg.eigvalsh(A[:, :, b].astype(np.float64))
        tol = 64 * n * 2.0 ** -52 * np.max(np.abs(want))
        if T == np.float32:
            tol += 2.0 ** -24 * np.max(np.abs(want))
        assert np.all(np.diff(got[b]) >= 0), (n, b)
        assert np.max(np.abs(got[b].astype(np.float64) - want)) <= tol, (n, T, b)


def test_eigvals_sym_batched_status_and_limits(dab, rt1):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((6, 6, 5))
    A = X + X.transpose(1, 0, 2)
    for val, bit in ((np.nan, 1), (np.inf, 1), (-np.inf, 1)):
        B = A.copy()
        B[1, 2, 3] = val
        got, status, back = _eig_batch(dab, rt1, B, np.float64)
        assert status == bit and np.all(np.isnan(got[3])) and np.all(np.isfinite(np.delete(got, 3, axis=0)))
        assert np.array_equal(back, B.reshape(-1, order="F"), equal_nan=True)   # the input is left intact
    B = A.copy()
    B[1, 2, 3] += 1e-3                                             # finite, not exactly symmetric (in Float32 too)
    got, status, _ = _eig_batch(dab, rt1, B, np.float32)
    assert status == 2 and np.all(np.isnan(got[3]))
    B[1, 2, 1] = np.nan                                            # one NaN slice and one non-symmetric slice
    assert _eig_batch(dab, rt1, B, np.float64)[1] == 3
    assert _eig_batch(dab, rt1, A, np.float64)[1] == 0             # the status word is cleared by every call
    with pytest.raises(dab.UnsupportedError, match="n <= 64"):
        _eig_batch(dab, rt1, np.ones((65, 65, 1)), np.float64)
    D = dab.distribute(np.ones((65, 65, 2)))
    n1 = rt1.launches()
    with pytest.raises(dab.UnsupportedError, match="64"):
        dab.ppeval(dab.eigvals, D)
    assert rt1.launches() == n1                                    # refused before any launch
    D.close()


def test_reference_testset(dab, rt8):
    """test/darray.jl:973-986 on 8 workers: ppeval(*, A, B) against the per-slice host product with Float64 drandn-like data, the trace
    identity of ppeval(eigvals, S), and the non-symmetric / generalised forms raising UnsupportedError."""
    po.check_reference_testset(dab)


def test_reference_testset_drandn(dab, rt8):
    P = len(dab.workers())
    A = dab.drandn((10, 10, P), dab.workers(), [1, 1, P])
    B = dab.drandn((10, P), dab.workers(), [1, P])
    R = dab.to_array(dab.ppeval(__import__("operator").matmul, A, B))
    a, b = dab.to_array(A), dab.to_array(B)
    assert np.allclose(R, np.stack([a[:, :, i] @ b[:, i] for i in range(P)], axis=1), rtol=1e-13, atol=1e-13)
    with pytest.raises(dab.UnsupportedError):
        dab.ppeval(dab.eigvals, A)
    with pytest.raises(dab.UnsupportedError):
        dab.ppeval(dab.eigvals, A, np.eye(10))


def test_layouts_and_results_vs_oracle(dab, rt8):
    po.check_layouts(dab)


def test_errors_raise_before_any_launch(dab, rt8):
    po.check_errors_before_launch(dab, rt8)


def test_status_errors(dab, rt8):
    po.check_status_errors(dab)
