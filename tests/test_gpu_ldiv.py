"""GPU tests of K27 (``dab_ldiv_batched`` / ``dab_det_batched``) and of the public ``ppeval(ldiv, A, B)``, ``ppeval(det, A)`` and
``mapslices(det, D, dims)`` forms: residual and determinant bounds against NumPy, the diagonal path bit for bit, the path, ``info`` and
non-finite handling of every path against the model of Julia's dispatch in tests/ldiv_hostmem.py, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import ldiv_hostmem as lh

pytestmark = pytest.mark.gpu

NS = (1, 2, 10, 31, 32, 33, 63, 64)


@pytest.fixture(autouse=True)
def _k27_on_the_host_memory_abi():
    """Under ``DAB_HOSTMEM=1`` the library is the host-memory emulation: give it the model of K27 (a no-op on the GPU)."""
    import hostmem_abi
    from darray_b200 import _lib
    if isinstance(_lib._lib, hostmem_abi.HostMemABI):
        lh.install(_lib._lib)


def _ldiv(dab, rt, A, B, T, bcast_a=False, bcast_b=False):
    """X[:, :, b] = A[:, :, b] \\ B[:, :, b] on the GPU; a broadcast operand is passed as its one slice with stride 0.  Returns X, the status
    word and the inputs read back."""
    from darray_b200 import _lib
    n, _, batch = A.shape
    nrhs = B.shape[1]
    a = A[:, :, :1] if bcast_a else A
    b = B[:, :, :1] if bcast_b else B
    dA = dab.B200Array.from_numpy(rt, np.asfortranarray(a, dtype=T).reshape(-1, order="F"))
    dB = dab.B200Array.from_numpy(rt, np.asfortranarray(b, dtype=T).reshape(-1, order="F")) if b.size else None
    dX = dab.B200Array.empty(rt, (max(1, n * nrhs * batch),), T)
    st = dab.B200Array.empty(rt, (1,), np.int64)
    try:
        _lib.call("dab_ldiv_batched", rt.ctx, dab.dab_dtype(np.dtype(T)), n, nrhs, C.c_void_p(dA.ptr), 0 if bcast_a else n * n,
                  C.c_void_p(dB.ptr if dB else 0), 0 if bcast_b else n * nrhs, C.c_void_p(dX.ptr), batch, C.c_void_p(st.ptr))
        X = dX.to_numpy()[:n * nrhs * batch].reshape((n, nrhs, batch), order="F")
        return X, int(st.to_numpy()[0]) & lh.STATUS_CLEAR, dA.to_numpy(), (dB.to_numpy() if dB else None)
    finally:
        for x in (dA, dB, dX, st):
            if x is not None:
                x.free()


def _det(dab, rt, A, T):
    from darray_b200 import _lib
    n, _, batch = A.shape
    dA = dab.B200Array.from_numpy(rt, np.asfortranarray(A, dtype=T).reshape(-1, order="F")) if A.size else None
    dD = dab.B200Array.empty(rt, (batch,), T)
    try:
        _lib.call("dab_det_batched", rt.ctx, dab.dab_dtype(np.dtype(T)), n, C.c_void_p(dA.ptr if dA else 0), n * n, C.c_void_p(dD.ptr), batch)
        return dD.to_numpy()
    finally:
        for x in (dA, dD):
            if x is not None:
                x.free()


def _well_conditioned(rng, n, batch):
    return rng.standard_normal((n, n, batch)) + 3 * np.sqrt(n) * np.eye(n)[:, :, None]


@pytest.mark.parametrize("T", [np.float64, np.float32])
@pytest.mark.parametrize("n", NS)
def test_ldiv_residual_and_det(dab, rt1, T, n):
    """‖A x − b‖∞ <= c n ε (‖A‖∞ ‖x‖∞ + ‖b‖∞) for every slice, nrhs 1 / 3 / 65, A or B broadcast; |det − numpy| <= c n ε |det|."""
    rng = np.random.default_rng(100 + n)
    eps = float(np.finfo(T).eps)
    batch = 37
    for nrhs in (1, 3, 65):
        for ba, bb in ((False, False), (True, False), (False, True)):
            A = _well_conditioned(rng, n, batch).astype(T)
            B = rng.standard_normal((n, nrhs, batch)).astype(T)
            if ba:
                A = np.repeat(A[:, :, :1], batch, axis=2)
            if bb:
                B = np.repeat(B[:, :, :1], batch, axis=2)
            X, st, _, _ = _ldiv(dab, rt1, A, B, T, ba, bb)
            assert st == lh.STATUS_CLEAR and X.dtype == np.dtype(T)
            for b in range(batch):
                a, x, r = A[:, :, b].astype(np.float64), X[:, :, b].astype(np.float64), B[:, :, b].astype(np.float64)
                res = np.max(np.abs(a @ x - r))
                bound = 8 * n * eps * (np.max(np.abs(a).sum(axis=1)) * np.max(np.abs(x)) + np.max(np.abs(r)))
                assert res <= bound, (n, nrhs, ba, bb, b, res, bound)
    A = (_well_conditioned(rng, n, 64) / (3 * np.sqrt(n))).astype(T)           # |det| near 1: inside Float32 range
    got = _det(dab, rt1, A, T)
    want = np.linalg.det(A.astype(np.float64).transpose(2, 0, 1))
    assert got.dtype == np.dtype(T)
    rel = np.abs(got.astype(np.float64) - want) / np.abs(want)
    assert np.all(rel <= 64 * n * eps), (n, float(np.max(rel)))


@pytest.mark.parametrize("T", [np.float64, np.float32])
def test_ldiv_diagonal_path_bit_exact(dab, rt1, T):
    rng = np.random.default_rng(4)
    for n in (1, 5, 32, 33, 64):
        d = (rng.standard_normal((n, 7)) * 10.0 ** rng.integers(-30, 30, (n, 7))).astype(T)
        A = np.zeros((n, n, 7), dtype=T)
        for b in range(7):
            A[:, :, b] = np.diag(d[:, b])
        if n > 1:
            A[0, n - 1, 3] = -0.0                                  # -0.0 off the diagonal is still zero
        B = (rng.standard_normal((n, 3, 7)) * 10.0 ** rng.integers(-30, 30, (n, 3, 7))).astype(T)
        B[0, 0, 1], B[n - 1, 1, 2] = np.inf, np.nan
        X, st, _, _ = _ldiv(dab, rt1, A, B, T)
        assert st == lh.STATUS_CLEAR
        assert np.array_equal(X.view(np.uint32 if T == np.float32 else np.uint64),
                              (B / d[:, None, :]).astype(T).view(np.uint32 if T == np.float32 else np.uint64)), n


def _model_case(A, B):
    """The model's result and status word for a batch."""
    best, xs = lh.STATUS_CLEAR, []
    for b in range(A.shape[2]):
        x, fail = lh.jl_ldiv(A[:, :, b], B[:, :, b])
        xs.append(x)
        if fail is not None:
            best = min(best, lh.status_key(b, fail))
    return np.stack(xs, axis=2), best


@pytest.mark.parametrize("T", [np.float64, np.float32])
@pytest.mark.parametrize("n", [2, 5, 16, 32, 40, 64])
def test_paths_status_and_values_vs_model(dab, rt1, T, n):
    """Every path with and without a singular or non-finite entry, against the model of Julia's dispatch: the status word (lowest failing
    slice, info, non-finite flag), the values of the slices that succeed, det on each path, and the input left intact."""
    rng = np.random.default_rng(n)
    M = [_well_conditioned(rng, n, 1)[:, :, 0] for _ in range(4)]
    mats = [np.diag(np.diag(M[0])), np.tril(M[1]), np.triu(M[2]), M[3]]
    cases = []
    for base in mats:
        cases.append(base)
        for k in sorted({0, n // 2, n - 1}):
            Z = base.copy()
            Z[k, k] = 0.0                                          # a zero diagonal entry
            if np.array_equal(base, M[3]):
                Z = base.copy()
                Z[:, k] = 0.0                                      # a zero column: pivot k + 1 is exactly zero
            cases.append(Z)
        for v in (np.nan, np.inf):
            Z = base.copy()
            Z[n - 1, 0] = v                                        # below the diagonal
            cases.append(Z)
            Z = base.copy()
            Z[0, n - 1] = v                                        # above the diagonal
            cases.append(Z)
    L = np.tril(M[1])
    L[0, 0] = 0.0                                                  # lower: info 1, where LU pivoting would report another index
    cases.append(L)
    A = np.stack(cases, axis=2).astype(T)
    B = rng.standard_normal((n, 2, A.shape[2])).astype(T)
    for lo in range(A.shape[2]):                                   # the status word is the lowest failing slice
        X, st, a_back, b_back = _ldiv(dab, rt1, A[:, :, lo:], B[:, :, lo:], T)
        Xw, stw = _model_case(A[:, :, lo:].astype(np.float64), B[:, :, lo:].astype(np.float64))
        assert st == stw, (n, lo, hex(st), hex(stw))
        if lo == 0:
            assert np.array_equal(a_back, A.reshape(-1, order="F"), equal_nan=True)
            assert np.array_equal(b_back, B.reshape(-1, order="F"), equal_nan=True)
            eps = float(np.finfo(T).eps)
            for b in range(A.shape[2]):
                _, fail = lh.jl_ldiv(A[:, :, b].astype(np.float64), B[:, :, b].astype(np.float64))
                if fail is not None:
                    continue
                w, g = Xw[:, :, b], X[:, :, b].astype(np.float64)
                assert np.array_equal(np.isnan(g), np.isnan(w)), (n, b)
                fin = np.isfinite(w)
                assert np.all(np.abs(g[fin] - w[fin]) <= 1e4 * n * eps * np.maximum(1.0, np.abs(w[fin]))), (n, b)
        if lo > 4:
            break
    got = _det(dab, rt1, A, T)
    for b in range(A.shape[2]):
        with np.errstate(over="ignore"):
            want = float(np.asarray(lh.jl_det(A[:, :, b].astype(np.float64))).astype(T))    # rounded once to T
        g = float(got[b])
        if np.isnan(want):
            assert np.isnan(g), b
        elif want == 0.0:
            assert g == 0.0 and (np.signbit(g) == np.signbit(want) or lh.path_of(A[:, :, b]) == "lu"), b
        else:
            assert g == want if np.isinf(want) else abs(g - want) <= 64 * n * float(np.finfo(T).eps) * abs(want), (b, g, want)


def test_status_cleared_launches_and_refusals(dab, rt1):
    rng = np.random.default_rng(9)
    A = _well_conditioned(rng, 10, 1000)
    B = rng.standard_normal((10, 1, 1000))
    Z = A.copy()
    Z[:, :, 500] = 0.0
    assert _ldiv(dab, rt1, Z, B, np.float64)[1] == lh.status_key(500, ("singular", 1))
    assert _ldiv(dab, rt1, A, B, np.float64)[1] == lh.STATUS_CLEAR      # the word is cleared by every call
    for batch in (1, 1000):                                       # one launch whatever the batch
        n0 = rt1.launches()
        _ldiv(dab, rt1, A[:, :, :batch], B[:, :, :batch], np.float64)
        assert rt1.launches() - n0 == 1
        n0 = rt1.launches()
        _det(dab, rt1, A[:, :, :batch], np.float64)
        assert rt1.launches() - n0 == 1
    assert np.array_equal(_det(dab, rt1, np.zeros((0, 0, 3)), np.float64), np.ones(3))
    with pytest.raises(dab.UnsupportedError):
        _ldiv(dab, rt1, A.astype(np.int32), B.astype(np.int32), np.int32)
    with pytest.raises(dab.UnsupportedError):
        _ldiv(dab, rt1, np.ones((65, 65, 1)), np.ones((65, 1, 1)), np.float64)
    with pytest.raises(dab.UnsupportedError):
        _det(dab, rt1, np.ones((65, 65, 1)), np.float64)
    with pytest.raises(dab.UnsupportedError):
        _det(dab, rt1, np.ones((3, 3, 1), dtype=np.int64), np.int64)


@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_reference_testset_shapes(dab, request, rtname):
    """The reference's ppeval testset shapes: drandn((10, 10, P)) with drandn((10, P)); ldiv against a per-slice numpy.linalg.solve and
    det against numpy.linalg.det."""
    request.getfixturevalue(rtname)
    P = len(dab.workers())
    A = dab.drandn((10, 10, P), dab.workers(), [1, 1, P])
    B = dab.drandn((10, P), dab.workers(), [1, P])
    a, b = dab.to_array(A), dab.to_array(B)
    X = dab.ppeval(dab.ldiv, A, B)
    assert X.dims == (10, P) and X.layout.grid == (1, P)
    want = np.stack([np.linalg.solve(a[:, :, i], b[:, i]) for i in range(P)], axis=1)
    assert np.allclose(dab.to_array(X), want, rtol=1e-10, atol=1e-10)
    Dt = dab.ppeval(dab.det, A)
    assert Dt.dims == (P,)
    assert np.allclose(dab.to_array(Dt), [np.linalg.det(a[:, :, i]) for i in range(P)], rtol=1e-12, atol=0)


@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_public_forms_vs_oracle(dab, request, rtname):
    request.getfixturevalue(rtname)
    lh.check_forms(dab)


@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_refusals_before_any_launch(dab, request, rtname):
    rt = request.getfixturevalue(rtname)
    lh.check_errors_before_launch(dab, rt)


@pytest.mark.parametrize("rtname", ["rt1", "rt8"])
def test_singular_and_nonfinite_errors(dab, request, rtname):
    request.getfixturevalue(rtname)
    lh.check_status_errors(dab)
