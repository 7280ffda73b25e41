"""TEST INFRASTRUCTURE -- K27 (``dab_ldiv_batched`` / ``dab_det_batched``) for the host-memory emulation of the C ABI (tests/hostmem_abi.py),
and the NumPy / SciPy model of Julia's ``A \\ B`` and ``det(A)`` of one slice that both the emulation and the GPU tests compare against.

  * ``jl_ldiv(A, B)``    Julia's ``\\`` of a square matrix (LinearAlgebra 1.10, generic.jl), restated: the path from the exact structure
                         tests, ``b ./ d`` on the diagonal path, substitution on the triangular ones, ``lu(A) \\ B`` otherwise; returns
                         ``(X, failure)`` with failure None, ``("singular", info)`` or ``("nonfinite", 0)``;
  * ``jl_det(A)``        ``det``: the diagonal product of a triangular matrix, else ``det(lu(A; check=false))``;
  * ``install(fake)``    adds both entries (and the ppeval / mapslices ones of tests/ppeval_oracle.py) to one emulation instance.

The model is restated from LinearAlgebra's source, not checked against a Julia run.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

import hostmem_abi as H
import ppeval_oracle as po

LU_MAX_N = 64                                                    # DAB_LU_MAX_N
STATUS_CLEAR = (1 << 64) - 1
NONFINITE = 0x80


def path_of(A) -> str:
    """``"diag"``, ``"lower"``, ``"upper"`` or ``"lu"``: Julia's istril / istriu with exact ``== 0`` (-0.0 is zero, NaN is not)."""
    lower = not np.any(np.triu(A, 1) != 0)
    upper = not np.any(np.tril(A, -1) != 0)
    if lower and upper:
        return "diag"
    return "lower" if lower else "upper" if upper else "lu"


def _first_zero(d) -> int:
    z = np.flatnonzero(np.asarray(d) == 0)
    return int(z[0]) + 1 if z.size else 0


def _forward(L, B):
    X = np.array(B, dtype=np.float64)
    for s in range(L.shape[0]):
        X[s] = X[s] / L[s, s]
        X[s + 1:] -= np.outer(L[s + 1:, s], X[s])
    return X


def _backward(U, B):
    X = np.array(B, dtype=np.float64)
    for s in range(U.shape[0] - 1, -1, -1):
        X[s] = X[s] / U[s, s]
        X[:s] -= np.outer(U[:s, s], X[s])
    return X


def lu_factor(A):
    """LAPACK getrf (via SciPy) without a finiteness check: (LU, 0-based piv, info) with info the first exactly-zero pivot, 1-based."""
    with np.errstate(all="ignore"):
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            lu, piv = sla.lu_factor(np.asarray(A, dtype=np.float64), check_finite=False)
    return lu, piv, _first_zero(np.diag(lu))


def jl_ldiv(A, B):
    A = np.asarray(A, dtype=np.float64)
    B2 = np.asarray(B, dtype=np.float64).reshape((A.shape[0], -1), order="F")
    path = path_of(A)
    with np.errstate(all="ignore"):
        if path == "diag":
            d = np.diag(A)
            info = _first_zero(d) if B2.shape[1] else 0
            X = B2 / d[:, None]
        elif path == "lower":
            info, X = _first_zero(np.diag(A)), _forward(A, B2)
        elif path == "upper":
            info, X = _first_zero(np.diag(A)), _backward(A, B2)
        else:
            if not np.all(np.isfinite(A)):
                return np.full(B2.shape, np.nan), ("nonfinite", 0)
            lu, piv, info = lu_factor(A)
            X = sla.lu_solve((lu, piv), B2, check_finite=False) if not info else np.full(B2.shape, np.nan)
    return X.reshape(np.shape(B), order="F"), (("singular", info) if info else None)


def jl_det(A) -> float:
    A = np.asarray(A, dtype=np.float64)
    with np.errstate(all="ignore"):
        if path_of(A) != "lu":
            p = 1.0
            for d in np.diag(A):
                p = p * d
            return p
        lu, piv, info = lu_factor(A)
        if info:
            return 0.0
        p = 1.0
        for d in np.diag(lu):
            p = p * d
        swaps = int(np.sum(piv != np.arange(A.shape[0])))
        return -p if swaps % 2 else p


def status_key(b: int, failure) -> int:
    kind, info = failure
    return (b << 8) | (NONFINITE if kind == "nonfinite" else info)


def install(fake):
    """K27 on one emulation instance (with the ppeval / mapslices entries it runs beside)."""
    po.install_hostmem(fake)

    def dab_ldiv_batched(ctx, dtype, n, nrhs, A, sa, B, sb, X, batch, status):
        n, nrhs, sa, sb, batch, dtype = (int(v) for v in (n, nrhs, sa, sb, batch, dtype))
        if dtype not in (H.F32, H.F64) or n > LU_MAX_N:
            return 6                                               # DAB_ERR_UNSUPPORTED, before anything else
        st = H._view(status, 1, np.uint64)
        st[0] = STATUS_CLEAR
        if batch == 0 or n == 0:
            return 0
        dt = H._NP[dtype]
        av = H._view(A, (batch - 1) * sa + n * n, dt)
        bv = H._view(B, (batch - 1) * sb + n * nrhs, dt) if nrhs else np.zeros(0, dt)
        out = H._view(X, n * nrhs * batch, dt)
        best = STATUS_CLEAR
        for b in range(batch):
            Ab = av[b * sa:b * sa + n * n].reshape((n, n), order="F")
            Bb = bv[b * sb:b * sb + n * nrhs].reshape((n, nrhs), order="F")
            x, fail = jl_ldiv(Ab, Bb)
            out[b * n * nrhs:(b + 1) * n * nrhs] = np.asarray(x).astype(dt).reshape(-1, order="F")
            if fail is not None:
                best = min(best, status_key(b, fail))
        st[0] = best
        fake.launches += 1
        return 0

    def dab_det_batched(ctx, dtype, n, A, sa, D, batch):
        n, sa, batch, dtype = (int(v) for v in (n, sa, batch, dtype))
        if dtype not in (H.F32, H.F64) or n > LU_MAX_N:
            return 6
        if batch == 0:
            return 0
        dt = H._NP[dtype]
        av = H._view(A, (batch - 1) * sa + n * n, dt) if n else np.zeros(0, dt)
        out = H._view(D, batch, dt)
        for b in range(batch):
            out[b] = dt.type(jl_det(av[b * sa:b * sa + n * n].reshape((n, n), order="F")))
        fake.launches += 1
        return 0

    fake.dab_ldiv_batched = dab_ldiv_batched
    fake.dab_det_batched = dab_det_batched
    return fake


# ---- scenarios shared by the GPU tier (real K27) and the CPU tier (this emulation) ---------------------------------------------------------


def _close(got, want, T, scale=1.0):
    eps = float(np.finfo(T).eps)
    w = np.asarray(want, dtype=np.float64)
    return np.max(np.abs(np.asarray(got, dtype=np.float64) - w), initial=0.0) <= 1e3 * eps * max(1.0, float(np.max(np.abs(w), initial=0.0))) * scale


def check_forms(dab, seed=27):
    """The public forms on ``dab.workers()`` against the oracle's ``ppeval`` / ``mapslices`` with NumPy's solve and det: the reference's
    testset shapes, a broadcast host operand on either side, matrix right-hand sides, dim not last, Int32 / Int64, mapslices(det)."""
    import operator  # noqa: F401
    import mapslices_oracle as mo
    from oracle import darray_oracle as orc
    rng = np.random.default_rng(seed)
    pids = list(dab.workers())
    P = len(pids)
    nb = 2 * P + 3
    last = lambda a: [1] * (a.ndim - 1) + [P]

    def both(a, dist):
        return dab.distribute(a, procs=pids, dist=dist), orc.distribute(a, procs=pids, dist=dist)

    def compare(got, want, T):
        po.assert_same_layout(got, want)
        RT = np.float32 if np.dtype(T) == np.float32 else np.float64
        assert got.dtype == RT, (got.dtype, T)
        assert _close(dab.to_array(got), orc.to_array(want), RT), T

    solve = lambda a, b: np.linalg.solve(np.asarray(a, np.float64), np.asarray(b, np.float64))
    det = lambda a: np.linalg.det(np.asarray(a, np.float64))
    for T in (np.float64, np.float32, np.int32, np.int64):
        fl = np.dtype(T).kind == "f"
        mk = (lambda s: rng.standard_normal(s).astype(T)) if fl else (lambda s: rng.integers(-9, 10, s).astype(T))
        A = mk((10, 10, nb)) + (10 * np.eye(10, dtype=T))[:, :, None]          # well conditioned, also for the integers
        X, Bm, H, h = mk((10, nb)), mk((10, 3, nb)), (mk((10, 10)) + 10 * np.eye(10, dtype=T)).astype(T), mk((10,))
        (dA, oA), (dX, oX), (dB, oB) = both(A, last(A)), both(X, last(X)), both(Bm, last(Bm))
        for f, fo, args, oargs in ((dab.ldiv, solve, (dA, dX), (oA, oX)), (dab.ldiv, solve, (dA, dB), (oA, oB)),
                                   (lambda a: dab.ldiv(a, h), lambda a: solve(a, h), (dA,), (oA,)),
                                   (lambda b: dab.ldiv(H, b), lambda b: solve(H, b), (dB,), (oB,)),
                                   (dab.ldiv, solve, (dA, h), (oA, h))):
            compare(dab.ppeval(f, *args), po.darray_ppeval(fo, *oargs), T)
        compare(dab.ppeval(dab.det, dA), po.darray_ppeval(det, oA), T)
        # dim not last: (2P, 10, 10) along 1 with (10, 2P) along 2
        A3, X3 = np.ascontiguousarray(A[:, :, :2 * P].transpose(2, 0, 1)), np.ascontiguousarray(X[:, :2 * P])
        (dA3, oA3), (dX3, oX3) = both(A3, [P, 1, 1]), both(X3, [1, P])
        compare(dab.ppeval(dab.ldiv, dA3, dX3, dim=(1, 2)), po.darray_ppeval(solve, oA3, oX3, dim=(1, 2)), T)
        if P == 1:
            compare(dab.ppeval(dab.det, dA3, dim=(1,)), po.darray_ppeval(det, oA3, dim=(1,)), T)
        else:                                                      # scalar results on the procs grid (P, 1, 1): reshape(refs, (1,)) fails
            try:
                dab.ppeval(dab.det, dA3, dim=(1,))
            except dab.DimensionMismatch:
                pass
            else:
                raise AssertionError("det of slices along 1 accepted on a grid the reference cannot reshape")
        # mapslices(det) over dims (1, 3) of a (10, nb, 10) array
        (dS, oS) = both(np.ascontiguousarray(A.transpose(0, 2, 1)), [1, P, 1])
        gm, wm = dab.mapslices(dab.det, dS, dims=(1, 3)), mo.darray_mapslices(det, oS, (1, 3))
        po.assert_same_layout(gm, wm)
        assert gm.dims == (1, nb, 1) and _close(dab.to_array(gm), orc.to_array(wm), np.float32 if T == np.float32 else np.float64)
        dab.d_closeall()
    # structured slices take Julia's other paths: diagonal, lower, upper, and a 1 x 1 slice
    D = np.zeros((6, 6, nb))
    for b in range(nb):
        M = rng.standard_normal((6, 6)) + 6 * np.eye(6)
        D[:, :, b] = [np.diag(np.diag(M)), np.tril(M), np.triu(M)][b % 3]
    (dD, oD), (dX6, oX6) = both(D, last(D)), both(rng.standard_normal((6, nb)), [1, P])
    compare(dab.ppeval(dab.ldiv, dD, dX6), po.darray_ppeval(solve, oD, oX6), np.float64)
    compare(dab.ppeval(dab.det, dD), po.darray_ppeval(det, oD), np.float64)
    (d1, o1), (x1, ox1) = both(rng.standard_normal((1, 1, nb)), [1, 1, P]), both(rng.standard_normal((1, nb)), [1, P])
    compare(dab.ppeval(dab.ldiv, d1, x1), po.darray_ppeval(solve, o1, ox1), np.float64)
    dab.d_closeall()


def check_errors_before_launch(dab, rt):
    """Every refusal raises before anything is launched or registered."""
    pids = list(dab.workers())
    P = len(pids)
    A = dab.distribute(np.ones((10, 10, 2 * P)), procs=pids, dist=[1, 1, P])
    A32 = dab.distribute(np.ones((10, 10, 2 * P), dtype=np.float32), procs=pids, dist=[1, 1, P])
    B = dab.distribute(np.ones((10, 2 * P)), procs=pids, dist=[1, P])
    Bool = dab.distribute(np.ones((10, 10, 2 * P), dtype=bool), procs=pids, dist=[1, 1, P])
    Rect = dab.distribute(np.ones((4, 6, 2 * P)), procs=pids, dist=[1, 1, P])
    Big = dab.distribute(np.ones((65, 65, P)), procs=pids, dist=[1, 1, P])
    Z = dab.distribute(np.ones((3, 3, P), dtype=np.complex128), procs=pids, dist=[1, 1, P])
    F16 = dab.distribute(np.ones((3, 3, P), dtype=np.float16), procs=pids, dist=[1, 1, P])
    n0, reg0 = rt.launches(), dab.registry_size()
    cases = [
        (lambda: dab.ppeval(dab.ldiv, A, dab.distribute(np.ones((10, 2 * P), dtype=np.float32), procs=pids, dist=[1, P])),
         dab.UnsupportedError, "eltypes"),
        (lambda: dab.ppeval(dab.ldiv, A32, np.ones(10)), dab.UnsupportedError, "eltypes"),
        (lambda: dab.ppeval(dab.ldiv, Bool, np.ones((10, 2), dtype=bool)), dab.UnsupportedError, "eltypes"),
        (lambda: dab.ppeval(dab.ldiv, Rect, np.ones(4)), dab.UnsupportedError, "least-squares"),
        (lambda: dab.ppeval(dab.ldiv, Big, np.ones(65)), dab.UnsupportedError, "64"),
        (lambda: dab.ppeval(dab.ldiv, A, np.ones(9)), dab.DimensionMismatch, "B has leading dimension 9, but needs 10"),
        (lambda: dab.ppeval(dab.ldiv, A, np.ones((11, 2))), dab.DimensionMismatch, "11"),
        (lambda: dab.ppeval(dab.ldiv, B, B), dab.UnsupportedError, "square matrix"),
        (lambda: dab.ppeval(lambda a, b: dab.ldiv(a * 2, b), A, B), dab.UnsupportedError, "expression"),
        (lambda: dab.ppeval(dab.ldiv, Z, np.ones(3)), dab.UnsupportedError, "complex"),
        (lambda: dab.ppeval(dab.det, F16), dab.UnsupportedError, "Float16"),
        (lambda: dab.ppeval(dab.det, Rect), dab.DimensionMismatch, "matrix is not square: dimensions are (4, 6)"),
        (lambda: dab.ppeval(dab.det, Big), dab.UnsupportedError, "64"),
        (lambda: dab.ppeval(dab.det, B), dab.UnsupportedError, "matrix slices"),
        (lambda: dab.ppeval(dab.det, Bool), dab.UnsupportedError, "eltype"),
        (lambda: dab.ppeval(lambda a: dab.det(a + 1), A), dab.UnsupportedError, "expression"),
        (lambda: dab.mapslices(lambda a: dab.ldiv(a, np.ones(10)), A, dims=(1, 2)), dab.UnsupportedError, "ppeval"),
        (lambda: dab.mapslices(dab.det, A, dims=(1,)), dab.UnsupportedError, "matrix slices"),
        (lambda: dab.mapslices(dab.det, Rect, dims=(1, 2)), dab.DimensionMismatch, "not square"),
        (lambda: dab.mapslices(dab.det, A[1:5, 1:5, 0:2], dims=(1, 2)), dab.UnsupportedError, "view"),
        (lambda: dab.ppeval(lambda a: np.linalg.solve(a, np.ones(10)), A), dab.UnsupportedError, "ldiv"),
    ]
    for call, exc, text in cases:
        try:
            call()
        except exc as e:
            assert text in str(e), (text, str(e))
        else:
            raise AssertionError(f"accepted: expected {exc.__name__} '{text}'")
    assert rt.launches() == n0
    assert dab.registry_size() == reg0
    for x in (A, A32, B, Bool, Rect, Big, Z, F16):
        x.close()
    for f in (lambda: dab.ldiv(np.eye(3), np.ones(3)), lambda: dab.det(np.eye(3))):
        try:
            f()
        except dab.UnsupportedError as e:
            assert "ppeval" in str(e)
        else:
            raise AssertionError("a host ldiv / det was accepted")
    dab.d_closeall()


def check_status_errors(dab):
    """SingularException(k) and ArgumentError from the kernel's status word: the first failing slice in the order of the result's last
    dimension decides, every rank raises the same exception, nothing stays registered and the input is left intact."""
    pids = list(dab.workers())
    P = len(pids)
    nb = 2 * P + 1
    rng = np.random.default_rng(6)
    A = rng.standard_normal((5, 5, nb)) + 5 * np.eye(5)[:, :, None]
    B = rng.standard_normal((5, nb))
    dB = dab.distribute(B, procs=pids, dist=[1, P])
    lower_sing = np.tril(A[:, :, 0])
    lower_sing[0, 0] = 0.0                                         # lower: info 1 (LU pivoting would report another index)
    upper_sing = np.triu(A[:, :, 0])
    upper_sing[3, 3] = -0.0                                        # upper: info 4 (-0.0 is zero)
    lu_sing = A[:, :, 0].copy()
    lu_sing[:, 2] = 0.0                                            # dense with a zero column: the third pivot is exactly zero
    diag_sing = np.diag([1.0, 2.0, 0.0, 3.0, 0.0])
    lu_nan = A[:, :, 0].copy()
    lu_nan[4, 1] = np.nan
    cases = [(lower_sing, dab.SingularException, 1), (upper_sing, dab.SingularException, 4), (lu_sing, dab.SingularException, 3),
             (diag_sing, dab.SingularException, 3), (lu_nan, dab.ArgumentError, None)]
    for M, exc, info in cases:
        for where in sorted({nb - 1, nb // 2}):
            T = A.copy()
            T[:, :, where] = M
            D = dab.distribute(T, procs=pids, dist=[1, 1, P])
            before = dab.to_array(D)
            reg1 = dab.registry_size()
            try:
                dab.ppeval(dab.ldiv, D, dB)
            except exc as e:
                assert info is None or (e.info == info and str(e) == f"SingularException({info})"), (str(e), info)
                assert info is not None or "Infs or NaNs" in str(e)
            else:
                raise AssertionError(f"accepted: {exc.__name__}")
            assert dab.registry_size() == reg1                     # nothing left registered
            assert np.array_equal(dab.to_array(D), before, equal_nan=True)
            assert np.isfinite(dab.to_array(dab.ppeval(dab.det, D))).all() == (info is not None)
            D.close()
    # two failing slices on different workers: the one earlier in the result's last dimension wins, whatever its kind
    T = A.copy()
    T[:, :, nb - 1] = lu_nan
    T[:, :, 1] = upper_sing
    D = dab.distribute(T, procs=pids, dist=[1, 1, P])
    try:
        dab.ppeval(dab.ldiv, D, dB)
    except dab.SingularException as e:
        assert e.info == 4
    else:
        raise AssertionError("accepted")
    D.close()
    # NaN / Inf flow through the diagonal and triangular paths; a NaN above the diagonal of an upper slice never reaches det
    T = A.copy()
    T[:, :, 0] = np.diag([1.0, np.nan, 2.0, np.inf, 4.0])
    T[:, :, 1] = np.tril(A[:, :, 1])
    T[3, 0, 1] = np.nan
    T[:, :, 2] = np.triu(A[:, :, 2])
    T[0, 4, 2] = np.nan
    D = dab.distribute(T, procs=pids, dist=[1, 1, P])
    got = dab.to_array(dab.ppeval(dab.ldiv, D, dB))
    for b in range(3):
        want, fail = jl_ldiv(T[:, :, b], B[:, b])
        assert fail is None and np.array_equal(np.isnan(got[:, b]), np.isnan(want))
    dets = dab.to_array(dab.ppeval(dab.det, D))
    assert np.isnan(dets[0]) and np.isfinite(dets[2]) and dets[2] == jl_det(T[:, :, 2])
    dab.d_closeall()
