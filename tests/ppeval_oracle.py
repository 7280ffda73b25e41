"""Test infrastructure for ``ppeval`` (the product never imports it).

  * ``jl_ppeval``       NumPy restatement of the reference's ``_ppeval(f, A...; dim)`` (src/mapreduce.jl:210-255) on host arrays;
  * ``darray_ppeval``   the reference's ``ppeval(f, D...; dim)`` (:300-323) on the CPU oracle: the distributed-dimension check, one
                        ``_ppeval`` per worker of ``procs(D[1])`` on the localparts, and ``DArray(reshape(refs, (sd[1:nd-1]..., sd[end])))``
                        built with ``oracle.darray_oracle.from_chunks``;
  * ``install_hostmem`` NumPy methods for ``dab_matmul_batched`` / ``dab_eigvals_sym_batched`` on the host-memory emulation of the C ABI
                        (tests/hostmem_abi.py), so the host runtime's ``ppeval`` flow runs on a CPU-only machine.
"""
from __future__ import annotations

import operator

import numpy as np

import mapslices_oracle as mo
from oracle import darray_oracle as orc


class RefError(Exception):
    """What the reference throws: ``kind`` is the Julia exception type."""

    def __init__(self, kind: str, msg: str = ""):
        super().__init__(f"{kind}: {msg}")
        self.kind = kind


def _slice(A, d, i):
    idx = [slice(None)] * A.ndim
    idx[d - 1] = i
    return A[tuple(idx)]


def jl_ppeval(f, *A, dim):
    """``_ppeval(f, A...; dim)``: slice every argument with ``dim[i] > 0`` along it, stack ``f``'s results along a new last dimension."""
    if len(dim) != len(A):
        raise RefError("ArgumentError", f"dim argument has wrong length. length(dim) = {len(dim)} but should be {len(A)}")
    n = A[0].shape[dim[0] - 1]
    for i in range(1, len(A)):
        if dim[i] > 0 and n != A[i].shape[dim[i] - 1]:
            raise RefError("ArgumentError", "lengths of broadcast dimensions must be the same")
    if n == 0:
        raise RefError("BoundsError", "view(A[1], ..., 1, ...) of an empty localpart")
    args = lambda i: [_slice(a, d, i) if d > 0 else a for a, d in zip(A, dim)]
    R1 = np.asarray(f(*args(0)))
    R = np.empty(R1.shape + (n,), dtype=R1.dtype, order="F")
    for i in range(n):
        R[..., i] = f(*args(i))
    return R


def _localpart(d, pid):
    for p, ch in zip(d.pids, d.chunks):
        if p == pid:
            return ch
    return np.empty((0,) * len(d.dims), dtype=d.chunks[0].dtype)


def result_grid(sd, nd, nprocs):
    if nd - 1 > len(sd):
        raise RefError("BoundsError", "sd[1:nd-1]")
    grid = tuple(sd[:nd - 1]) + (sd[-1],)
    if int(np.prod(grid)) != nprocs:
        raise RefError("DimensionMismatch", "reshape(refs, grid)")
    return grid


def tiles_consistently(shapes, grid):
    """Whether ``DArray(refs)`` gets a consistent array: along each grid axis the chunks agree on their extent."""
    for lin, s in enumerate(shapes):
        c = np.unravel_index(lin, grid, order="F")
        for x in range(len(grid)):
            first = [0] * len(grid)
            first[x] = c[x]
            if s[x] != shapes[int(np.ravel_multi_index(first, grid, order="F"))][x]:
                return False
    return True


def darray_ppeval(f, *D, dim=None):
    """The reference's ``ppeval`` on ODArrays (and host arrays, which are broadcast with dim 0)."""
    isd = [isinstance(x, orc.ODArray) for x in D]
    if dim is None:
        dim = tuple(len(x.dims) if b else 0 for x, b in zip(D, isd))
    if len(dim) != len(D):
        raise RefError("ArgumentError", f"dim argument has wrong length. length(dim) = {len(dim)} but should be {len(D)}")
    for x, b, dm in zip(D, isd, dim):
        if b:
            for idxs in x.indices:
                for d in range(1, len(x.dims) + 1):
                    if d != dm and orc.rlen(idxs[d - 1]) != x.dims[d - 1]:
                        raise RefError("DimensionMismatch", f"dimension {d} is distributed. ppeval requires dimension {d} to be completely "
                                       "available on all processors.")
    parts = [jl_ppeval(f, *[_localpart(x, p) if b else x for x, b in zip(D, isd)], dim=dim) for p in D[0].pids]
    grid = result_grid(list(D[0].grid), parts[0].ndim, len(D[0].pids))
    if not tiles_consistently([q.shape for q in parts], grid):
        raise RefError("Inconsistent", "the chunks do not tile the grid")
    return orc.from_chunks(parts, grid, D[0].pids)


# ---- host-memory emulation of the two entry points -------------------------------------------------------------------------------------


def install_hostmem(fake):
    """Adds ``dab_matmul_batched`` / ``dab_eigvals_sym_batched`` (and the mapslices entry points) to a ``hostmem_abi.HostMemABI``:
    products exactly (integers modulo 2^bits, floats in fp64 rounded once), eigenvalues from ``numpy.linalg.eigvalsh`` with the kernel's
    status bits."""
    import hostmem_abi as H
    mo.install_hostmem(fake)

    def dab_matmul_batched(ctx, dtype, m, n, k, A, sa, B, sb, Cp, batch):
        m, n, k, sa, sb, batch = (int(v) for v in (m, n, k, sa, sb, batch))
        dt = H._NP[int(dtype)]
        if m == 0 or n == 0 or batch == 0:
            return 0
        a_n = (batch - 1) * sa + m * k
        b_n = (batch - 1) * sb + k * n
        av = H._view(A, a_n, dt) if k else np.zeros(0, dt)
        bv = H._view(B, b_n, dt) if k else np.zeros(0, dt)
        out = H._view(Cp, m * n * batch, dt)
        for b in range(batch):
            Ab = av[b * sa:b * sa + m * k].reshape((m, k), order="F")
            Bb = bv[b * sb:b * sb + k * n].reshape((k, n), order="F")
            out[b * m * n:(b + 1) * m * n] = exact_matmul(Ab, Bb).reshape(-1, order="F")
        fake.launches += 1
        return 0

    def dab_eigvals_sym_batched(ctx, dtype, A, n, batch, W, status):
        n, batch = int(n), int(batch)
        if n > 64:
            return 6                                               # DAB_ERR_UNSUPPORTED
        dt = np.float32 if int(dtype) == H.F32 else np.float64
        st = H._view(status, 1, np.int32)
        st[0] = 0
        if batch and n:
            a = H._view(A, n * n * batch, dt).astype(np.float64).reshape((n, n, batch), order="F")
            out = H._view(W, n * batch, dt)
            for b in range(batch):
                M = a[:, :, b]
                flag = 1 if not np.all(np.isfinite(M)) else (2 if np.any(M != M.T) else 0)
                st[0] |= flag
                out[b * n:(b + 1) * n] = np.nan if flag else np.linalg.eigvalsh(M).astype(dt)
            fake.launches += 1
        return 0

    fake.dab_matmul_batched = dab_matmul_batched
    fake.dab_eigvals_sym_batched = dab_eigvals_sym_batched
    return fake


def exact_matmul(A, B):
    """Julia's product of one pair of slices: integers exactly with wraparound (Python integers reduced modulo 2^bits), Float64 in fp64,
    Float32 in fp64 rounded once."""
    dt = A.dtype
    if dt.kind == "i":
        bits = dt.itemsize * 8
        P = (A.astype(object) @ B.astype(object)) if A.size and B.size else np.zeros((A.shape[0], B.shape[1]), dtype=object)
        P = np.vectorize(lambda v: ((int(v) + (1 << (bits - 1))) % (1 << bits)) - (1 << (bits - 1)), otypes=[object])(P)
        return np.asarray(P.astype(np.int64) if bits == 64 else P.astype(np.int64).astype(dt), dtype=dt)
    return (A.astype(np.float64) @ B.astype(np.float64)).astype(dt)


# ---- scenarios shared by the GPU tier (real kernels, rt8) and the CPU tier (host-memory emulation) ---------------------------------------


def assert_same_layout(got, want):
    mo.assert_same_layout(got, want)


def _close(got, want, dtype=np.float64):
    w = np.asarray(want, dtype=np.float64)
    tol = (1e-12 if np.dtype(dtype) == np.float64 else 2e-6) * max(1.0, float(np.max(np.abs(w))) if w.size else 1.0)
    return np.max(np.abs(np.asarray(got, dtype=np.float64) - w)) <= tol if w.size else True


def check_reference_testset(dab, seed=973):
    """test/darray.jl:973-986 on ``dab.workers()``: ``ppeval(*, A, B)`` against the per-slice host product, the trace identity of
    ``ppeval(eigvals, S)`` for a symmetrised S, and the two eigvals forms the reference uses on its non-symmetric A."""
    rng = np.random.default_rng(seed)
    pids = list(dab.workers())
    P = len(pids)
    A = rng.standard_normal((10, 10, P))
    B = rng.standard_normal((10, P))
    dA, dB = dab.distribute(A, procs=pids, dist=[1, 1, P]), dab.distribute(B, procs=pids, dist=[1, P])
    R = np.stack([A[:, :, i] @ B[:, i] for i in range(P)], axis=1)
    got = dab.ppeval(operator.matmul, dA, dB)
    assert got.dims == (10, P) and _close(dab.to_array(got), R)
    assert_same_layout(got, darray_ppeval(operator.matmul, orc.distribute(A, procs=pids, dist=[1, 1, P]),
                                          orc.distribute(B, procs=pids, dist=[1, P])))
    assert _close(dab.to_array(dab.ppeval(lambda a, b: a @ b, dA, dB)), R)
    assert _close(dab.to_array(dab.ppeval(dab.matmul, dA, dB)), R)
    S = A + A.transpose(1, 0, 2)
    dS = dab.distribute(S, procs=pids, dist=[1, 1, P])
    E = dab.ppeval(dab.eigvals, dS)
    assert E.dims == (10, P)
    assert abs(float(np.sum(dab.to_array(E))) - float(np.trace(S, axis1=0, axis2=1).sum())) <= 1e-10 * np.abs(S).sum()
    want = np.stack([np.linalg.eigvalsh(S[:, :, i]) for i in range(P)], axis=1)
    assert _close(dab.to_array(E), want)
    for call in (lambda: dab.ppeval(dab.eigvals, dA), lambda: dab.ppeval(dab.eigvals, dA, np.eye(10))):
        try:
            call()
        except dab.UnsupportedError:
            pass
        else:
            raise AssertionError("eigvals of a non-symmetric slice was accepted")
    for x in (dA, dB, dS, got, E):
        x.close()
    dab.d_closeall()


def _compare(dab, got_fn, want_fn, T):
    """The product and the oracle agree: same layout and values, or both refuse (the reference's reshape / BoundsError / inconsistent
    DArray are the product's DimensionMismatch)."""
    try:
        want = want_fn()
    except RefError as e:
        assert e.kind in ("DimensionMismatch", "BoundsError", "Inconsistent"), e
        try:
            got_fn()
        except dab.DimensionMismatch:
            return
        raise AssertionError(f"accepted where the reference fails with {e}")
    got = got_fn()
    assert_same_layout(got, want)
    w = orc.to_array(want)
    if np.dtype(T).kind == "i":
        assert np.array_equal(dab.to_array(got), w.astype(got.dtype)), T
    else:
        assert _close(dab.to_array(got), w, T), T


def check_layouts(dab, seed=11):
    """Results and layouts against the oracle's on ``dab.workers()``: products with sliced and broadcast operands, dim last and not last
    (the packing path), scalar / vector / matrix results of the mapslices forms, eigvals through ppeval and mapslices, four dtypes."""
    rng = np.random.default_rng(seed)
    pids = list(dab.workers())
    P = len(pids)
    nb = 2 * P + 3                                                 # several slices per worker, uneven counts
    last = lambda a: [1] * (a.ndim - 1) + [P]

    def both(a, dist):
        return dab.distribute(a, procs=pids, dist=dist), orc.distribute(a, procs=pids, dist=dist)

    for T in (np.float64, np.float32, np.int32, np.int64):
        fl = T in (np.float32, np.float64)
        mk = (lambda s: (rng.standard_normal(s) * 4).astype(T)) if fl else (lambda s: rng.integers(-2 ** 20, 2 ** 20, s).astype(T))
        A, X, Bm, H, H2 = mk((7, 5, nb)), mk((5, nb)), mk((5, 3, nb)), mk((5, 4)), mk((4, 5))
        (dA, oA), (dX, oX), (dB, oB) = both(A, last(A)), both(X, last(X)), both(Bm, last(Bm))
        # products: matrix x vector, matrix x matrix, a broadcast host operand on either side
        for f, args, oargs in ((operator.matmul, (dA, dX), (oA, oX)), (operator.matmul, (dA, dB), (oA, oB)),
                               (lambda a, h: a @ h, (dA, H), (oA, H)), (lambda b, h: h @ b, (dB, H2), (oB, H2))):
            _compare(dab, lambda: dab.ppeval(f, *args), lambda: darray_ppeval(f, *oargs), T)
        # dim not last: the slices are packed first.  (7, nb, 5) along 2 with (nb, 5) along 1 -- the reference's grid (1, 1) only fits
        # one worker -- and (2P, 7, 5) along 1 with (5, 2P) along 2, whose grid (P, 1) fits
        (dA2, oA2), (dX2, oX2) = both(np.ascontiguousarray(A.transpose(0, 2, 1)), [1, P, 1]), both(np.ascontiguousarray(X.T), [P, 1])
        _compare(dab, lambda: dab.ppeval(operator.matmul, dA2, dX2, dim=(2, 1)), lambda: darray_ppeval(operator.matmul, oA2, oX2, dim=(2, 1)), T)
        A3, X3 = mk((2 * P, 7, 5)), mk((5, 2 * P))
        (dA3, oA3), (dX3, oX3) = both(A3, [P, 1, 1]), both(X3, [1, P])
        _compare(dab, lambda: dab.ppeval(operator.matmul, dA3, dX3, dim=(1, 2)), lambda: darray_ppeval(operator.matmul, oA3, oX3, dim=(1, 2)), T)
        # one sliced argument: the mapslices forms, scalar / matrix / constant vector results
        wide = np.float64 if fl else np.int64
        forms = [(lambda a: dab.sum(a * 2), lambda a: np.sum(a.astype(wide) * 2)), (lambda a: a * 3, lambda a: a.astype(wide) * 3),
                 (lambda a: np.ones(4), lambda a: np.ones(4))]
        if fl:
            forms.append((dab.svdvals, mo.svdvals_np))
        for f, fo in forms:
            _compare(dab, lambda: dab.ppeval(f, dA), lambda: darray_ppeval(fo, oA), T)
            _compare(dab, lambda: dab.ppeval(f, dA3, dim=(1,)), lambda: darray_ppeval(fo, oA3, dim=(1,)), T)
        _compare(dab, lambda: dab.ppeval(dab.sort, dX), lambda: darray_ppeval(np.sort, oX), T)
        # eigvals: dim last, dim first, and mapslices over (1, 3) of the same slices
        S = mk((6, 6, nb))
        S = S + S.transpose(1, 0, 2)
        eig = lambda M: np.linalg.eigvalsh(np.asarray(M, dtype=np.float64))
        ET = np.float32 if T == np.float32 else np.float64
        (dS, oS) = both(S, [1, 1, P])
        _compare(dab, lambda: dab.ppeval(dab.eigvals, dS), lambda: darray_ppeval(eig, oS), ET)
        assert dab.ppeval(dab.eigvals, dS).dtype == ET
        S3 = np.ascontiguousarray(S[:, :, :2 * P].transpose(2, 0, 1))
        (dS3, oS3) = both(S3, [P, 1, 1])
        _compare(dab, lambda: dab.ppeval(dab.eigvals, dS3, dim=(1,)), lambda: darray_ppeval(eig, oS3, dim=(1,)), ET)
        (dS2, oS2) = both(np.ascontiguousarray(S.transpose(0, 2, 1)), [1, P, 1])
        gm, wm = dab.mapslices(dab.eigvals, dS2, dims=(1, 3)), mo.darray_mapslices(eig, oS2, (1, 3))
        assert_same_layout(gm, wm)
        assert gm.dtype == ET and _close(dab.to_array(gm), orc.to_array(wm), ET)
        dab.d_closeall()


def check_errors_before_launch(dab, rt):
    """Every error the issue lists raises before any launch (and leaves nothing behind)."""
    pids = list(dab.workers())
    P = len(pids)
    A = dab.distribute(np.ones((10, 10, 2 * P)), procs=pids, dist=[1, 1, P])
    B = dab.distribute(np.ones((10, 2 * P)), procs=pids, dist=[1, P])
    Bodd = dab.distribute(np.ones((10, 2 * P + 1)), procs=pids, dist=[1, P])
    Int = dab.distribute(np.ones((10, 10, 2 * P), dtype=np.int64), procs=pids, dist=[1, 1, P])
    Rect = dab.distribute(np.ones((4, 6, 2 * P)), procs=pids, dist=[1, 1, P])
    Big = dab.distribute(np.ones((65, 65, P)), procs=pids, dist=[1, 1, P])
    n0 = rt.launches()
    reg0 = dab.registry_size()
    cases = [
        (lambda: dab.ppeval(operator.matmul, A, B, dim=(3,)), dab.ArgumentError, "wrong length"),
        (lambda: dab.ppeval(operator.matmul, A, B, dim=(3, 2, 1)), dab.ArgumentError, "wrong length"),
        (lambda: dab.ppeval(operator.matmul, np.ones((2, 2)), B), dab.ArgumentError, "first argument"),
        (lambda: dab.ppeval(operator.matmul, A, B, dim=(3, 0)), dab.UnsupportedError, "dim"),
        (lambda: dab.ppeval(operator.matmul, A, Bodd), dab.ArgumentError, "lengths of broadcast dimensions") if P > 1 else None,
        (lambda: dab.ppeval(operator.matmul, A, Int), dab.UnsupportedError, "eltypes"),
        (lambda: dab.ppeval(lambda a, b: b @ a, A, B), dab.UnsupportedError, "dimensions"),
        (lambda: dab.ppeval(operator.matmul, A, np.ones((9, 3))), dab.DimensionMismatch, "matrix A has dimensions"),
        (lambda: dab.ppeval(operator.matmul, A, np.ones(9)), dab.DimensionMismatch, "does not match length"),
        (lambda: dab.ppeval(lambda a, b: a * b, A, A), dab.UnsupportedError, "sliced DArrays"),
        (lambda: dab.ppeval(lambda a, b: (2 * a) @ b, A, B), dab.UnsupportedError, "expression"),
        (lambda: dab.ppeval(dab.eigvals, Rect), dab.DimensionMismatch, "matrix is not square: dimensions are (4, 6)"),
        (lambda: dab.ppeval(dab.eigvals, Big), dab.UnsupportedError, "64"),
        (lambda: dab.ppeval(dab.eigvals, A, np.eye(10)), dab.UnsupportedError, "generalised"),
        (lambda: dab.ppeval(dab.eigvals, B), dab.UnsupportedError, "matrix slices"),
        (lambda: dab.ppeval(np.median, A), dab.UnsupportedError, "not a served"),
        (lambda: dab.ppeval(lambda a: a[0], A), dab.UnsupportedError, "not a served"),
        (lambda: dab.mapslices(lambda x: x @ x, A, dims=(1, 2)), dab.UnsupportedError, "ppeval"),
        (lambda: dab.mapslices(dab.eigvals, A, dims=(1,)), dab.UnsupportedError, "matrix slices"),
        (lambda: dab.mapslices(dab.eigvals, Rect, dims=(1, 2)), dab.DimensionMismatch, "not square"),
        (lambda: dab.ppeval(lambda a: dab.sum(a), B, dim=(1,)), dab.DimensionMismatch, "dimension 2 is distributed") if P > 1 else None,
        # the grid formula: scalar results of slices along 1 of a DVector on a (P,) grid are fine; vector results need a (P, P) grid
        (lambda: dab.ppeval(lambda a: np.ones(3), dab.distribute(np.ones(3 * P), procs=pids, dist=[P])), dab.DimensionMismatch, "grid")
        if P > 1 else None,
    ]
    for c in cases:
        if c is None:
            continue
        call, exc, text = c
        try:
            call()
        except exc as e:
            assert text in str(e), (text, str(e))
        else:
            raise AssertionError(f"accepted: expected {exc.__name__} '{text}'")
    assert rt.launches() == n0
    assert dab.registry_size() == reg0
    for x in (A, B, Bodd, Int, Rect, Big):
        x.close()
    try:
        dab.eigvals(np.eye(3))
    except dab.UnsupportedError as e:
        assert "ppeval" in str(e)
    else:
        raise AssertionError("eigvals of a host matrix was accepted")


def check_status_errors(dab):
    """NaN / Inf and non-symmetric slices raise the right error after the kernel has flagged them; nothing is left registered."""
    pids = list(dab.workers())
    P = len(pids)
    rng = np.random.default_rng(5)
    X = rng.standard_normal((5, 5, 2 * P))
    S = X + X.transpose(1, 0, 2)
    reg0 = dab.registry_size()
    for bad, exc, text in ((np.nan, dab.ArgumentError, "Infs or NaNs"), (np.inf, dab.ArgumentError, "Infs or NaNs"),
                           (None, dab.UnsupportedError, "complex")):
        T = S.copy()
        if bad is None:
            T[1, 3, P] += 1e-3                                     # one slice, on one worker, is not exactly symmetric
        else:
            T[2, 2, 2 * P - 1] = bad
        D = dab.distribute(T, procs=pids, dist=[1, 1, P])
        before = dab.to_array(D)
        for call in (lambda: dab.ppeval(dab.eigvals, D), lambda: dab.mapslices(dab.eigvals, D, dims=(1, 2))):
            try:
                call()
            except exc as e:
                assert text in str(e)
            else:
                raise AssertionError(text)
        assert np.array_equal(dab.to_array(D), before, equal_nan=True)
        D.close()
    T = S.copy()
    T[0, 0, 0] = -0.0
    T[1, 0, 0], T[0, 1, 0] = 0.0, -0.0                              # == semantics: -0.0 equals 0.0, so this is symmetric
    D = dab.distribute(T, procs=pids, dist=[1, 1, P])
    assert dab.ppeval(dab.eigvals, D).dims == (5, 2 * P)
    dab.d_closeall()
    assert dab.registry_size() == reg0
