"""Test infrastructure for ``mapslices`` (the product never imports it).

  * ``jl_mapslices``      NumPy restatement of ``Base.mapslices``: the result-shape rule, scalar results, empty ``dims`` (= ``map``);
  * ``darray_mapslices``  the reference's DArray-level ``mapslices`` (src/mapreduce.jl:191-208) on the CPU oracle: redistribution grid,
                          per-localpart ``mapslices`` and the result layout of ``DArray(reshape(refs, size(procs(D))))``, built from
                          ``oracle.darray_oracle``'s ``make_layout`` / ``distribute`` / ``from_chunks``;
  * ``install_hostmem``   NumPy methods for ``dab_sort_slices`` / ``dab_svdvals_batched`` on the host-memory emulation of the C ABI
                          (tests/hostmem_abi.py), so the host runtime's ``mapslices`` flow runs on a CPU-only machine.
"""
from __future__ import annotations

import itertools

import numpy as np

from oracle import darray_oracle as orc


def result_shape(shape, dims, rshape):
    """Base.mapslices: dimension ``dims[j]`` (ascending) takes ``size(r1, j)``, 1 past ``ndims(r1)``; the others are kept."""
    n = len(dims)
    if len(rshape) > n and any(s > 1 for s in rshape[n:]):
        raise ValueError("DimensionMismatch")
    out = list(shape)
    for j, d in enumerate(dims):
        out[d - 1] = rshape[j] if j < len(rshape) else 1
    return tuple(out)


def jl_mapslices(f, A: np.ndarray, dims) -> np.ndarray:
    """``Base.mapslices(f, A; dims)`` for a NumPy array and a NumPy ``f``."""
    A = np.asarray(A)
    dims = sorted({int(d) for d in dims})
    if not dims:                                                   # isempty(dims) && return map(f, A)
        vals = [np.asarray(f(x))[()] for x in A.ravel(order="F")]
        return np.asarray(vals).reshape(A.shape, order="F")
    N = A.ndim
    others = [k for k in range(N) if k + 1 not in dims]

    def idx_of(combo):
        idx = [slice(None)] * N
        for k, i in zip(others, combo):
            idx[k] = i
        return tuple(idx)

    combos = list(itertools.product(*[range(A.shape[k]) for k in others]))
    r1 = np.asarray(f(A[idx_of(combos[0])]))
    Rsize = result_shape(A.shape, dims, r1.shape)
    R = np.empty(Rsize, dtype=r1.dtype, order="F")
    target = tuple(Rsize[d - 1] for d in dims)
    for combo in combos:
        r = np.asarray(f(A[idx_of(combo)]))
        R[idx_of(combo)] = r.reshape(target, order="F")
    return R


def redistribution_grid(dims_D, grid, dims, nprocs):
    """src/mapreduce.jl:195-199: None when every slice dimension is local, else ``p``."""
    if all(grid[d - 1] == 1 for d in dims):
        return None
    N = len(dims_D)
    p = [1] * N
    nondims = [t for t in range(1, N + 1) if t not in dims]
    if nondims:
        for t, g in zip(nondims, orc.defaultdist_grid([dims_D[t - 1] for t in nondims], nprocs)):
            p[t - 1] = g
    return p


def darray_mapslices(f, d: orc.ODArray, dims) -> orc.ODArray:
    """The reference's ``mapslices(f, D::DArray; dims)`` on the oracle."""
    dims = sorted({int(x) for x in dims})
    p = redistribution_grid(d.dims, d.grid, dims, len(d.pids))
    if p is not None:
        d = orc.distribute(orc.to_array(d), procs=d.pids, dist=p)
    parts = [jl_mapslices(f, ch, dims) for ch in d.chunks]
    return orc.from_chunks(parts, d.grid, d.pids)


# ---- host-memory emulation of the two slice entry points -------------------------------------------------------------------------------


def install_hostmem(fake):
    """Adds ``dab_sort_slices`` / ``dab_svdvals_batched`` to a ``hostmem_abi.HostMemABI`` instance: the fibre sort through the same
    radix-key bijection as the kernels, and the singular values from ``numpy.linalg.svd`` in fp64."""
    import hostmem_abi as H

    def dab_sort_slices(ctx, dtype, inp, out, inner, ln, outer):
        inner, ln, outer = int(inner), int(ln), int(outer)
        n = inner * ln * outer
        if n:
            u = H._utype(dtype)
            raw = H._view(inp, n, u).copy().reshape((inner, ln, outer), order="F")
            s = H.radix_dec(np.sort(H.radix_enc(raw, dtype), axis=1), dtype)
            H._view(out, n, u)[:] = s.reshape(-1, order="F")
            fake.launches += 1
        return 0

    def dab_svdvals_batched(ctx, dtype, A, m, n, batch, S, status):
        m, n, batch = int(m), int(n), int(batch)
        k = min(m, n)
        if k > 32 or m * n > 4096:
            return 6                                               # DAB_ERR_UNSUPPORTED
        dt = np.float32 if int(dtype) == H.F32 else np.float64
        H._view(status, 1, np.int32)[0] = 0
        if batch and k:
            a = H._view(A, m * n * batch, dt).astype(np.float64).reshape((m, n, batch), order="F")
            out = H._view(S, k * batch, dt)
            for b in range(batch):
                M = a[:, :, b]
                if not np.all(np.isfinite(M)):
                    H._view(status, 1, np.int32)[0] = 1
                    out[b * k:(b + 1) * k] = np.nan
                    continue
                out[b * k:(b + 1) * k] = np.linalg.svd(M, compute_uv=False).astype(dt)
            fake.launches += 1
        return 0

    fake.dab_sort_slices = dab_sort_slices
    fake.dab_svdvals_batched = dab_svdvals_batched
    return fake


# ---- scenarios shared by the GPU tier (real kernels, rt8) and the CPU tier (host-memory emulation) ---------------------------------------


def svdvals_np(M):
    return np.linalg.svd(np.asarray(M, dtype=np.float64), compute_uv=False)


def assert_same_layout(got, want):
    """dims, pids, cuts and indices of a product DArray equal the oracle's."""
    assert tuple(got.dims) == tuple(want.dims), (got.dims, want.dims)
    assert list(got.layout.pids) == list(want.pids), (got.layout.pids, want.pids)
    assert [list(c) for c in got.cuts] == [list(c) for c in want.cuts], (got.cuts, want.cuts)
    assert list(got.indices) == list(want.indices)


def check_reference_testset(dab, seed=804):
    """The reference's ``test mapslices`` testset (test/darray.jl:804-841), line by line, on ``dab.workers()``."""
    rng = np.random.default_rng(seed)
    pids = list(dab.workers())
    nw = len(pids)
    A = rng.standard_normal((5, 5, 5))                                              # :805
    D = dab.distribute(A, procs=pids, dist=[1, 1, min(nw, 5)])                      # :806
    oD = orc.distribute(A, procs=pids, dist=[1, 1, min(nw, 5)])
    for dims in ((1, 2), (1, 3), (2, 3)):                                           # :807-809
        got, want = dab.mapslices(dab.svdvals, D, dims=dims), darray_mapslices(svdvals_np, oD, dims)
        assert_same_layout(got, want)
        w = orc.to_array(want)
        assert np.max(np.abs(dab.to_array(got) - w)) <= 1e-12 * np.max(np.abs(w)), dims
    for dims in ((1,), (2,), (3,)):                                                 # :810-812
        got, want = dab.mapslices(dab.sort, D, dims=dims), darray_mapslices(np.sort, oD, dims)
        assert_same_layout(got, want)
        assert np.array_equal(dab.to_array(got), orc.to_array(want)), dims
    # issue #3613 (:814-817)
    ones3 = dab.dones((2, 3, 4), pids, [1, 1, min(nw, 4)])
    B = dab.mapslices(dab.sum, ones3, dims=[1, 2])
    assert B.dims == (1, 1, 4)
    assert np.all(dab.to_array(B) == 6)
    assert_same_layout(B, darray_mapslices(np.sum, orc.distribute(np.ones((2, 3, 4)), procs=pids, dist=[1, 1, min(nw, 4)]), [1, 2]))
    # issue #5141 (:819-821)
    C1 = dab.mapslices(lambda x: dab.maximum(-x), D, dims=[])
    assert np.array_equal(dab.to_array(C1), dab.to_array(-D)) and np.array_equal(dab.to_array(C1), -A)
    assert_same_layout(C1, darray_mapslices(lambda x: np.max(-x), oD, []))
    # issue #5177 (:823-836)
    c = dab.dones((2, 3, 4, 5), pids, [1, 1, 1, min(nw, 5)])
    oc = orc.distribute(np.ones((2, 3, 4, 5)), procs=pids, dist=[1, 1, 1, min(nw, 5)])
    sizes = {}
    for name, const, dims in (("m1", (2, 3), [1, 2]), ("m2", (2, 4), [1, 3]), ("m3", (3, 4), [2, 3]),
                              ("n1", (6,), [1, 2]), ("n2", (6,), [1, 3]), ("n3", (6,), [2, 3]),
                              ("n1a", (1, 6), [1, 2]), ("n2a", (1, 6), [1, 3]), ("n3a", (1, 6), [2, 3])):
        m = dab.mapslices(lambda x, s=const: np.ones(s), c, dims=dims)
        want = darray_mapslices(lambda x, s=const: np.ones(s), oc, dims)
        assert_same_layout(m, want)
        assert m.dtype == np.float64 and np.all(dab.to_array(m) == 1.0)
        sizes[name] = m.dims
    assert sizes["m1"] == sizes["m2"] == sizes["m3"] == c.dims                      # :828
    assert sizes["n1a"] == (1, 6, 4, 5) and sizes["n2a"] == (1, 3, 6, 5) and sizes["n3a"] == (2, 1, 6, 5)   # :835
    assert sizes["n1"] == (6, 1, 4, 5) and sizes["n2"] == (6, 3, 1, 5) and sizes["n3"] == (2, 6, 1, 5)      # :836
    D.close()                                                                       # :837-839
    c.close()
    dab.d_closeall()


def check_layouts(dab, seed=5):
    """Result layouts against the oracle's, for slice dimensions that are already local (no redistribution) and ones that are split
    (redistribution through halo reads), over several element types and slice functions."""
    rng = np.random.default_rng(seed)
    pids = list(dab.workers())
    cases = [((24, 20), None), ((7, 30, 6), None), ((12, 10, 9), [1, 2, min(len(pids) // 2, 4) or 1]), ((40, 16), [len(pids), 1])]
    for shape, dist in cases:
        for T in (np.float64, np.float32, np.int32, np.int64):
            A = (rng.standard_normal(shape) * 100).astype(T)
            D = dab.distribute(A, procs=pids, dist=dist)
            oD = orc.distribute(A, procs=pids, dist=dist if dist is not None else orc.defaultdist_grid(shape, len(pids)))
            assert list(D.layout.pids) == list(oD.pids) and D.indices == oD.indices
            for dims in [(k,) for k in range(1, len(shape) + 1)]:
                got, want = dab.mapslices(dab.sort, D, dims=dims), darray_mapslices(np.sort, oD, dims)
                assert_same_layout(got, want)
                assert np.array_equal(dab.to_array(got), orc.to_array(want)), (shape, dist, T, dims)
            for dims in itertools.combinations(range(1, len(shape) + 1), 2):
                got, want = dab.mapslices(dab.svdvals, D, dims=dims), darray_mapslices(svdvals_np, oD, dims)
                assert_same_layout(got, want)
                w = orc.to_array(want)
                tol = (2e-6 if T == np.float32 else 1e-12) * max(1.0, float(np.max(np.abs(w))))
                assert got.dtype == (np.float32 if T == np.float32 else np.float64)
                assert np.max(np.abs(dab.to_array(got) - w)) <= tol, (shape, dist, T, dims)
            for dims in [(1,), (len(shape),), tuple(range(1, len(shape) + 1))]:
                got = dab.mapslices(lambda x: dab.sum(x * 2), D, dims=dims)
                wt = np.float64 if T in (np.float32, np.float64) else np.int64
                want = darray_mapslices(lambda x: np.sum(x.astype(wt) * 2), oD, dims)
                assert_same_layout(got, want)
                w = orc.to_array(want)
                if T in (np.int32, np.int64):
                    assert np.array_equal(dab.to_array(got), w) and got.dtype == np.int64, (shape, T, dims)
                else:                                               # Float32 sums: fp32 over <= 16-element groups, bound by sum |2x|
                    mag = orc.to_array(darray_mapslices(lambda x: np.sum(np.abs(x.astype(wt)) * 2), oD, dims))
                    tol = 2e-6 if T == np.float32 else 1e-13
                    assert np.all(np.abs(dab.to_array(got) - w) <= tol * mag) and got.dtype == T, (shape, T, dims)
            D.close()
    dab.d_closeall()


def check_errors_before_launch(dab, rt):
    """Invalid ``dims``, ``sort`` over two dimensions, ``svdvals`` over one, and closures that are not served raise before any launch."""
    D = dab.distribute(np.arange(60.0).reshape((3, 4, 5), order="F"))
    n0 = rt.launches()
    for bad in (0, 4, -1, 1.5, "1", [1, 0], (2, 7), None, True):
        try:
            dab.mapslices(dab.sort, D, dims=bad)
        except dab.ArgumentError:
            pass
        else:
            raise AssertionError(f"dims={bad!r} was accepted")
    cases = [(dab.sort, (1, 2), dab.ArgumentError), (dab.sort, (), dab.ArgumentError), (dab.svdvals, (1,), dab.UnsupportedError),
             (dab.svdvals, (1, 2, 3), dab.UnsupportedError), (lambda x: x[0], (1,), dab.UnsupportedError),
             (lambda x: float(x), (1,), dab.UnsupportedError), (lambda x: dab.sort(x * 2), (1,), dab.UnsupportedError),
             (lambda x: dab.sum(x, dims=1), (1,), dab.UnsupportedError), (lambda x: np.fft.fft(x), (1,), dab.UnsupportedError),
             (lambda x: dab.sum(x > 0), (1,), dab.UnsupportedError),
             # NumPy functions of the slice: the tracer refuses array conversion, so none of them is mistaken for a map or a constant
             (np.median, (1,), dab.UnsupportedError), (np.mean, (1,), dab.UnsupportedError), (np.average, (2,), dab.UnsupportedError),
             (np.flip, (1,), dab.UnsupportedError), (lambda x: np.dot(x, x), (1,), dab.UnsupportedError), (np.size, (1,), dab.UnsupportedError),
             (lambda x: np.median(-x), (1,), dab.UnsupportedError), (lambda x: np.percentile(x, 50), (1, 2), dab.UnsupportedError),
             (lambda x: np.asarray(x) * 0 + 1, (1,), dab.UnsupportedError), (np.sum, (1,), dab.UnsupportedError),
             (lambda x: sum(x), (1,), dab.UnsupportedError), (lambda x: len(x), (1,), dab.UnsupportedError)]
    for f, dims, exc in cases:
        try:
            dab.mapslices(f, D, dims=dims)
        except exc:
            pass
        else:
            raise AssertionError(f"{f} over {dims} was accepted")
    try:
        dab.svdvals(D)
    except dab.UnsupportedError as e:
        assert "mapslices" in str(e)
    else:
        raise AssertionError("svdvals(D) was accepted")
    Big = dab.distribute(np.ones((40, 40, 2)), dist=[1, 1, 2] if len(dab.workers()) >= 2 else None)
    n1 = rt.launches()
    try:
        dab.mapslices(dab.svdvals, Big, dims=(1, 2))
    except dab.UnsupportedError as e:
        assert "32" in str(e)
    else:
        raise AssertionError("40x40 slices were accepted")
    assert rt.launches() == n1
    assert rt.launches() == n0
    Big.close()
    D.close()
