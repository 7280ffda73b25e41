"""GPU tests of sparse DArrays (row f9): K18 ``dab_spmv`` and K19 ``dab_csc_to_csr`` against the model of SparseArrays' loops
(tests/sparse_oracle.py), bit for bit (NaN payloads aside), and the public API around them -- ``distribute`` of a scipy.sparse matrix,
``nnz``, ``to_array``, ``copyto``, ``A*x`` / ``A'*x`` / ``mul!`` on 8-worker grids, the launch and lifetime contracts and the refusals."""
import ctypes as C
import gc
import os

import numpy as np
import pytest
import scipy.sparse as sp

import sparse_oracle as so

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets the sparse entry points too
    import sparse_hostmem
    sparse_hostmem.install()
DTYPES = [np.float32, np.float64, np.int32, np.int64]
GROUPS = (0,) if HOSTMEM else (0, 1, 2, 4, 8, 16, 32)      # 0: the mix as it is; the emulation has no group sizes


def _values(rng, dtype, k, special=True):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = rng.standard_normal(k).astype(dt) * dt.type(3)
        if special and k:
            pos = rng.integers(0, k, max(1, k // 16))
            v[pos] = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e30, -1e-30], dtype=dt), pos.size)
        return v
    hi = 2 ** 30 if dt == np.int32 else 2 ** 62                   # products and sums overflow: the wrap-around is part of the contract
    v = rng.integers(-hi, hi, k).astype(dt)
    if special and k:
        v[rng.integers(0, k, max(1, k // 16))] = 0
    return v


def _sparse(rng, dtype, m, n, density, zero_block=None, empty_rows=(), empty_cols=()):
    """A random m x n CSC matrix with explicit zeros, ±0 / NaN / ±Inf entries, and the given empty rows, columns and zero block."""
    k = int(m * n * density)
    r = rng.integers(0, m, k)
    c = rng.integers(0, n, k)
    keep = ~np.isin(r, list(empty_rows)) & ~np.isin(c, list(empty_cols))
    if zero_block is not None:
        (ra, rb), (ca, cb) = zero_block
        keep &= ~((r >= ra) & (r < rb) & (c >= ca) & (c < cb))
    r, c = r[keep], c[keep]
    S = sp.csc_matrix((_values(rng, dtype, r.size), (r, c)), shape=(m, n), dtype=dtype)
    S.data[::7] = 0                                               # explicitly stored zeros
    return S


def _dense(S):
    """Matrix(S): every stored value in its place, -0.0 included (scipy's toarray() adds into zeros and turns -0.0 into +0.0)."""
    r, c, v = so.canonical_triplets(S)
    a = np.zeros(S.shape, dtype=S.dtype)
    a[r, c] = v
    return a


def _rows_csr(rng, dtype, lengths, ncols):
    """CSR arrays whose rows have exactly the given lengths (columns ascending within a row)."""
    ptr = np.zeros(len(lengths) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum(lengths)
    idx = np.concatenate([np.sort(rng.choice(ncols, L, replace=False)) if L else np.zeros(0, np.int64) for L in lengths]).astype(np.int32)
    return ptr, idx, _values(rng, dtype, int(ptr[-1]))


def _spmv(dab, rt, ptr, idx, val, x):
    from darray_b200 import _lib
    nrows, nnz = len(ptr) - 1, int(ptr[-1])
    bufs = [dab.B200Array.from_numpy(rt, a) for a in (ptr, idx, val, x)]
    out = dab.B200Array.empty(rt, (nrows,), val.dtype)
    _lib.call("dab_spmv", rt.ctx, dab.dab_dtype(val.dtype), nrows, nnz, *[C.c_void_p(b.ptr) for b in bufs], C.c_void_p(out.ptr))
    got = out.to_numpy()
    for b in bufs + [out]:
        b.free()
    return got


def _spmv_group(nrows, nnz):
    """Lanes per row that ``spmv_group()`` (dab_sparse.cu) picks: the smallest power of two >= the mean row length, 1..32."""
    mean = -(-nnz // nrows) if nrows else 0
    return min(32, 1 << max(mean - 1, 0).bit_length())


def _pad_to_group(lengths, g):
    """The row-length mix followed by empty rows (to lower the mean) or rows of 32 entries (to raise it) until it selects G = g."""
    nrows, nnz = len(lengths), int(sum(lengths))
    empty = full = 0
    while (G := _spmv_group(nrows, nnz)) != g:
        if G > g:
            empty += 1
        else:
            full += 1
            nnz += 32
        nrows += 1
    return list(lengths) + [0] * empty + [32] * full


@pytest.mark.parametrize("dtype", DTYPES)
def test_spmv_kernel_padded_to_every_group_size(dab, rt1, dtype):
    """K18 on rows of 0, 1, 31, 33, 1024 and 10^5 entries mixed with short rows, each mix as it is and padded until its mean row length
    selects each lanes-per-row choice: the ordered fold, bit for bit."""
    rng = np.random.default_rng(101)
    ncols = 120000
    x = _values(rng, dtype, ncols)
    for mix in ([1] * 300, [31] * 70 + [0] * 5, [33] * 64, [1024] * 9 + [0, 1, 2], [100000, 3, 0, 31, 33, 1024], [0] * 17,
                list(rng.integers(0, 40, 2000))):
        for g in GROUPS:
            lengths = _pad_to_group(mix, g) if g else mix
            ptr, idx, val = _rows_csr(rng, dtype, lengths, ncols)
            assert g == 0 or _spmv_group(len(lengths), int(ptr[-1])) == g
            got = _spmv(dab, rt1, ptr, idx, val, x)
            assert so.same_bits(got, so.fold_rows(ptr, idx, val, x)), (np.dtype(dtype), mix[:4], g)


@pytest.mark.parametrize("dtype", DTYPES)
def test_csc_to_csr_kernel(dab, rt1, dtype):
    """K19: rows ascending, columns ascending within a row, values carried along; empty rows and columns, an empty chunk, one long row."""
    from darray_b200 import _lib
    rng = np.random.default_rng(7)
    for (m, n, dens) in [(50, 40, 0.2), (1, 3000, 0.5), (3000, 2, 0.3), (9, 9, 0.0), (0, 5, 0.0), (5, 0, 0.0), (700, 900, 0.01)]:
        S = _sparse(rng, dtype, m, n, dens, empty_rows=range(0, m, 5), empty_cols=range(0, n, 7))
        colptr, rowval, nzval = S.indptr.astype(np.int64), S.indices.astype(np.int32), S.data
        nnz = int(colptr[-1])
        bufs = [dab.B200Array.from_numpy(rt1, a) for a in (colptr, rowval, nzval)]
        outs = [dab.B200Array.empty(rt1, (m + 1,), np.int64), dab.B200Array.empty(rt1, (nnz,), np.int32), dab.B200Array.empty(rt1, (nnz,), dtype)]
        _lib.call("dab_csc_to_csr", rt1.ctx, dab.dab_dtype(dtype), m, n, nnz, *[C.c_void_p(b.ptr) for b in bufs + outs])
        got = [o.to_numpy() for o in outs]
        want = so.csc_to_csr(m, colptr, rowval, nzval)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and so.same_bits(got[2], want[2]), (m, n)
        for b in bufs + outs:
            b.free()


def _check_products(dab, S, DS, x_host, rng, dtype):
    trip = so.canonical_triplets(S)
    cuts = DS.layout.cuts
    for trans in (False, True):
        xs = x_host[1] if trans else x_host[0]
        W = dab.transpose(DS) if trans else DS
        y = W @ xs
        want = so.mul_model(trip, S.shape, cuts, xs, trans)
        assert so.same_bits(dab.to_array(y), want), ("A'*x" if trans else "A*x", np.dtype(dtype))
        # x as a DVector in another layout: its blocks are halo-fetched
        y2 = (dab.adjoint(DS) if trans else DS) @ dab.distribute(xs, procs=[3, 1, 4], dist=[3])
        assert so.same_bits(dab.to_array(y2), want)
        assert list(y2.layout.pids) == list(y.layout.pids) and y2.layout.grid == y.layout.grid
        # mul!(y, A, x, α, β) on an existing dense y
        y0 = _values(rng, dtype, len(want), special=False)
        Y = dab.distribute(y0, procs=list(y.layout.pids), dist=[len(y.layout.pids)])
        dab.mul_(Y, W, xs, 3, 2)
        assert so.same_bits(dab.to_array(Y), so.mul_model(trip, S.shape, cuts, xs, trans, 3, 2, y0))
        dab.mul_(Y, W, xs, 1, 1)
        assert so.same_bits(dab.to_array(Y), so.mul_model(trip, S.shape, cuts, xs, trans, 1, 1, so.mul_model(trip, S.shape, cuts, xs, trans, 3, 2, y0)))


@pytest.mark.parametrize("grid", [(2, 4), (4, 2), (8, 1), (1, 8), None])
@pytest.mark.parametrize("dtype", DTYPES)
def test_products_on_8_workers(dab, rt8, dtype, grid):
    """A*x, A'*x, transpose(A)*x and mul! on 8-worker grids with uneven cuts: empty rows and columns, a chunk with no stored entry,
    explicit zeros, ±0, NaN and ±Inf in the matrix and in x, Int32 / Int64 overflow -- bit for bit against the model."""
    rng = np.random.default_rng(211)
    m, n = 203, 157
    S = _sparse(rng, dtype, m, n, 0.12, zero_block=((0, 110), (0, 90)), empty_rows=(5, 150, 202), empty_cols=(0, 77, 156))
    DS = dab.distribute(S, dist=grid)
    assert isinstance(DS, dab.SparseDArray)
    if grid in ((2, 4), (4, 2)):
        assert min(DS.chunk_nnz) == 0                             # the zero block covers a whole chunk
    x_host = (_values(rng, dtype, n), _values(rng, dtype, m))
    _check_products(dab, S, DS, x_host, rng, dtype)


def test_distribute_layout_nnz_and_to_array(dab, rt8):
    """The layout is dense distribute's; chunks are A[I...] with stored zeros kept; nnz counts stored entries; Array(S) densifies."""
    rng = np.random.default_rng(5)
    S = _sparse(rng, np.float64, 61, 47, 0.2)
    S.data[:5] = 0.0
    for grid in (None, (2, 4), (8, 1)):
        DS = dab.distribute(S, dist=grid)
        D = dab.distribute(S.toarray(), dist=grid)
        assert DS.layout.indices == D.layout.indices and list(DS.layout.pids) == list(D.layout.pids)
        assert dab.nnz(DS) == S.nnz and DS.dims == S.shape
        assert so.same_bits(dab.to_array(DS), _dense(S))
        for pid, ch in DS.chunks.items():
            (r0, r1), (c0, c1) = DS.layout.localindices(pid)
            shape, colptr, rowval, nzval = dab.localpart(DS, pid).to_host()
            sub = S[r0 - 1:r1, c0 - 1:c1].tocsc()
            assert shape == sub.shape and np.array_equal(colptr, sub.indptr) and np.array_equal(rowval, sub.indices)
            assert so.same_bits(nzval, sub.data)
    # `like` takes the layout of another DArray
    DS2 = dab.distribute(S, like=dab.distribute(S.toarray(), dist=(1, 8)))
    assert DS2.layout.grid == (1, 8)


def test_reference_nnz_testset(dab, rt8):
    """test/darray.jl:990-993: nnz(distribute(sprandn(10, 10, 0.5))) == nnz(A)."""
    A = sp.random(10, 10, density=0.5, random_state=np.random.default_rng(3), data_rvs=np.random.default_rng(4).standard_normal)
    assert dab.nnz(dab.distribute(A)) == A.nnz


def test_reference_matrix_multiplication_testset(dab, rt8):
    """test/darray.jl:916-929 with a sparse A: A*b and A'*b within sqrt(eps) of the dense products."""
    rng = np.random.default_rng(17)
    A = sp.random(20, 20, density=0.3, random_state=rng, data_rvs=rng.standard_normal, format="csc")
    b = rng.standard_normal(20)
    DA, Db = dab.distribute(A), dab.distribute(b)
    assert np.abs(dab.to_array(DA @ Db) - A.toarray() @ b).max() < np.sqrt(np.finfo(np.float64).eps)
    assert np.abs(dab.to_array(DA.T @ Db) - A.toarray().T @ b).max() < np.sqrt(np.finfo(np.float64).eps)
    DA.close()
    Db.close()


def test_copyto_from_host_sparse(dab, rt8):
    rng = np.random.default_rng(23)
    S = _sparse(rng, np.float32, 40, 30, 0.3)
    D = dab.dzeros((40, 30), dtype=np.float32)
    dab.copyto(D, S)
    assert so.same_bits(dab.to_array(D), _dense(S))


def test_deferred_affine_is_flushed_before_the_product(dab, rt1):
    """y .= a.*x .+ b may be held back by the library; the product that reads y must see it."""
    rng = np.random.default_rng(29)
    S = _sparse(rng, np.float64, 300, 400, 0.05)
    DS = dab.distribute(S)
    x = dab.distribute(rng.standard_normal(400))
    y = dab.similar(x)
    dab.broadcast_into(y, lambda v: 1.5 * v + 0.25, x)
    got = dab.to_array(DS @ y)
    yh = np.float64(1.5) * dab.to_array(x) + np.float64(0.25)
    assert so.same_bits(got, so.mul_model(so.canonical_triplets(S), S.shape, DS.layout.cuts, yh, False))


def test_row_major_copy_is_built_once(dab, rt8):
    """The first A*x builds the row-major copy of every chunk (K19); a second A*x reuses it and launches no K19 kernel; A'*x never
    needs it."""
    rng = np.random.default_rng(31)
    S = _sparse(rng, np.float64, 120, 90, 0.1)
    DS = dab.distribute(S)
    x, xt = rng.standard_normal(90), rng.standard_normal(120)
    l0 = rt8.launches()
    DS.T @ xt
    assert not any(ch.csr_built for ch in DS.chunks.values())
    l1 = rt8.launches()
    y1 = DS @ x
    l2 = rt8.launches()
    assert all(ch.csr_built for ch in DS.chunks.values())
    ptrs = [ch.csr()[0].ptr for ch in DS.chunks.values()]
    y2 = DS @ x
    l3 = rt8.launches()
    assert [ch.csr()[0].ptr for ch in DS.chunks.values()] == ptrs
    assert l3 - l2 == len(DS.chunks) + y1.layout.grid[0] < l2 - l1  # one K18 per tile and one fold per y chunk: no K19 kernel
    assert so.same_bits(dab.to_array(y1), dab.to_array(y2))


def test_close_and_finalizer_release_csc_and_csr(dab, rt8):
    rng = np.random.default_rng(37)
    S = _sparse(rng, np.float32, 80, 60, 0.1)
    n0 = dab.registry_size()
    DS = dab.distribute(S)
    DS @ rng.standard_normal(60).astype(np.float32)
    chunks = list(DS.chunks.values())
    arrays = [a for ch in chunks for a in (ch.colptr, ch.rowval, ch.nzval) + ch.csr()]
    assert dab.registry_size() == n0 + 1 and all(a.ptr for a in arrays)
    DS.close()
    assert all(a.ptr == 0 for a in arrays) and dab.registry_size() == n0 and not DS.chunks
    DS2 = dab.distribute(S)
    DS2 @ rng.standard_normal(60).astype(np.float32)
    arrays = [a for ch in DS2.chunks.values() for a in (ch.colptr, ch.rowval, ch.nzval) + ch.csr()]
    del DS2
    gc.collect()
    assert all(a.ptr == 0 for a in arrays) and dab.registry_size() == n0


def test_refusals_launch_nothing(dab, rt8):
    """Every operation other than the served ones raises UnsupportedError naming what is served, and launches and registers nothing."""
    import operator
    rng = np.random.default_rng(41)
    S = _sparse(rng, np.float64, 30, 20, 0.2)
    DS = dab.distribute(S)
    D = dab.distribute(rng.standard_normal((30, 20)))
    v20, v30 = dab.distribute(rng.standard_normal(20)), dab.distribute(rng.standard_normal(30))
    ops = {
        "broadcast": lambda: dab.broadcast(lambda a: a + 1, DS),
        "broadcast_into": lambda: dab.broadcast_into(D, lambda a: a * 2, DS),
        "broadcast into S": lambda: dab.broadcast_into(DS, lambda a: a * 2, D),
        "map": lambda: dab.map_(lambda a: a * 2, DS),
        "map!": lambda: dab.map_inplace(lambda a: a * 2, DS, DS),
        "sum": lambda: dab.sum(DS),
        "sum dims": lambda: dab.sum(DS, dims=1),
        "maximum": lambda: dab.maximum(DS),
        "mapreduce": lambda: dab.mapreduce(abs, "+", DS),
        "count": lambda: dab.count(DS, lambda a: a > 0),
        "norm": lambda: dab.norm(DS),
        "getindex": lambda: DS[3, 4],
        "view": lambda: DS[1:5, 2:7],
        "similar": lambda: dab.similar(DS),
        "sort": lambda: dab.sort(DS),
        "cumsum": lambda: dab.cumsum(DS, dims=1),
        "mapslices": lambda: dab.mapslices(dab.sum, DS, dims=1),
        "ppeval": lambda: dab.ppeval(operator.matmul, DS, D),
        "==": lambda: DS == D,
        "isequal": lambda: dab.isequal(DS, D),
        "copy(transpose)": lambda: dab.transpose(DS).copy(),
        "SpMM": lambda: DS @ D,
        "SpMM host": lambda: DS @ rng.standard_normal((20, 3)),
        "S'*B": lambda: DS.T @ D,
        "dense * sparse": lambda: D.T @ DS,
        "mul! into S": lambda: dab.mul_(DS, D, v20),
        "operator +": lambda: DS + D,
        "np.asarray": lambda: np.asarray(DS),
        "copyto! into S": lambda: dab.copyto(DS, S),
        "complex": lambda: dab.distribute(sp.random(5, 5, density=0.5, format="csc").astype(np.complex128)),
        "bool": lambda: dab.distribute(sp.random(5, 5, density=0.5, format="csc").astype(np.bool_)),
        "uint8": lambda: dab.distribute(sp.random(5, 5, density=0.5, format="csc").astype(np.uint8)),
    }
    if hasattr(sp, "coo_array"):
        try:
            vec = sp.coo_array(np.array([1.0, 0.0, 2.0]))
        except Exception:
            vec = None
        if vec is not None and len(vec.shape) == 1:
            ops["sparse vector"] = lambda: dab.distribute(vec)
    rt8.sync()
    for name, f in ops.items():
        l0, r0 = rt8.launches(), dab.registry_size()
        with pytest.raises(dab.UnsupportedError) as e:
            f()
        assert rt8.launches() == l0 and dab.registry_size() == r0, name
        if name not in ("complex", "bool", "uint8", "sparse vector"):
            assert "serves distribute, nnz" in str(e.value), (name, str(e.value))
    # the served products keep the dense error contract
    with pytest.raises(dab.DimensionMismatch):
        DS @ np.zeros(21)
    with pytest.raises(dab.UnsupportedError):
        dab.distribute(S.astype(np.int32)) @ np.zeros(20)     # an Int32 matrix with a Float64 vector needs a converted copy of A
    assert so.same_bits(dab.to_array(DS @ v20), so.mul_model(so.canonical_triplets(S), S.shape, DS.layout.cuts, dab.to_array(v20), False))
    assert so.same_bits(dab.to_array(DS.T @ v30), so.mul_model(so.canonical_triplets(S), S.shape, DS.layout.cuts, dab.to_array(v30), True))
