"""GPU tests of ``d[key] = v`` (row f14): K24 (``dab_scatter_check`` / ``dab_scatter_winners`` / ``dab_scatter``) and K25 (``dab_expand``)
through the C ABI against a byte-exact sequential model, and the distributed flow of every key form and value form against NumPy models of
Julia's ``setindex!`` (0-based host keys; 1-based column-major DArray keys; last occurrence wins), its identities with ``sortperm``,
``findall`` and ``getindex``, aliasing, and the error contracts.  Every result must equal the model exactly."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets K24, K25 and what their flow shares
    import setindex_hostmem
    import sortperm_hostmem
    setindex_hostmem.install()
    sortperm_hostmem.install()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (0, 1, 3, 4, 5, 1023, (1 << 20) + 3)
UNITS = {1: np.bool_, 4: np.float32, 8: np.int64, 16: np.complex128}
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128]
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


def _bits(T, n, rng):
    """n elements of random bit patterns of type T (NaNs with payloads, -0.0, denormals included)."""
    T = np.dtype(T)
    if T == np.bool_:
        return rng.integers(0, 2, n).astype(np.bool_)
    return rng.integers(0, 256, n * T.itemsize, dtype=np.uint8).view(T)


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def model_take(a, I, v):
    """Julia's sequential ``A[I] = v`` (1-based linear ``I``; scalar or array ``v``): the last occurrence of a position wins."""
    out = np.asarray(a).copy()
    flat = out.reshape(-1, order="F")
    g = np.asarray(I, dtype=np.int64).reshape(-1, order="F") - 1
    vals = np.broadcast_to(np.asarray(v, dtype=a.dtype), g.shape) if np.ndim(v) == 0 else np.asarray(v).astype(a.dtype).reshape(-1, order="F")
    _, last_rev = np.unique(g[::-1], return_index=True)
    last = g.size - 1 - last_rev
    flat[g[last]] = vals[last]
    return flat.reshape(a.shape, order="F")


def model_mask(a, m, v):
    out = np.asarray(a).copy()
    flat = out.reshape(-1, order="F")
    sel = np.asarray(m).reshape(-1, order="F")
    flat[sel] = np.asarray(v, dtype=a.dtype) if np.ndim(v) == 0 else np.asarray(v).astype(a.dtype).reshape(-1, order="F")
    return flat.reshape(a.shape, order="F")


def model_view(a, key, v):
    """Julia's ``view(A, key...) .= v`` with 0-based host keys, written element by element in column-major order of the key."""
    out = np.asarray(a).copy()
    key = key if isinstance(key, tuple) else (key,)
    iv = []
    for k, s in zip(key, a.shape):
        if isinstance(k, slice):
            iv.append(np.arange(*k.indices(s)))
        elif isinstance(k, (int, np.integer)):
            iv.append(np.array([int(k) % s]))
        else:
            iv.append(np.asarray(k, dtype=np.int64) % s)
    full = tuple(len(x) for x in iv)
    vals = np.broadcast_to(np.asarray(v, dtype=a.dtype), full) if np.ndim(v) == 0 else np.asarray(v).astype(a.dtype).reshape(full, order="F")
    g = np.ravel_multi_index(np.ix_(*iv), a.shape, order="F")
    g = np.broadcast_to(g, full).reshape(-1, order="F")
    flat = out.reshape(-1, order="F")
    _, last_rev = np.unique(g[::-1], return_index=True)
    last = g.size - 1 - last_rev
    flat[g[last]] = vals.reshape(-1, order="F")[last]
    return flat.reshape(a.shape, order="F")


# ---- K24 at the C ABI ------------------------------------------------------------------------------------------------------------------


def _cut(dim, g, rng, empty=False):
    inner = np.sort(rng.integers(0, dim + 1, g - 1)) if g > 1 else np.zeros(0, dtype=np.int64)
    if empty and g > 1:
        inner[len(inner) // 2] = inner[len(inner) // 2 - 1] if len(inner) > 1 else 0
    return [0] + [int(x) for x in inner] + [dim]


def _scatter(dab, rt, A, cuts, I, V, idx_off=0):
    """The host sequence of K24 on the column-major host array ``A`` chunked by ``cuts``: check, then (with duplicates) winners, then the
    stores of ``V`` (an array of I's length, or a 0-d scalar) at the 1-based indices ``I`` (one block, one run), the index block
    ``idx_off`` elements into its allocation.  Returns the result, the bad position, the duplicates flag and the launch count."""
    from darray_b200 import _lib
    grid = [len(c) - 1 for c in cuts]
    chunks, ptrs, bms, bptrs, wins, wptrs = [], [], [], [], [], []
    n = I.size
    wb = 4
    for lin in range(int(np.prod(grid))):
        g = np.unravel_index(lin, grid, order="F")
        blk = A[tuple(slice(cuts[k][g[k]], cuts[k][g[k] + 1]) for k in range(A.ndim))]
        if blk.size:
            ch = dab.B200Array.from_numpy(rt, np.asfortranarray(blk))
            bm = dab.B200Array.from_numpy(rt, np.zeros(-(-blk.size // 32), dtype=np.int32))
            wn = dab.B200Array.from_numpy(rt, np.zeros(blk.size, dtype=np.int32))
            chunks.append(ch), bms.append(bm), wins.append(wn)
            ptrs.append(ch.ptr), bptrs.append(bm.ptr), wptrs.append(wn.ptr)
        else:
            ptrs.append(None), bptrs.append(None), wptrs.append(None)
    ib = dab.B200Array.from_numpy(rt, np.concatenate([np.zeros(idx_off, dtype=I.dtype), I.ravel(order="F")]))
    scalar = np.ndim(V) == 0
    vb = None if scalar else dab.B200Array.from_numpy(rt, np.asarray(V).ravel(order="F"))
    sv = np.asarray(V, dtype=A.dtype).reshape(1) if scalar else None
    st = dab.B200Array.from_numpy(rt, np.array([-1, 0], dtype=np.int64))
    lin = dab.B200Array.from_numpy(rt, np.zeros(1, dtype=np.int64))
    flat = [x for c in cuts for x in c]
    tab = ((C.c_size_t * A.ndim)(*A.shape), (C.c_int32 * A.ndim)(*grid), (C.c_size_t * len(flat))(*flat))
    VP = C.c_void_p * len(ptrs)
    idx = C.c_void_p(ib.ptr + idx_off * I.dtype.itemsize)
    code = dab.dab_dtype(I.dtype)
    l0 = rt.launches()
    _lib.call("dab_scatter_check", rt.ctx, idx, code, n, A.ndim, *tab, VP(*bptrs), C.c_void_p(st.ptr))
    bad, dup = st.to_numpy().view(np.uint64)
    if bad == NONE:
        if dup:
            _lib.call("dab_scatter_winners", rt.ctx, idx, code, n, max(n, 1), C.c_void_p(lin.ptr), wb, A.ndim, *tab, VP(*wptrs))
        _lib.call("dab_scatter", rt.ctx, A.dtype.itemsize, idx, code, n, None if scalar else C.c_void_p(vb.ptr),
                  C.c_void_p(sv.ctypes.data) if scalar else None, max(n, 1), C.c_void_p(lin.ptr), wb if dup else 0, A.ndim, *tab, VP(*ptrs),
                  VP(*wptrs) if dup else None)
    launched = rt.launches() - l0
    out = A.copy(order="F")
    it = iter(chunks)
    for li in range(int(np.prod(grid))):
        g = np.unravel_index(li, grid, order="F")
        sl = tuple(slice(cuts[k][g[k]], cuts[k][g[k] + 1]) for k in range(A.ndim))
        if out[sl].size:
            out[sl] = next(it).to_numpy().reshape(out[sl].shape)
    for x in chunks + bms + wins + [ib, st, lin] + ([vb] if vb is not None else []):
        x.free()
    return out, bad, bool(dup), launched


@pytest.mark.parametrize("es", [1, 4, 8, 16])
@pytest.mark.parametrize("IT", [np.int32, np.int64])
@pytest.mark.parametrize("shape,grid", [((5000,), (4,)), ((37, 29), (3, 2)), ((6, 5, 7), (2, 1, 3)),
                                        ((3, 2, 2, 3, 2, 2, 2, 3), (2, 1, 1, 2, 1, 1, 1, 2))])
def test_kernel_scatter(dab, rt1, es, IT, shape, grid):
    """1-, 2-, 3- and 8-d destinations with irregular cuts and empty chunks, every element size, both index types, aligned and unaligned
    index blocks: unique indices (a permutation), heavy duplicates (random with many repeats, all equal) and a scalar, each against the
    sequential last-wins model; the same call twice gives the same bytes."""
    rng = np.random.default_rng(len(shape) * 31 + es)
    T = UNITS[es]
    A = _bits(T, int(np.prod(shape)), rng).reshape(shape, order="F")
    cuts = [_cut(s, g, rng, empty=(k == len(shape) - 1)) for k, (s, g) in enumerate(zip(shape, grid))]
    perm = (rng.permutation(A.size)[:min(A.size, 3001)] + 1).astype(IT)
    cases = [(perm, False), (rng.integers(1, 60, 4099).astype(IT), True), (np.full(777, A.size, dtype=IT), True), (perm[:5], False)]
    for I, dup in cases:
        for idx_off in (0, 1):
            V = _bits(T, I.size, rng)
            got, bad, flagged, launched = _scatter(dab, rt1, A, cuts, I, V, idx_off)
            assert bad == NONE and flagged == dup and launched == (3 if dup else 2)
            _same(got, model_take(A, I, V))
            again, _, _, _ = _scatter(dab, rt1, A, cuts, I, V, idx_off)
            _same(again, got)
    x = _bits(T, 1, rng)[0]
    got, _, _, _ = _scatter(dab, rt1, A, cuts, cases[1][0], np.asarray(x))
    _same(got, model_take(A, cases[1][0], x))


@pytest.mark.parametrize("IT", [np.int32, np.int64])
def test_kernel_scatter_bounds(dab, rt1, IT):
    """0, length + 1, negative and the type's extremes: the first bad position is reported by the check pass, which writes nothing."""
    rng = np.random.default_rng(9)
    A = _bits(np.float64, 120, rng).reshape(12, 10, order="F")
    cuts = [[0, 5, 12], [0, 3, 3, 10]]
    info = np.iinfo(IT)
    for n, bads in [(8, {0: 0}), (5000, {4999: A.size + 1}), (5000, {3000: -1, 4000: 0}), (4100, {2049: info.min, 2050: info.max})]:
        I = rng.integers(1, A.size + 1, n).astype(IT)
        for p, v in bads.items():
            I[p] = v
        got, bad, _, launched = _scatter(dab, rt1, A, cuts, I, _bits(np.float64, n, rng))
        assert bad == np.uint64(min(bads)) and launched == 1
        _same(got, A)


def test_kernel_scatter_largest_cut_table(dab, rt1):
    """Grid (1024, 1, ..., 1) over 8 dims: 1039 cuts, with duplicates."""
    rng = np.random.default_rng(8)
    shape = (1024, 1, 1, 1, 1, 1, 1, 2)
    A = _bits(np.int64, 2048, rng).reshape(shape, order="F")
    cuts = [list(range(1025))] + [[0, s] for s in shape[1:]]
    I = rng.integers(1, A.size + 1, 5000).astype(np.int64)
    V = _bits(np.int64, I.size, rng)
    got, bad, dup, _ = _scatter(dab, rt1, A, cuts, I, V)
    assert bad == NONE and dup
    _same(got, model_take(A, I, V))


def test_kernel_refusals(dab, rt1):
    """Unserved element sizes, index types and winner widths, bad cuts, a NULL non-empty chunk: status codes, nothing launched."""
    from darray_b200 import _lib
    a = dab.B200Array.from_numpy(rt1, np.arange(8.0))
    ix = dab.B200Array.from_numpy(rt1, np.arange(1, 9, dtype=np.int64))
    L = _lib.lib()

    def call(es=8, it=_lib.I64, wb=0, cuts=(0, 8), ptrs=None):
        ptrs = ptrs if ptrs is not None else [a.ptr] * (len(cuts) - 1)
        g = len(cuts) - 1
        return L.dab_scatter(rt1.ctx, es, C.c_void_p(ix.ptr), it, 8, C.c_void_p(a.ptr), None, 8, None, wb, 1, (C.c_size_t * 1)(8),
                             (C.c_int32 * 1)(g), (C.c_size_t * len(cuts))(*cuts), (C.c_void_p * g)(*ptrs), None)
    l0 = rt1.launches()
    assert call(es=2) == _lib.ERR_ARG
    assert call(it=_lib.F64) == _lib.ERR_ARG
    assert call(wb=2) == _lib.ERR_ARG
    assert call(cuts=(0, 7)) == _lib.ERR_ARG
    assert call(cuts=(0, 4, 8), ptrs=[a.ptr, None]) == _lib.ERR_ARG
    assert L.dab_expand(rt1.ctx, 2, C.c_void_p(a.ptr), C.c_void_p(a.ptr), 8, 1, None, None, 1, None, None, C.c_void_p(a.ptr)) == _lib.ERR_ARG
    assert rt1.launches() == l0


# ---- the distributed flow --------------------------------------------------------------------------------------------------------------


def _values_of(dab, form, T, shape, rng, like=None):
    """A value of the given form holding _bits(T) in ``shape``: (value, its host array, or None for a scalar)."""
    h = _bits(T, int(np.prod(shape)), rng).reshape(shape, order="F")
    procs = dict(procs=[1]) if h.size == 0 else {}
    if form == "scalar":
        return _bits(T, 1, rng)[0], None
    if form == "host":
        return h, h
    if form == "same":
        return (dab.distribute(h, like=like) if like is not None and like.dims == tuple(shape) else dab.distribute(h, **procs)), h
    if form == "other":
        return dab.distribute(h, procs=[1] if h.size == 0 else [3, 1, 2]), h
    big = _bits(T, int(np.prod([s + 3 for s in shape])), rng).reshape([s + 3 for s in shape], order="F")   # a view of a larger DArray
    key = tuple(slice(2, 2 + s) for s in shape)
    return dab.distribute(big)[key], big[key]


def _want(model, a, key, v, h):
    return model(a, key, v if h is None else h)


@pytest.mark.parametrize("T", ELTYPES)
@pytest.mark.parametrize("form", ["scalar", "host", "same", "other", "view"])
def test_darray_key(dab, rt8, T, form):
    """d[I] = v with I a DArray of Int32 / Int64 (with duplicates, 2-d I into a 2-d d), every value form and element type."""
    rng = np.random.default_rng(np.dtype(T).itemsize * 7 + len(form))
    a = _bits(T, 97 * 61, rng).reshape(97, 61, order="F")
    for IT in (np.int32, np.int64):
        Ih = rng.integers(1, a.size + 1, (300, 7)).astype(IT)
        Ih[0, :3] = [5, 5, a.size]
        d = dab.distribute(a)
        I = dab.distribute(Ih, procs=list(range(1, 9)), dist=[4, 2])
        v, h = _values_of(dab, form, T, Ih.shape, rng, like=I)
        d[I] = v
        _same(dab.to_array(d), _want(model_take, a, Ih, v, h))


@pytest.mark.parametrize("T", ELTYPES)
@pytest.mark.parametrize("form", ["scalar", "host", "same", "other", "view"])
def test_mask_key(dab, rt8, T, form):
    """d[m] = v with a Bool mask in d's layout and in another one, densities 0, 0.5 and 1."""
    rng = np.random.default_rng(np.dtype(T).itemsize * 11 + len(form))
    a = _bits(T, 37 * 29, rng).reshape(37, 29, order="F")
    for density, mprocs in ((0.5, None), (0.0, [2, 4]), (1.0, [5, 6, 7])):
        mh = rng.random(a.shape) < density
        d = dab.distribute(a, procs=list(range(1, 7)), dist=[3, 2])
        m = dab.distribute(mh) if mprocs is None else dab.distribute(mh, procs=mprocs)
        v, h = _values_of(dab, form, T, (int(mh.sum()),), rng, like=None)
        d[m] = v
        _same(dab.to_array(d), _want(model_mask, a, mh, v, h))


KEYS = [(slice(2, 30), slice(None)), (slice(1, 36, 3), slice(28, 2, -5)), ([5, 1, 9, 5, 36], slice(3, 20)), (4, slice(None)),
        (slice(None), [0, 28, 0, 3]), (10, 11)]


@pytest.mark.parametrize("T", ELTYPES)
@pytest.mark.parametrize("form", ["scalar", "host", "same", "other", "view"])
def test_host_keys(dab, rt8, T, form):
    """d[key] = v for unit, strided and reversed ranges, int lists with repeats and ints, and the same through a view of d."""
    rng = np.random.default_rng(np.dtype(T).itemsize * 13 + len(form))
    a = _bits(T, 37 * 29, rng).reshape(37, 29, order="F")
    d = dab.distribute(a, procs=list(range(1, 7)), dist=[3, 2])
    want = a
    for key in KEYS:
        shape = np.zeros(a.shape)[key].shape
        if not shape and form != "scalar":
            continue                                              # d[i, j] = x: one element, a scalar value
        v, h = _values_of(dab, form, T, shape, rng)
        d[key] = v
        want = _want(model_view, want, key, v, h)
        _same(dab.to_array(d), want)
    s = d[1:36, 2:27]                                             # writes through a view reach the parent
    s[3:9, ::4] = 0 if T != np.bool_ else False
    want = model_view(want, (slice(4, 10), slice(2, 27, 4)), np.zeros((), T))
    _same(dab.to_array(d), want)
    h = _bits(T, 35, rng)
    dab.copyto(d[1:36, 5], h)
    want = model_view(want, (slice(1, 36), 5), h)
    _same(dab.to_array(d), want)


def test_value_conversion(dab, rt8):
    """A Float32 DArray value into a Float64 d goes through copyto's identity broadcast; a host Int value is converted with astype."""
    rng = np.random.default_rng(2)
    a = rng.standard_normal(1000)
    d = dab.distribute(a)
    I = (rng.permutation(1000)[:300] + 1).astype(np.int64)
    v = rng.standard_normal(300).astype(np.float32)
    d[dab.distribute(I)] = dab.distribute(v)
    want = model_take(a, I, v.astype(np.float64))
    _same(dab.to_array(d), want)
    d[0:10] = np.arange(10)
    want[0:10] = np.arange(10.0)
    _same(dab.to_array(d), want)


@pytest.mark.parametrize("n", SIZES)
def test_sizes(dab, rt8, n):
    """I of n in {0, 1, 3, 4, 5, 1023, 2^20 + 3} elements: an empty I launches nothing."""
    rng = np.random.default_rng(n)
    a = rng.standard_normal(1 << 20)
    d = dab.distribute(a)
    Ih = rng.integers(1, a.size + 1, n).astype(np.int64)
    I = dab.distribute(Ih, procs=[1]) if n == 0 else dab.distribute(Ih)
    v = rng.standard_normal(n)
    l0 = rt8.launches()
    d[I] = v
    if n == 0:
        assert rt8.launches() == l0
    _same(dab.to_array(d), model_take(a, Ih, v))


@pytest.mark.skipif(HOSTMEM, reason="a 2^26-element scatter is a device-memory case")
def test_2_pow_26(dab, rt8):
    n = 1 << 26
    rng = np.random.default_rng(26)
    d = dab.dzeros((n,), dtype=np.float32)
    Ih = (rng.permutation(n) + 1).astype(np.int64)
    v = rng.standard_normal(n).astype(np.float32)
    d[dab.distribute(Ih)] = dab.distribute(v)
    want = np.empty(n, np.float32)
    want[Ih - 1] = v
    _same(dab.to_array(d), want)


@pytest.mark.skipif(HOSTMEM, reason="a chunk of more than 2^31 elements is a device-memory case")
def test_mask_past_2_pow_31(dab, rt1):
    """One Bool chunk of 2^31 + 12293 elements: d[m] = v and d[m] = x reach selected positions beyond 2^31."""
    n = (1 << 31) + 3 * 4096 + 5
    pos = np.array([7, (1 << 31) - 1, 1 << 31, (1 << 31) + 4097, n - 1], dtype=np.int64)
    d = dab.dzeros((n,), dtype=np.bool_)
    m = dab.dzeros((n,), dtype=np.bool_)
    m[pos] = True
    d[m] = np.array([True, False, True, True, True])
    got = np.asarray(d[pos])
    _same(got, np.array([True, False, True, True, True]))
    d[m] = False
    _same(np.asarray(d[pos]), np.zeros(5, dtype=np.bool_))


def test_identities(dab, rt8):
    """w[sortperm(v)] = sort(v) reproduces v (sample true and false); d[findall(m)] = x equals d[m] = x; d[m] = d[m] and d[I] = d[I]
    leave d unchanged; d[I] += v is getindex-then-setindex."""
    import darray_b200
    rng = np.random.default_rng(5)
    h = np.round(rng.standard_normal(100003), 2)
    h[rng.integers(0, h.size, 5000)] = -0.0
    for sample in (False, True):
        v = dab.distribute(h)
        w = dab.similar(v)
        w[dab.sortperm(v, sample=sample)] = dab.sort(v, sample=sample)
        _same(dab.to_array(w), h)
    a = _bits(np.float64, 4000, rng).reshape(80, 50, order="F")
    mh = rng.random(a.shape) < 0.3
    d1, d2 = dab.distribute(a), dab.distribute(a)
    m = dab.distribute(mh, procs=[2, 3, 5])
    d1[darray_b200.findall(m)] = 7.5
    d2[m] = 7.5
    _same(dab.to_array(d1), dab.to_array(d2))
    d = dab.distribute(a)
    d[m] = d[m]
    I = dab.distribute(rng.integers(1, a.size + 1, 3000).astype(np.int64))
    d[I] = d[I]
    _same(dab.to_array(d), a)
    Ih = rng.integers(1, a.size + 1, 900).astype(np.int64)
    vh = rng.standard_normal(900)
    d = dab.distribute(a)
    I, v = dab.distribute(Ih), dab.distribute(vh)
    d[I] += v
    _same(dab.to_array(d), model_take(a, Ih, a.reshape(-1, order="F")[Ih - 1] + vh))


def test_aliasing(dab, rt8):
    """d[p] = d, d[d_as_index] = v and overlapping view copies give the sequential model's result (the value is copied first)."""
    rng = np.random.default_rng(6)
    h = rng.standard_normal(5000)
    d = dab.distribute(h)
    p = rng.permutation(5000) + 1
    d[dab.distribute(p)] = d
    want = model_take(h, p, h)
    _same(dab.to_array(d), want)
    ih = rng.integers(1, 3001, 3000).astype(np.int64)
    di = dab.distribute(ih)
    di[di] = np.arange(3000, dtype=np.int64)
    _same(dab.to_array(di), model_take(ih, ih, np.arange(3000, dtype=np.int64)))
    A = rng.standard_normal((40, 30))
    D = dab.distribute(A)
    D[0:5, :] = D[5:10, :]
    D[3:20, 2:9] = D[0:17, 0:7]
    W = A.copy()
    W[0:5, :] = W[5:10, :].copy()
    W[3:20, 2:9] = W[0:17, 0:7].copy()
    _same(dab.to_array(D), W)


def test_errors(dab, rt8):
    """Refusals and shape mismatches launch nothing; a BoundsError leaves d byte for byte unchanged with nothing registered, and the next
    call succeeds; a mask count mismatch raises DimensionMismatch before any store."""
    import scipy.sparse as sp
    rng = np.random.default_rng(7)
    a = rng.standard_normal((30, 20))
    d = dab.distribute(a)
    I = dab.distribute(rng.integers(1, 601, 50).astype(np.int64))
    S = dab.distribute(sp.random(8, 8, density=0.3, format="csc", random_state=1))
    cases = [(dab.UnsupportedError, lambda: d.__setitem__(dab.distribute(np.ones(7, dtype=np.bool_)), 1.0)),
             (dab.ArgumentError, lambda: d.__setitem__(dab.distribute(np.ones(3)), 1.0)),
             (dab.UnsupportedError, lambda: d.__setitem__(S, 1.0)),
             (dab.UnsupportedError, lambda: d.__setitem__((I, slice(None)), 1.0)),
             (dab.DimensionMismatch, lambda: d.__setitem__(I, np.zeros(49))),
             (dab.DimensionMismatch, lambda: d.__setitem__(I, dab.distribute(np.zeros((5, 10))))),
             (dab.DimensionMismatch, lambda: d.__setitem__((slice(0, 3), slice(0, 4)), np.zeros((4, 3)))),
             (dab.DimensionMismatch, lambda: dab.copyto(d[0:3, 0:4], np.zeros(12))),
             (dab.DimensionMismatch, lambda: d.__setitem__(dab.distribute(a > 0), np.zeros((3, 3)))),
             (IndexError, lambda: d.__setitem__((slice(0, 3), 25), 1.0))]
    for exc, f in cases:
        l0, r0 = rt8.launches(), dab.registry_size()
        with pytest.raises(exc):
            f()
        assert (rt8.launches(), dab.registry_size()) == (l0, r0), exc
    m = dab.distribute(a > 0)
    with pytest.raises(dab.DimensionMismatch):
        d[m] = np.zeros(int((a > 0).sum()) + 1)
    _same(dab.to_array(d), a)
    good = rng.integers(1, a.size + 1, 5000).astype(np.int64)
    for pos, v in [(0, 0), (2500, a.size + 1), (17, -5), (4999, 0)]:
        Ih = good.copy()
        Ih[pos] = v
        J = dab.distribute(Ih)
        r0 = dab.registry_size()
        with pytest.raises(IndexError, match=rf"BoundsError: .* at index \[{v}\]"):
            d[J] = 1.0
        assert dab.registry_size() == r0
        _same(dab.to_array(d), a)
        J.close()
    d[dab.distribute(good)] = 2.0
    _same(dab.to_array(d), model_take(a, good, 2.0))


def test_multi_gpu():
    """tools/multi_gpu_setindex.py under torchrun on two GPUs: d split across ranks, I and v in other layouts, duplicates across ranks,
    masks and views, and the same BoundsError on every rank."""
    import torch
    if HOSTMEM or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.join(ROOT, "tools", "multi_gpu_setindex.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "multi-gpu setindex passed" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
