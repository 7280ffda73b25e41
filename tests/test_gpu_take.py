"""GPU tests of ``d[I::DArray]`` (row f12): K22 (``dab_index_gather``) through the C ABI on every dispatch path against a byte-exact
model, the distributed flow against Julia's ``A[I]``, its compositions with ``sortperm`` and ``findmax(A; dims)``, and the bounds
contract.  The kernel only moves bytes: every result must equal the model exactly."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets K22, K20 and K21 too
    import findmax_oracle
    import sortperm_hostmem
    import take_hostmem
    take_hostmem.install()
    sortperm_hostmem.install()
    findmax_oracle.install()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (0, 1, 3, 4, 5, 1023, (1 << 20) + 3)
UNITS = {1: np.bool_, 4: np.float32, 8: np.int64, 16: np.complex128}   # carriers of 1-, 4-, 8- and 16-byte elements
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


def model(a, I):
    """Julia's ``A[I]`` for 1-based linear indices ``I``."""
    return np.asarray(a).ravel(order="F")[np.asarray(I) - 1].reshape(np.shape(I), order="F")


def _bits(es, n, rng):
    """n elements of random bit patterns (NaNs with payloads, -0.0, denormals included) in the carrier of ``es`` bytes."""
    if es == 1:
        return rng.integers(0, 2, n).astype(np.bool_)
    return rng.integers(0, 256, n * es, dtype=np.uint8).view(UNITS[es])


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def _cut(dim, g, rng, empty=False):
    """0-based cuts of ``dim`` into ``g`` pieces of random sizes (``empty``: at least one empty piece when g > 1)."""
    inner = np.sort(rng.integers(0, dim + 1, g - 1)) if g > 1 else np.zeros(0, dtype=np.int64)
    if empty and g > 1:
        inner[len(inner) // 2] = inner[len(inner) // 2 - 1] if len(inner) > 1 else 0
    return [0] + [int(x) for x in inner] + [dim]


def _gather(dab, rt, A, cuts, I, idx_off=0, out_off=0):
    """``dab_index_gather`` of the column-major host array ``A`` chunked by ``cuts`` (0-based, per dim) at the 1-based linear indices
    ``I`` (Int32 / Int64), the index block ``idx_off`` and the output ``out_off`` elements into their allocations.  Returns the output
    (elements at bad positions keep a sentinel fill), the bad position, and the launch count."""
    from darray_b200 import _lib
    grid = [len(c) - 1 for c in cuts]
    chunks, ptrs = [], []
    for lin in range(int(np.prod(grid))):
        g = np.unravel_index(lin, grid, order="F")
        blk = A[tuple(slice(cuts[k][g[k]], cuts[k][g[k] + 1]) for k in range(A.ndim))]
        if blk.size:
            ch = dab.B200Array.from_numpy(rt, np.asfortranarray(blk))
            chunks.append(ch)
            ptrs.append(ch.ptr)
        else:
            ptrs.append(None)
    n = I.size
    ib = dab.B200Array.from_numpy(rt, np.concatenate([np.zeros(idx_off, dtype=I.dtype), I.ravel(order="F")]))
    fill = _bits(A.dtype.itemsize, n + out_off, np.random.default_rng(0)).astype(A.dtype)
    ob = dab.B200Array.from_numpy(rt, fill)
    bad = dab.B200Array.from_numpy(rt, np.full(1, -1, dtype=np.int64))
    flat = [x for c in cuts for x in c]
    l0 = rt.launches()
    _lib.call("dab_index_gather", rt.ctx, A.dtype.itemsize, C.c_void_p(ob.ptr + out_off * A.dtype.itemsize),
              C.c_void_p(ib.ptr + idx_off * I.dtype.itemsize), dab.dab_dtype(I.dtype), n, A.ndim, (C.c_size_t * A.ndim)(*A.shape),
              (C.c_int32 * A.ndim)(*grid), (C.c_size_t * len(flat))(*flat), (C.c_void_p * len(ptrs))(*ptrs), C.c_void_p(bad.ptr))
    launched = rt.launches() - l0
    out = ob.to_numpy()
    assert np.array_equal(out[:out_off].view(np.uint8), fill[:out_off].view(np.uint8))     # nothing written before the block
    b = bad.to_numpy().view(np.uint64)[0]
    for x in chunks + [ib, ob, bad]:
        x.free()
    return out[out_off:], fill[out_off:], b, launched


def _expect(A, I, got, fill, bad):
    g = np.asarray(I, dtype=np.int64).ravel(order="F") - 1
    ok = (g >= 0) & (g < A.size)
    want = fill.copy()
    want[ok] = A.ravel(order="F")[g[ok]]
    _same(got, want)
    assert bad == (NONE if ok.all() else np.uint64(np.argmin(ok)))


@pytest.mark.parametrize("es", [1, 4, 8, 16])
@pytest.mark.parametrize("IT", [np.int32, np.int64])
@pytest.mark.parametrize("n", SIZES)
def test_kernel_1d(dab, rt1, es, IT, n):
    """1-D source of 4 chunks (one empty): every element size, both index types, aligned (16-byte index loads) and unaligned index
    blocks and outputs, with duplicates; no launch for n == 0."""
    rng = np.random.default_rng(n * 7 + es)
    A = _bits(es, 5000, rng)
    cuts = [[0, 1200, 1200, 4100, 5000]]
    I = rng.integers(1, A.size + 1, n).astype(IT)
    for idx_off, out_off in ((0, 0), (1, 0), (0, 1), (3, 5)):
        got, fill, bad, launched = _gather(dab, rt1, A, cuts, I, idx_off, out_off)
        _expect(A, I, got, fill, bad)
        assert launched == (1 if n else 0)


@pytest.mark.parametrize("es", [1, 4, 8, 16])
@pytest.mark.parametrize("IT", [np.int32, np.int64])
@pytest.mark.parametrize("shape,grid", [((37, 29), (3, 2)), ((6, 5, 7), (2, 1, 3)), ((3, 2, 2, 3, 2, 2, 2, 3), (2, 1, 1, 2, 1, 1, 1, 2))])
def test_kernel_nd(dab, rt1, es, IT, shape, grid):
    """N-d sources (2-, 3- and 8-d) with irregular cuts and empty chunks: linear indices split into coordinates, each chunk found by the
    cut search, aligned and unaligned index blocks."""
    rng = np.random.default_rng(len(shape) * 31 + es)
    A = _bits(es, int(np.prod(shape)), rng).reshape(shape, order="F")
    cuts = [_cut(s, g, rng, empty=(k == len(shape) - 1)) for k, (s, g) in enumerate(zip(shape, grid))]
    for n in (2, 5, 1023, 4099):
        I = rng.integers(1, A.size + 1, n).astype(IT)
        I[:2] = [1, A.size]
        for idx_off in (0, 1):
            got, fill, bad, _ = _gather(dab, rt1, A, cuts, I, idx_off, idx_off)
            _expect(A, I, got, fill, bad)


@pytest.mark.parametrize("IT", [np.int32, np.int64])
def test_kernel_bounds(dab, rt1, IT):
    """Out-of-range indices (0, length + 1, negative, the type's extremes) store nothing there; *bad_pos is the first bad position."""
    rng = np.random.default_rng(9)
    A = _bits(8, 12 * 10, rng).reshape(12, 10, order="F")
    cuts = [[0, 5, 12], [0, 3, 3, 10]]
    info = np.iinfo(IT)
    for n, bads in [(8, {0: 0}), (5000, {4999: A.size + 1}), (5000, {3000: -1, 4000: 0}), (4100, {2049: info.min, 2050: info.max}),
                    (3, {1: A.size + 1, 2: 0})]:
        for src, src_cuts in ((A, cuts), (A.ravel(order="F"), [[0, 50, 120]])):
            I = rng.integers(1, A.size + 1, n).astype(IT)
            for p, v in bads.items():
                I[p] = v
            for idx_off in (0, 1):
                got, fill, bad, _ = _gather(dab, rt1, src, src_cuts, I, idx_off)
                _expect(src, I, got, fill, bad)


def test_kernel_refusals(dab, rt1):
    """Unserved element sizes and index types, more than 8 dims or 1024 chunks, bad cuts and a NULL non-empty chunk: status codes,
    nothing launched."""
    from darray_b200 import _lib
    a = dab.B200Array.from_numpy(rt1, np.arange(8.0))
    ix = dab.B200Array.from_numpy(rt1, np.arange(1, 9, dtype=np.int64))
    out = dab.B200Array.empty(rt1, (8,), np.float64)
    bad = dab.B200Array.from_numpy(rt1, np.full(1, -1, dtype=np.int64))

    def call(es=8, it=_lib.I64, nd=1, dims=(8,), grid=(1,), cuts=(0, 8), ptrs=None):
        ptrs = ptrs if ptrs is not None else [a.ptr] * int(np.prod(grid))
        return _lib.lib().dab_index_gather(rt1.ctx, es, C.c_void_p(out.ptr), C.c_void_p(ix.ptr), it, 8, nd, (C.c_size_t * len(dims))(*dims),
                                           (C.c_int32 * len(grid))(*grid), (C.c_size_t * len(cuts))(*cuts), (C.c_void_p * len(ptrs))(*ptrs),
                                           C.c_void_p(bad.ptr))
    l0 = rt1.launches()
    assert call(es=2) == _lib.ERR_ARG
    assert call(it=_lib.F64) == _lib.ERR_ARG
    assert call(nd=9, dims=(1,) * 8 + (8,), grid=(1,) * 9, cuts=(0, 1) * 8 + (0, 8)) == _lib.ERR_UNSUPPORTED
    assert call(grid=(1025,), cuts=(0,) * 1025 + (8,)) == _lib.ERR_UNSUPPORTED
    assert call(cuts=(0, 7)) == _lib.ERR_ARG
    assert call(grid=(2,), cuts=(0, 9, 8)) == _lib.ERR_ARG
    assert call(grid=(2,), cuts=(0, 4, 8), ptrs=[a.ptr, None]) == _lib.ERR_ARG
    assert rt1.launches() == l0
    assert call() == _lib.OK and rt1.launches() == l0 + 1
    _same(out.to_numpy(), np.arange(8.0))


@pytest.mark.parametrize("IT", [np.int32, np.int64])
@pytest.mark.parametrize("shape", [(1024, 1, 1, 1, 1, 1), (1024, 1, 1, 1, 1, 1, 1, 2)])
def test_kernel_largest_cut_table(dab, rt1, IT, shape):
    """The most cuts a table of at most 1024 chunks can have: grid (1024, 1, ...) over 6 and 8 dims gives 1035 and 1039 cuts, more than
    chunks + dims.  Every element equals the model, and the first bad position is still reported."""
    rng = np.random.default_rng(len(shape))
    A = _bits(8, int(np.prod(shape)), rng).reshape(shape, order="F")
    cuts = [list(range(1025))] + [[0, s] for s in shape[1:]]
    assert sum(len(c) for c in cuts) == 1024 + 2 * len(shape) - 1
    I = rng.integers(1, A.size + 1, 5000).astype(IT)
    I[:2] = [1, A.size]
    got, fill, bad, launched = _gather(dab, rt1, A, cuts, I)
    _expect(A, I, got, fill, bad)
    assert launched == 1
    I[4000] = A.size + 1
    got, fill, bad, _ = _gather(dab, rt1, A, cuts, I, 1, 1)
    _expect(A, I, got, fill, bad)


@pytest.mark.skipif(HOSTMEM, reason="a 2^26-element gather is a device-memory case")
def test_kernel_2_pow_26(dab, rt1):
    """One 2^26-element gather with Int64 indices from a 2^26-element Float64 source in one chunk (a random permutation)."""
    n = 1 << 26
    rng = np.random.default_rng(26)
    A = rng.standard_normal(n)
    I = (rng.permutation(n) + 1).astype(np.int64)
    got, fill, bad, _ = _gather(dab, rt1, A, [[0, n]], I)
    assert bad == NONE
    _same(got, A[I - 1])


# ---- the distributed flow ----------------------------------------------------------------------------------------------------------


def test_sortperm_composition(dab, rt8):
    """v[sortperm(v)] equals sort(v) bit for bit (Float64 with NaNs and -0.0, Int64), with sample true and false."""
    rng = np.random.default_rng(1)
    n = 100003
    for T in (np.float64, np.int64):
        if T == np.float64:
            a = np.round(rng.standard_normal(n), 2)
            a[rng.integers(0, n, n // 20)] = -0.0
            a[rng.integers(0, n, n // 20)] = 0.0
            nan = a.copy()
            nan[rng.integers(0, n, n // 30)] = np.nan
            cases = [(a, False), (nan, True)]           # sample=false needs finite min / max
        else:
            a = rng.integers(-500, 500, n).astype(T)
            cases = [(a, False), (a, True)]
        for h, sample in cases:
            v = dab.distribute(h)
            w = v[dab.sortperm(v, sample=sample)]
            got = dab.to_array(w)
            _same(got, h[orc.jl_sortperm_stable(h)])
            s = dab.to_array(dab.sort(v, sample=sample))
            nanm = np.isnan(s) if s.dtype.kind == "f" else np.zeros(n, dtype=bool)
            if not nanm.any() or nanm[np.argmax(nanm):].all():   # sort itself in isless order (see sortperm's docstring)
                _same(got, s)


def test_sortperm_of_other_vector(dab, rt8):
    """y[sortperm(x)] == y_h[argsort(x_h, stable)] for y of every element type, x and y in different layouts."""
    rng = np.random.default_rng(4)
    n = 50001
    xh = rng.integers(-100, 100, n).astype(np.float32)
    x = dab.distribute(xh)
    p = dab.sortperm(x)
    for T in (np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128):
        yh = _bits(np.dtype(T).itemsize, n, rng)
        yh = yh if T == np.bool_ else yh.view(T)
        y = dab.distribute(yh, procs=[2, 5, 7], dist=[3])
        _same(dab.to_array(y[p]), yh[np.argsort(xh, kind="stable")])


@pytest.mark.parametrize("shape", [(300, 47), (40, 30, 7)])
@pytest.mark.parametrize("k", [1, 2])
def test_findmax_composition(dab, rt8, shape, k):
    """A[findmax(A; dims=k)[2]] (the index DArray, N-d linear indices into an N-d source) equals maximum(A; dims=k) bit for bit."""
    rng = np.random.default_rng(sum(shape) + k)
    A = dab.distribute(rng.standard_normal(shape).astype(np.float32))
    vals, idx = dab.findmax(A, dims=k)
    R = A[idx]
    assert R.dims == idx.dims and R.dtype == np.float32
    _same(dab.to_array(R), dab.to_array(dab.maximum(A, dims=k)))
    _same(dab.to_array(R), dab.to_array(vals))


def test_new_path_against_the_host_path(dab, rt8):
    """For a 1-D d, d[p] equals the existing host route d[np.asarray(p) - 1]."""
    rng = np.random.default_rng(8)
    d = dab.distribute(rng.standard_normal(20011))
    p = dab.distribute(rng.integers(1, 20012, 7001))
    _same(dab.to_array(d[p]), np.asarray(d[np.asarray(p) - 1]))


@pytest.mark.parametrize("T", [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128])
def test_every_element_type(dab, rt8, T):
    """Random I with duplicates (Int32 and Int64) for every element type, on a 2-d source; complex NaN payloads compared byte for byte."""
    rng = np.random.default_rng(np.dtype(T).itemsize)
    es = np.dtype(T).itemsize
    h = _bits(es, 97 * 61, rng)
    h = (h if T == np.bool_ else h.view(T)).reshape(97, 61, order="F")
    d = dab.distribute(h)
    for IT in (np.int32, np.int64):
        Ih = rng.integers(1, 20, (3000,)).astype(IT) * rng.integers(1, 300, 3000).astype(IT)
        Ih = np.minimum(Ih, h.size).astype(IT)
        for dist in ([8], [4]):
            I = dab.distribute(Ih, procs=list(range(1, 9)), dist=dist)
            _same(dab.to_array(d[I]), model(h, Ih))


def test_irregular_index_layout(dab, rt8):
    """I in an irregular layout (an empty chunk, uneven sizes, other workers) unlike d's and R's, 2-d I into a 3-d d."""
    rng = np.random.default_rng(12)
    h = rng.standard_normal((20, 9, 11))
    d = dab.distribute(h, procs=[3, 1, 4, 8], dist=[1, 1, 4])
    Ih = rng.integers(1, h.size + 1, (60, 7)).astype(np.int64)
    parts = [Ih[:13], Ih[13:13], Ih[13:60]]
    I = dab.darray_from_chunks(parts, (3, 1), pids=[6, 2, 7])
    R = d[I]
    S = dab.similar(d, dims=I.dims)
    assert R.layout.pids == S.layout.pids and R.layout.indices == S.layout.indices
    _same(dab.to_array(R), model(h, Ih))


@pytest.mark.parametrize("n", SIZES)
def test_sizes(dab, rt8, n):
    """n in {0, 1, 3, 4, 5, 1023, 2^20 + 3}: results of I's dims and d's type, empty without a launch."""
    rng = np.random.default_rng(n)
    h = rng.standard_normal(4099)
    d = dab.distribute(h)
    Ih = rng.integers(1, h.size + 1, n).astype(np.int64)
    I = dab.distribute(Ih, procs=[1]) if n == 0 else dab.distribute(Ih)
    l0 = rt8.launches()
    R = d[I]
    if n == 0:
        assert rt8.launches() == l0
    assert R.dims == (n,)
    _same(dab.to_array(R), model(h, Ih))


@pytest.mark.skipif(HOSTMEM, reason="a 2^26-element gather is a device-memory case")
def test_2_pow_26_on_8_workers(dab, rt8):
    n = 1 << 26
    rng = np.random.default_rng(3)
    h = rng.standard_normal(n).astype(np.float32)
    d = dab.distribute(h)
    Ih = (rng.permutation(n) + 1).astype(np.int64)
    _same(dab.to_array(d[dab.distribute(Ih)]), h[Ih - 1])


def test_bounds_error_leaves_nothing(dab, rt8):
    """Each BoundsError names the first bad value in column-major order of I, leaves nothing registered, and the next call on the same
    runtime succeeds."""
    rng = np.random.default_rng(6)
    h = rng.standard_normal((30, 20))
    d = dab.distribute(h)
    good = rng.integers(1, h.size + 1, 5000).astype(np.int64)
    for pos, v in [(0, 0), (2500, h.size + 1), (17, -5), (4999, 0)]:
        Ih = good.copy()
        Ih[pos] = v
        I = dab.distribute(Ih)
        r0 = dab.registry_size()
        with pytest.raises(IndexError, match=rf"BoundsError: .* at index \[{v}\]"):
            d[I]
        assert dab.registry_size() == r0
        I.close()
        _same(dab.to_array(d[dab.distribute(good)]), model(h, good))


def test_multi_gpu():
    """tools/multi_gpu_take.py under torchrun on two GPUs: d split across ranks, I in a different layout, v[sortperm(v)] across ranks,
    and the same BoundsError on every rank."""
    import torch
    if HOSTMEM or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.join(ROOT, "tools", "multi_gpu_take.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "multi-gpu take passed" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
