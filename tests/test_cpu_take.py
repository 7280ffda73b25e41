"""CPU tier of ``d[I::DArray]`` (row f12): the host flow of _take.py through the host-memory emulation of the C ABI (with
tests/take_hostmem.py) against the NumPy model of Julia's ``A[I]``, the refusals, the GPU module run against that emulation, and the
no-spill compile of dab_take.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import take_hostmem

take_hostmem.install()                                          # dab_index_gather for the host-memory emulation of the C ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128]


def model(a, I):
    """Julia's ``A[I]`` for 1-based linear indices ``I``: the column-major ravel of ``A`` read at ``I - 1``, in ``I``'s shape."""
    return np.asarray(a).ravel(order="F")[np.asarray(I) - 1].reshape(np.shape(I), order="F")


def _values(T, shape, rng):
    T = np.dtype(T)
    n = int(np.prod(shape))
    if T == np.bool_:
        a = rng.random(n) > 0.5
    elif T.kind == "i":
        a = rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T)
    elif T.kind == "c":
        a = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(T)
    else:
        a = rng.standard_normal(n).astype(T)
        a[::7] = -0.0
    return a.reshape(shape, order="F")


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def _layouts(dab, shape, nw):
    """(procs, dist) choices: the default, and the first dim cut nw ways."""
    out = [dict()]
    if 1 < nw <= shape[0]:
        out.append(dict(procs=list(range(1, nw + 1)), dist=[nw] + [1] * (len(shape) - 1)))
    return out


@pytest.mark.parametrize("nw", [1, 3, 8])
@pytest.mark.parametrize("dshape,ishape", [((50,), (37,)), ((6, 7), (40,)), ((4, 5, 3), (6, 5)), ((30,), (3, 2, 4)), ((9, 4), (5, 3, 2))])
def test_host_take_flow(hostmem, dab, nw, dshape, ishape):
    """1-, 2- and 3-d sources and indices, regular layouts of d and I on 1, 3 and 8 workers, Int32 and Int64 indices with duplicates:
    every element equals the model bit for bit, and the result's layout is similar(d, size(I))'s."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(len(dshape) * 10 + nw)
    a = _values(np.float64, dshape, rng)
    for dl in _layouts(dab, dshape, nw):
        d = dab.distribute(a, **dl)
        for IT in (np.int32, np.int64):
            Ih = rng.integers(1, a.size + 1, ishape).astype(IT)
            Ih.ravel()[:2] = [1, a.size]
            for il in _layouts(dab, ishape, nw):
                I = dab.distribute(Ih, **il)
                R = d[I]
                _same(dab.to_array(R), model(a, Ih))
                S = dab.similar(d, dims=I.dims)
                assert R.layout.pids == S.layout.pids and R.layout.cuts == S.layout.cuts and R.layout.indices == S.layout.indices
                for x in (R, S, I):
                    x.close()
        d.close()
    rt.shutdown()


@pytest.mark.parametrize("T", ELTYPES)
def test_host_take_every_element_type(hostmem, dab, T):
    """All seven element types (1-, 4-, 8- and 16-byte moves), NaN payloads and -0.0 kept, on 8 workers."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    rng = np.random.default_rng(3)
    a = _values(T, (13, 11), rng)
    if np.dtype(T).kind == "f":
        U = np.uint32 if np.dtype(T).itemsize == 4 else np.uint64
        a.ravel(order="F")[5] = np.array([0x7FC00123 if U is np.uint32 else 0x7FF8000000000123], dtype=U).view(T)[0]
    d = dab.distribute(a)
    Ih = rng.integers(1, a.size + 1, (57,)).astype(np.int64)
    Ih[3] = 6
    R = d[dab.distribute(Ih)]
    assert R.dtype == np.dtype(T)
    _same(dab.to_array(R), model(a, Ih))
    rt.shutdown()


def test_host_take_irregular_and_empty_chunks(hostmem, dab):
    """Irregular layouts of d and I (chunks of unequal size, one of them empty), and 7 elements over 8 workers (an empty chunk at the
    end), with I laid out differently from R."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    rng = np.random.default_rng(11)
    parts = [rng.standard_normal(k) for k in (5, 0, 17, 1, 9)]
    a = np.concatenate(parts)
    d = dab.darray_from_chunks(parts, (5,))
    for ipart in ([3, 30], [0, 12, 21]):
        Ih = rng.integers(1, a.size + 1, sum(ipart)).astype(np.int64)
        pieces, o = [], 0
        for k in ipart:
            pieces.append(Ih[o:o + k])
            o += k
        I = dab.darray_from_chunks(pieces, (len(ipart),))
        assert not I.layout.same_as(dab.similar(d, dims=I.dims).layout)
        _same(dab.to_array(d[I]), model(a, Ih))
    a7 = rng.standard_normal(7)
    d7 = dab.darray_from_chunks([a7[:3], a7[3:3], a7[3:4], a7[4:5], a7[5:6], a7[6:7], a7[7:], a7[7:]], (8,))
    assert sum(r[0][1] < r[0][0] for r in d7.indices) == 3
    Ih = np.array([7, 1, 7, 3, 2, 6, 5, 4, 4], dtype=np.int32)
    _same(dab.to_array(d7[dab.darray_from_chunks([Ih[:2], Ih[2:2], Ih[2:]], (3,))]), model(a7, Ih))
    _same(dab.to_array(d7[dab.distribute(Ih[:5], procs=[2, 3])]), model(a7, Ih[:5]))
    rt.shutdown()


def test_host_take_empty(hostmem, dab):
    """An empty I gives an empty result of I's dims with no launch; an empty d with a non-empty I raises BoundsError before any launch."""
    rt = dab.init(workers_per_rank=3, use_dist=False)
    d = dab.distribute(np.arange(10.0))
    for shape in ((0,), (3, 0)):
        I = dab.distribute(np.zeros(shape, dtype=np.int64), procs=[1])
        l0 = hostmem.launches
        R = d[I]
        assert R.dims == shape and R.dtype == d.dtype and hostmem.launches == l0
    E = dab.distribute(np.zeros(0), procs=[1])
    I = dab.distribute(np.array([4, 1], dtype=np.int64))
    n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
    with pytest.raises(IndexError, match=r"BoundsError.*\[4\]"):
        E[I]
    assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0)
    rt.shutdown()


@pytest.mark.parametrize("nw", [1, 8])
def test_host_take_bounds_errors(hostmem, dab, nw):
    """An index of 0, length + 1, a negative one, and a bad index only in a late chunk: IndexError naming the value of the first bad
    index in column-major order of I; no DArray and no device block outlives the call, and the next call succeeds."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(2)
    a = rng.standard_normal((10, 10))
    d = dab.distribute(a)
    good = rng.integers(1, 101, 200).astype(np.int64)
    d[dab.distribute(good)].close()                              # warm the emulation's pools, then count
    for bad_at, bad_vals in [(0, [0]), (17, [101]), (5, [-3]), (190, [0]), (150, [102, 0])]:
        Ih = good.copy()
        for j, v in enumerate(bad_vals):
            Ih[bad_at + 20 * j] = v
        I = dab.distribute(Ih)
        n0, r0 = len(hostmem.blocks), dab.registry_size()
        with pytest.raises(IndexError, match=rf"BoundsError: .* at index \[{bad_vals[0]}\]"):
            d[I]
        assert (len(hostmem.blocks), dab.registry_size()) == (n0, r0)
        I32 = dab.distribute(Ih.astype(np.int32))
        with pytest.raises(IndexError, match=rf"\[{bad_vals[0]}\]"):
            d[I32]
        I.close()
        I32.close()
    _same(dab.to_array(d[dab.distribute(good)]), model(a, good))
    rt.shutdown()


def test_host_take_refusals(hostmem, dab):
    """Bool, float and complex index DArrays, and sparse sources or indices, are refused before any allocation or launch; the
    existing refusals of a DArray mixed with other indices and of a SubDArray stay as they were."""
    import scipy.sparse as sp
    rt = dab.init(workers_per_rank=4, use_dist=False)
    d = dab.distribute(np.arange(16.0).reshape(4, 4))
    S = dab.distribute(sp.random(8, 8, density=0.3, format="csc", random_state=1))
    p = dab.distribute(np.array([1, 2, 3], dtype=np.int64))
    keys = [dab.distribute(np.array([True, False])), dab.distribute(np.array([1.0, 2.0])), dab.distribute(np.array([1.0, 2.0], dtype=np.float32)),
            dab.distribute(np.array([1 + 0j]))]
    cases = [(dab.UnsupportedError, lambda: d[keys[0]]),
             (dab.ArgumentError, lambda: d[keys[1]]),
             (dab.ArgumentError, lambda: d[keys[2]]),
             (dab.ArgumentError, lambda: d[keys[3]]),
             (dab.UnsupportedError, lambda: S[p]),
             (dab.UnsupportedError, lambda: d[S]),
             (dab.UnsupportedError, lambda: d[p, :]),
             (IndexError, lambda: d[0:2, 0:2][p])]
    for exc, f in cases:
        n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
        with pytest.raises(exc):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), exc
    rt.shutdown()


def test_host_take_1024_chunks_over_8_dims(hostmem, dab):
    """A source of 1024 chunks cut along its first of 8 dims (1039 cuts, the largest table a 1024-chunk layout gives) is served."""
    rt = dab.init(workers_per_rank=1024, use_dist=False)
    rng = np.random.default_rng(1024)
    a = rng.standard_normal((1024, 1, 1, 1, 1, 1, 1, 2))
    d = dab.distribute(a, dist=[1024, 1, 1, 1, 1, 1, 1, 1])
    assert d.layout.grid == (1024,) + (1,) * 7
    Ih = rng.integers(1, a.size + 1, (300, 2)).astype(np.int64)
    _same(dab.to_array(d[dab.distribute(Ih, procs=[1])]), model(a, Ih))
    rt.shutdown()


def test_host_take_failed_launch_leaves_nothing(hostmem, dab, monkeypatch):
    """A launch that fails part-way (the third chunk's, here by a stand-in status) raises the library's error and frees the result,
    the index blocks and the bad-position slots."""
    import hostmem_abi
    rt = dab.init(workers_per_rank=4, use_dist=False)
    d = dab.distribute(np.arange(40.0))
    I = dab.distribute(np.arange(1, 41, dtype=np.int64), procs=[4, 3, 2, 1])
    d[I].close()
    real, calls = hostmem_abi.HostMemABI.dab_index_gather, []

    def failing(self, *args):
        calls.append(1)
        return 1 if len(calls) == 3 else real(self, *args)                                      # DAB_ERR_CUDA

    monkeypatch.setattr(hostmem_abi.HostMemABI, "dab_index_gather", failing)
    n0, r0 = len(hostmem.blocks), dab.registry_size()
    with pytest.raises(dab.DabError):
        d[I]
    assert (len(hostmem.blocks), dab.registry_size()) == (n0, r0)
    rt.shutdown()


def test_host_take_refuses_too_many_chunks_before_any_launch(hostmem, dab):
    from darray_b200.layout import make_layout
    rt = dab.init(workers_per_rank=1, use_dist=False)
    d = dab.distribute(np.arange(2000.0), procs=[1])
    d.layout = make_layout((2000,), list(range(1, 1027)), [1026])  # only the layout is looked at before the refusal
    I = dab.distribute(np.array([1], dtype=np.int64))
    n0, l0 = len(hostmem.blocks), hostmem.launches
    with pytest.raises(dab.UnsupportedError, match="1024"):
        d[I]
    assert (len(hostmem.blocks), hostmem.launches) == (n0, l0)
    rt.shutdown()


def test_gpu_take_module_against_the_host_memory_abi():
    """tests/test_gpu_take.py with the C ABI emulated over host memory: the host flow around K22 (source tables, index blocks, layouts,
    bounds and refusal contracts) against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_take.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 20, tail


def test_take_instances_compile_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_take.cu for sm_90a: all 32 instances (4 element sizes x 2 index types x 1-D / N-d x vector / scalar
    index loads) use no stack frame and spill nothing."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_take.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 32 and all("take_kernel" in e for e in entries), entries
    assert len(frames) == len(entries) and all(f == ("0", "0", "0") for f in frames), list(zip(entries, frames))
