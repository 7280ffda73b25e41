"""CPU tier of ``d[mask]``, ``findall`` and ``filter`` (row f13): the host flow of _compact.py through the host-memory emulation of the
C ABI (with tests/compact_hostmem.py) against the NumPy model of Julia's logical indexing, the refusals, the cleanup after a failed
launch, the GPU module run against that emulation, and the no-spill compile of dab_compact.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import compact_hostmem
import take_hostmem

compact_hostmem.install()                                       # K23 (and the K17 scans) for the host-memory emulation of the C ABI
take_hostmem.install()                                          # K22, for d[findall(m)]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128]


def model(a, m):
    """Julia's ``A[M]`` for a Bool array ``M`` of ``A``'s size: the true positions in column-major order."""
    return np.asarray(a).ravel(order="F")[np.asarray(m).ravel(order="F")]


def model_findall(m):
    return np.flatnonzero(np.asarray(m).ravel(order="F")).astype(np.int64) + 1


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def _mask(shape, density, rng):
    if density in (0, 1):
        return np.full(shape, bool(density))
    return rng.random(shape) < density


def _same_layout(R, S):
    assert R.layout.pids == S.layout.pids and R.layout.cuts == S.layout.cuts and R.layout.indices == S.layout.indices


# (shape, dist) pairs: the default layout, and grids that split dim 1 (the runs interleave chunks in the global order)
LAYOUTS = [((50,), None), ((37, 29), [3, 2]), ((6, 5, 7), [2, 1, 3]), ((9, 4), [1, 3]), ((4, 3, 5, 2), [2, 1, 2, 2])]


@pytest.mark.parametrize("nw", [1, 3, 8])
@pytest.mark.parametrize("shape,dist", LAYOUTS)
@pytest.mark.parametrize("density", [0, 1, 0.3])
def test_host_compact_flow(hostmem, dab, nw, shape, dist, density):
    """d[m] and findall(m) on 1, 3 and 8 workers, d and m in the same layout and in different ones: every element equals the model
    bit for bit, and the results have the layouts of similar(d, (count,)) and similar(m, Int64, (count,))."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(len(shape) * 10 + nw)
    a = rng.standard_normal(shape)
    a.ravel()[::5] = -0.0
    mh = _mask(shape, density, rng)
    lays = [dict()]
    if dist is not None and int(np.prod(dist)) <= nw:
        lays.append(dict(procs=list(range(1, int(np.prod(dist)) + 1)), dist=dist))
    for dl in lays:
        d = dab.distribute(a, **dl)
        for ml in lays:
            m = dab.distribute(mh, **ml)
            l0 = hostmem.launches
            R = d[m]
            _same(dab.to_array(R), model(a, mh))
            _same_layout(R, dab.similar(d, dims=R.dims))
            F = dab.findall(m)
            _same(dab.to_array(F), model_findall(mh))
            _same_layout(F, dab.similar(m, np.int64, F.dims))
            _same(dab.to_array(d[F]), model(a, mh))                       # d[findall(m)] == d[m] through K22
            assert hostmem.launches > l0
            for x in (R, F, m):
                x.close()
        d.close()
    rt.shutdown()


def test_host_compact_run_plan(dab):
    """The runs of (37, 29) on grid (3, 2) interleave the chunks: 3 * 29 runs, run (o, b) at global linear index 37 * o + cut_b; a
    DVector has one run per chunk and one chunk one run; 4096^2 on grid (2, 4) has 8192 runs."""
    from darray_b200._compact import run_plan
    from darray_b200.layout import make_layout
    lay = make_layout((37, 29), list(range(1, 7)), [3, 2])
    runs, n = run_plan(lay)
    assert n == 3 * 29
    starts = np.zeros(n, dtype=np.int64)
    for c, (run_len, ids, lin) in enumerate(runs):
        assert run_len == lay.indices[c][0][1] - lay.indices[c][0][0] + 1
        starts[ids] = lin
    assert np.all(np.diff(starts) > 0) and starts[0] == 0
    assert run_plan(make_layout((100,), [1, 2, 3], [3]))[1] == 3
    assert run_plan(make_layout((10, 10), [1], [1, 1]))[1] == 1
    assert run_plan(make_layout((4096, 4096), list(range(1, 9)), [2, 4]))[1] == 8192


@pytest.mark.parametrize("T", ELTYPES)
def test_host_compact_every_element_type(hostmem, dab, T):
    """All seven element types (1-, 4-, 8- and 16-byte moves), NaN payloads and -0.0 kept, on 8 workers; filter with a traced
    predicate returns a DVector for a 2-d d."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    rng = np.random.default_rng(3)
    es = np.dtype(T).itemsize
    a = (rng.random((13, 11)) < 0.5) if T == np.bool_ else rng.integers(0, 256, 13 * 11 * es, dtype=np.uint8).view(T).reshape(13, 11)
    mh = rng.random((13, 11)) < 0.4
    d = dab.distribute(a)
    R = d[dab.distribute(mh)]
    assert R.dtype == np.dtype(T) and R.dims == (int(mh.sum()),)
    _same(dab.to_array(R), model(a, mh))
    if T in (np.int32, np.int64):
        _same(dab.to_array(dab.filter(lambda x: x > 0, d)), model(a, a > 0))
        _same(dab.to_array(dab.findall(lambda x: x > 0, d)), model_findall(a > 0))
    rt.shutdown()


def test_host_compact_irregular_and_empty_chunks(hostmem, dab):
    """Irregular chunks (one of them empty), 7 elements over 8 workers, and a mask laid out differently from d."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    rng = np.random.default_rng(11)
    parts = [rng.standard_normal(k) for k in (5, 0, 17, 1, 9)]
    a = np.concatenate(parts)
    d = dab.darray_from_chunks(parts, (5,))
    for density in (0, 1, 0.5):
        mh = _mask(a.shape, density, rng)
        for m in (dab.distribute(mh), dab.darray_from_chunks([mh[:20], mh[20:20], mh[20:]], (3,))):
            _same(dab.to_array(d[m]), model(a, mh))
            _same(dab.to_array(dab.findall(m)), model_findall(mh))
    a7 = rng.standard_normal(7)
    d7 = dab.darray_from_chunks([a7[:3], a7[3:3], a7[3:4], a7[4:5], a7[5:6], a7[6:7], a7[7:], a7[7:]], (8,))
    m7 = np.array([True, False, True, True, False, True, True])
    _same(dab.to_array(d7[dab.distribute(m7)]), model(a7, m7))
    rt.shutdown()


def test_host_compact_1024_workers(hostmem, dab):
    """1024 workers: a 1024-chunk d split along dim 1 of 2 dims (2048 runs), and a 1024-chunk result table."""
    rt = dab.init(workers_per_rank=1024, use_dist=False)
    rng = np.random.default_rng(1024)
    a = rng.standard_normal((2048, 2))
    mh = rng.random(a.shape) < 0.6
    d = dab.distribute(a, dist=[1024, 1])
    assert d.layout.grid == (1024, 1)
    m = dab.distribute(mh)
    R = d[m]
    assert len(R.layout.pids) == 1024
    _same(dab.to_array(R), model(a, mh))
    _same(dab.to_array(dab.findall(m)), model_findall(mh))
    rt.shutdown()


def test_host_compact_empty(hostmem, dab):
    """An all-false mask and an empty d give empty DVectors without a compaction launch."""
    rt = dab.init(workers_per_rank=3, use_dist=False)
    d = dab.distribute(np.arange(12.0).reshape(3, 4))
    m = dab.distribute(np.zeros((3, 4), dtype=bool))
    calls = []
    real = compact_hostmem.dab_compact
    import hostmem_abi
    hostmem_abi.HostMemABI.dab_compact = lambda self, *a: calls.append(1) or real(self, *a)
    try:
        R, F = d[m], dab.findall(m)
        assert R.dims == (0,) and R.dtype == d.dtype and F.dims == (0,) and F.dtype == np.int64
        E = dab.distribute(np.zeros((0, 4)))
        l0 = hostmem.launches
        R0 = E[dab.distribute(np.zeros((0, 4), dtype=bool))]
        assert R0.dims == (0,) and hostmem.launches == l0
        assert calls == []
    finally:
        hostmem_abi.HostMemABI.dab_compact = real
    rt.shutdown()


def test_host_compact_refusals(hostmem, dab):
    """Sparse sources and masks, a Bool key of other dims (the existing refusal), a non-Bool findall and a non-Bool predicate, and
    key forms served before: refused exactly as before, before any allocation or launch."""
    import scipy.sparse as sp
    rt = dab.init(workers_per_rank=4, use_dist=False)
    d = dab.distribute(np.arange(16.0).reshape(4, 4))
    S = dab.distribute(sp.random(8, 8, density=0.3, format="csc", random_state=1))
    m16 = dab.distribute(np.ones((4, 4), dtype=bool))
    short = dab.distribute(np.array([True, False]))
    flat = dab.distribute(np.ones(16, dtype=bool))
    cases = [(dab.UnsupportedError, lambda: d[short]),
             (dab.UnsupportedError, lambda: d[flat]),
             (dab.UnsupportedError, lambda: S[m16]),
             (dab.UnsupportedError, lambda: d[S]),
             (dab.UnsupportedError, lambda: dab.findall(S)),
             (dab.UnsupportedError, lambda: dab.filter(lambda x: x > 0, S)),
             (TypeError, lambda: dab.findall(d)),
             (TypeError, lambda: dab.findall(lambda x: x + 1, d)),
             (TypeError, lambda: dab.filter(lambda x: x * 2, d)),
             (dab.UnsupportedError, lambda: d[m16, :]),
             (IndexError, lambda: d[0:2, 0:2][m16])]
    for exc, f in cases:
        n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
        with pytest.raises(exc):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), exc
    with pytest.raises(TypeError, match=r"non-boolean \(Float64\) used in boolean context"):
        dab.findall(d)
    with pytest.raises(TypeError, match=r"non-boolean \(Float64\) used in boolean context"):
        dab.filter(lambda x: x + 1, d)
    rt.shutdown()


@pytest.mark.parametrize("which", ["dab_compact_count", "dab_compact"])
def test_host_compact_failed_launch_leaves_nothing(hostmem, dab, monkeypatch, which):
    """A launch that fails part-way (the third chunk's, by a stand-in status) raises the library's error and frees the result, the
    mask blocks, the tile tables and the run tables."""
    import hostmem_abi
    rt = dab.init(workers_per_rank=4, use_dist=False)
    rng = np.random.default_rng(5)
    d = dab.distribute(rng.standard_normal((40, 6)), dist=[4, 1])
    m = dab.distribute(rng.random((40, 6)) < 0.5, procs=[4, 3, 2, 1])
    d[m].close()
    real, calls = getattr(hostmem_abi.HostMemABI, which), []

    def failing(self, *args):
        calls.append(1)
        return 1 if len(calls) == 3 else real(self, *args)                                      # DAB_ERR_CUDA

    monkeypatch.setattr(hostmem_abi.HostMemABI, which, failing)
    n0, r0 = len(hostmem.blocks), dab.registry_size()
    with pytest.raises(dab.DabError):
        d[m]
    assert (len(hostmem.blocks), dab.registry_size()) == (n0, r0)
    rt.shutdown()


def test_gpu_compact_module_against_the_host_memory_abi():
    """tests/test_gpu_compact.py with the C ABI emulated over host memory: the host flow around K23 (run plans, tile tables, mask halo
    reads, destination tables, refusal contracts) against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_compact.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 20, tail


def test_compact_instances_compile_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_compact.cu for sm_90a: all 6 instances (the count kernel, and the compaction of 1-, 4-, 8- and
    16-byte elements and of indices) use no stack frame and spill nothing."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_compact.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 6 and all("compact" in e for e in entries), entries
    assert len(frames) == len(entries) and all(f == ("0", "0", "0") for f in frames), list(zip(entries, frames))
