"""CPU tier of ``d[key] = v`` (row f14): the host flow of _setindex.py through the host-memory emulation of the C ABI (with
tests/setindex_hostmem.py) against NumPy models of Julia's sequential ``setindex!`` on 1, 3 and 8 workers, the refusals and the cleanup
after a failed launch, the GPU module run against that emulation, and the no-spill compile of dab_scatter.cu and dab_expand.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import setindex_hostmem

setindex_hostmem.install()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model_take(a, I, v):
    out = np.asarray(a).copy()
    flat = out.reshape(-1, order="F")
    g = np.asarray(I, dtype=np.int64).reshape(-1, order="F") - 1
    vals = np.broadcast_to(np.asarray(v, dtype=a.dtype), g.shape) if np.ndim(v) == 0 else np.asarray(v).astype(a.dtype).reshape(-1, order="F")
    for k in range(g.size):                                     # sequential, as Julia's setindex! runs
        flat[g[k]] = vals[k]
    return flat.reshape(a.shape, order="F")


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


@pytest.mark.parametrize("nw", [1, 3, 8])
@pytest.mark.parametrize("dshape,ishape", [((50,), (37,)), ((6, 7), (40,)), ((4, 5, 3), (6, 5)), ((30,), (3, 2, 4))])
def test_host_scatter_flow(hostmem, dab, nw, dshape, ishape):
    """d[I] = v for 1-, 2- and 3-d d and I, Int32 and Int64 indices with duplicates, values as a scalar, a host array and DArrays in
    I's layout and in another one, against the sequential model."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(len(dshape) * 10 + nw)
    a = rng.standard_normal(dshape)
    for IT in (np.int32, np.int64):
        Ih = rng.integers(1, a.size + 1, ishape).astype(IT)
        Ih.ravel()[:3] = [1, a.size, 1]
        vh = rng.standard_normal(ishape)
        for v in (2.5, vh, "same", "other"):
            d = dab.distribute(a)
            I = dab.distribute(Ih)
            val = dab.distribute(vh, like=I) if isinstance(v, str) and v == "same" else \
                dab.distribute(vh, procs=list(range(nw, 0, -1))) if isinstance(v, str) else v
            d[I] = val
            _same(dab.to_array(d), model_take(a, Ih, 2.5 if np.ndim(v) == 0 and not isinstance(v, str) else vh))
            for x in (d, I):
                x.close()
    rt.shutdown()


@pytest.mark.parametrize("nw", [1, 3, 8])
def test_host_mask_and_views(hostmem, dab, nw):
    """d[m] = v and d[m] = x with masks in d's layout and in another one, and host keys (ranges, steps, repeated list entries, ints)."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(nw)
    a = rng.standard_normal((9, 13))
    d = dab.distribute(a)
    want = a.copy()
    for procs in (None, [1]):
        mh = rng.random(a.shape) < 0.5
        m = dab.distribute(mh) if procs is None else dab.distribute(mh, procs=procs)
        vals = rng.standard_normal(int(mh.sum()))
        d[m] = dab.distribute(vals)
        f = want.reshape(-1, order="F")
        f[mh.reshape(-1, order="F")] = vals
        d[m] = -1.0
        f[mh.reshape(-1, order="F")] = -1.0
        want = f.reshape(a.shape, order="F")
        _same(dab.to_array(d), want)
    d[1:8:3, [4, 2, 4]] = np.arange(9.0).reshape(3, 3)
    want[1:8:3, [2, 4]] = np.arange(9.0).reshape(3, 3)[:, 1:]
    d[0, :] = 7.0
    want[0, :] = 7.0
    _same(dab.to_array(d), want)
    rt.shutdown()


def test_host_refusals_and_bounds(hostmem, dab):
    """Refusals launch nothing and allocate nothing; a BoundsError leaves d unchanged and frees every temporary."""
    import scipy.sparse as sp
    rt = dab.init(workers_per_rank=4, use_dist=False)
    a = np.arange(16.0).reshape(4, 4)
    d = dab.distribute(a)
    S = dab.distribute(sp.random(8, 8, density=0.3, format="csc", random_state=1))
    p = dab.distribute(np.array([1, 2, 3], dtype=np.int64))
    cases = [(dab.UnsupportedError, lambda: d.__setitem__(dab.distribute(np.array([True, False])), 1.0)),
             (dab.ArgumentError, lambda: d.__setitem__(dab.distribute(np.array([1.0, 2.0])), 1.0)),
             (dab.UnsupportedError, lambda: d.__setitem__(S, 1.0)),
             (dab.UnsupportedError, lambda: d.__setitem__((p, slice(None)), 1.0)),
             (dab.DimensionMismatch, lambda: d.__setitem__(p, np.zeros(4))),
             (dab.DimensionMismatch, lambda: d.__setitem__((slice(0, 2), slice(0, 3)), np.zeros((3, 2)))),
             (NotImplementedError, lambda: S.__setitem__((0, 0), 1.0))]
    for exc, f in cases:
        n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
        with pytest.raises(exc):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), exc
    d[p] = 0.0                                                   # warm the emulation's pools, then count
    a[0:3, 0] = 0.0                                              # linear indices 1:3, column-major
    B = dab.distribute(np.array([2, 17, 0], dtype=np.int64), procs=[1])
    n0, r0 = len(hostmem.blocks), dab.registry_size()
    with pytest.raises(IndexError, match=r"BoundsError: .* at index \[17\]"):
        d[B] = 5.0
    assert (len(hostmem.blocks), dab.registry_size()) == (n0, r0)
    _same(dab.to_array(d), a)
    rt.shutdown()


def test_host_failed_store_leaves_nothing(hostmem, dab, monkeypatch):
    """A store launch that fails part-way raises the library's error and frees the bitmaps, winner tables, value blocks and slots."""
    import hostmem_abi
    rt = dab.init(workers_per_rank=4, use_dist=False)
    d = dab.distribute(np.arange(40.0))
    I = dab.distribute(np.array([3, 3] + list(range(1, 39)), dtype=np.int64), procs=[4, 3, 2, 1])
    v = np.arange(40.0)
    d[I] = v
    real, calls = hostmem_abi.HostMemABI.dab_scatter, []

    def failing(self, *args):
        calls.append(1)
        return 1 if len(calls) == 3 else real(self, *args)                                      # DAB_ERR_CUDA

    monkeypatch.setattr(hostmem_abi.HostMemABI, "dab_scatter", failing)
    n0, r0 = len(hostmem.blocks), dab.registry_size()
    with pytest.raises(dab.DabError):
        d[I] = v
    assert (len(hostmem.blocks), dab.registry_size()) == (n0, r0)
    rt.shutdown()


def test_gpu_setindex_module_against_the_host_memory_abi():
    """tests/test_gpu_setindex.py with the C ABI emulated over host memory: the host flow around K24 and K25 against the same models."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_setindex.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 100, tail


def _ptxas(src):
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", src), "-o", os.devnull],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(entries) and all(f == ("0", "0", "0") for f in frames), list(zip(entries, frames))
    return entries


def test_scatter_and_expand_compile_without_stack_or_spills():
    """``nvcc -Xptxas -v`` for sm_90a: the 28 instances of dab_scatter.cu (check 2 x 2, winners 2 x 2 x 2, stores 4 x 2 x 2) and the 8 of
    dab_expand.cu (values and scalar, 1-, 4-, 8- and 16-byte elements) use no stack frame and spill nothing."""
    assert len(_ptxas("dab_scatter.cu")) == 28
    entries = _ptxas("dab_expand.cu")
    assert len(entries) == 8 and all("expand" in e for e in entries), entries
