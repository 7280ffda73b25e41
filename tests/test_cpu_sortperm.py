"""CPU tier of ``sortperm`` (row f11): the host flow of _sort.py through the host-memory emulation of the C ABI (with
tests/sortperm_hostmem.py) against the model, the GPU module run against that emulation, and the no-spill compile of the pair
instances of dab_sort.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import sortperm_hostmem
from oracle import darray_oracle as orc

sortperm_hostmem.install()                                      # dab_sort_pairs for the host-memory emulation of the C ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _data(T, n, rng):
    if np.dtype(T).kind == "i":
        return rng.integers(-40, 40, n).astype(T)               # ties everywhere
    a = np.round(rng.standard_normal(n), 1).astype(T)
    if n > 20:
        a[rng.integers(0, n, n // 10)] = np.nan
        a[rng.integers(0, n, n // 10)] = -0.0
    return a


def _check(dab, d, a, sample, by=None, keys=None):
    p = dab.sortperm(d, sample=sample, by=by)
    k = a if keys is None else keys
    got = dab.to_array(p)
    assert p.dtype == np.int64 and np.array_equal(got, orc.jl_sortperm_stable(k) + 1)
    ref_d = d if keys is None else dab.distribute(keys, procs=list(d.layout.pids), dist=list(d.layout.grid))
    s, _ = dab.sort_with_boundaries(ref_d, sample=sample)
    nan = np.isnan(dab.to_array(s)) if k.dtype.kind == "f" else np.zeros(len(s), dtype=bool)
    if not nan.any() or nan[np.argmax(nan):].all():         # sort's result is in isless order (NaNs last): the same layout
        assert list(p.layout.pids) == list(s.layout.pids) and list(p.layout.indices) == list(s.layout.indices)
    s.close()
    if ref_d is not d:
        ref_d.close()
    p.close()


@pytest.mark.parametrize("T", [np.float64, np.float32, np.int64, np.int32])
@pytest.mark.parametrize("nw", [1, 2, 3, 5, 8])
def test_host_sortperm_flow(hostmem, dab, T, nw):
    """_sort.py's sortperm end to end on the host-memory ABI: values equal the stable isless permutation + 1 and the layout equals
    sort's, for every kind of `sample`, with and without `by`; no device block outlives the call."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(31 + nw)
    for n in (nw, 97, 3000):
        a = _data(T, n, rng)
        d = dab.distribute(a)
        fin = a[~np.isnan(a)] if a.dtype.kind == "f" else a
        lohi = (T(-40), T(40)) if np.dtype(T).kind == "i" else (T(-2), T(2))
        for sample in (True, False, lohi, _data(T, 64, rng)):
            if sample is False and len(fin) < len(a):
                continue                                        # minimum / maximum of NaN data are NaN: no uniform sample
            _check(dab, d, a, sample)
        _check(dab, d, a, True, by=abs, keys=np.abs(a))
        d.close()
    dab.sortperm(dab.distribute(_data(T, 500, rng))).close()    # warm the emulation's pools, then count
    n0 = len(hostmem.blocks)
    d = dab.distribute(_data(T, 500, rng))
    for by in (None, abs):
        dab.sortperm(d, by=by).close()
    d.close()
    assert len(hostmem.blocks) == n0
    assert hostmem.launches > 0
    rt.shutdown()


def test_host_sortperm_errors(hostmem, dab):
    """The errors of sort for the same arguments, raised before any launch, leaving no DArray and no device block behind."""
    rt = dab.init(workers_per_rank=4, use_dist=False)
    rng = np.random.default_rng(5)
    v = dab.distribute(rng.standard_normal(100))
    M = dab.distribute(rng.standard_normal((8, 8)))
    B = dab.distribute(rng.standard_normal(10) > 0)
    Z = dab.distribute(rng.standard_normal(10).astype(np.complex64))
    E = dab.distribute(np.zeros(0), procs=[1])
    n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
    for exc, f in [(dab.ArgumentError, lambda: dab.sortperm(v, rev=True)),
                   (dab.ArgumentError, lambda: dab.sortperm(v, sample="yes")),
                   (dab.ArgumentError, lambda: dab.sortperm(v, sample=(0.0, np.inf), by=abs)),
                   (dab.DimensionMismatch, lambda: dab.sortperm(M)),
                   (dab.UnsupportedError, lambda: dab.sortperm(B)),
                   (TypeError, lambda: dab.sortperm(Z)),
                   (dab.ArgumentError, lambda: dab.sortperm(E, sample=False))]:
        with pytest.raises(exc):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), exc
    rt.shutdown()


def test_more_than_256_workers_is_refused_before_any_launch(hostmem, dab):
    from darray_b200.layout import make_layout
    rt = dab.init(workers_per_rank=1, use_dist=False)
    d = dab.distribute(np.arange(300.0), procs=[1])
    lay = make_layout((300,), list(range(1, 258)), [257])
    d.layout = lay                                              # only the layout is looked at before the refusal
    l0 = hostmem.launches
    with pytest.raises(dab.UnsupportedError):
        dab.sortperm(d)
    assert hostmem.launches == l0
    rt.shutdown()


def test_gpu_sortperm_module_against_the_host_memory_abi():
    """tests/test_gpu_sortperm.py with the C ABI emulated over host memory: the host flow around K21 (samplesort steps, index plane
    exchange, layouts, refusals, launch and registry contracts) against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_sortperm.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 30, tail


def test_pair_instances_compile_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_sort.cu for sm_90a: every pair instance (payload uint32_t) uses no stack frame and spills nothing."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_sort.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) >= len(entries), r.stderr[-2000:]
    blocks = [(e, *f) for e, f in zip(entries, frames)]
    # the payload parameter follows the key type in the mangled name: I<key>j... is a pair instance (j = unsigned int)
    pairs = [(e, f) for e, *f in blocks if re.search(r"(sort_hist_kernel|sort_onesweep_kernel|sort_small_kernel)I[fdil]j", e)
             or re.search(r"sort_copy_if_kernelI[jm]j", e)]
    assert len(pairs) == 4 * 3 + 2, [e for e, _ in pairs]          # hist, onesweep, small per key type; copy_if per key width
    assert all(f == ["0", "0", "0"] for _, f in pairs), [e for e, f in pairs if f != ["0", "0", "0"]]
