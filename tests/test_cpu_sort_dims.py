"""CPU tier of ``sort(A; dims)`` / ``sortperm(A; dims)`` (row f15): K26 compiled for sm_90a without stack or spills, its per-element code
replayed on the host (tools/sortperm_slices_host_check.cu) against the stable ``isless`` permutation of every fibre, the host flow of
_sort.py through the host-memory emulation of the C ABI (tests/sort_dims_hostmem.py) on 1, 3 and 8 workers, the refusals, and the GPU
module run against that emulation."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import sort_dims_hostmem
from test_gpu_sort_dims import _bits, _data, model_perm

sort_dims_hostmem.install()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc")
L = sort_dims_hostmem.SMEM_LEN
CODES = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.int32): 2, np.dtype(np.int64): 3}


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


def test_limit_matches_the_header():
    from darray_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dab200.h")).read()
    assert int(re.search(r"#define DAB_SORTPERM_SLICES_SMEM_LEN (\d+)", hdr).group(1)) == L == _lib.SORTPERM_SLICES_SMEM_LEN


def test_k26_compiles_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_sortperm_slices.cu for sm_90a: every kernel uses no stack frame and spills nothing."""
    r = subprocess.run([_nvcc(), "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", os.path.join(CSRC, "dab_sortperm_slices.cu"), "-o", os.devnull],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 6 and len(frames) >= len(entries), r.stderr[-2000:]      # 4 network instances, fibre ids, finish
    assert all(f == ("0", "0", "0") for f in frames), r.stderr[-2000:]


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sps") / "sortperm_slices_host_check")
    subprocess.check_call([_nvcc(), "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", CSRC, "-I", os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(ROOT, "tools", "sortperm_slices_host_check.cu")])
    return exe


def _replay(exe, tmp_path, path, a, dim, lo=None, gdims=None):
    N = a.ndim
    lo = [0] * N if lo is None else list(lo)
    gdims = list(a.shape) if gdims is None else list(gdims)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    hdr = np.array([CODES[a.dtype], N, dim] + list(a.shape) + lo + gdims, dtype=np.int64)
    fin.write_bytes(hdr.tobytes() + np.ascontiguousarray(a.reshape(-1, order="F")).tobytes())
    subprocess.check_call([exe, path, str(fin), str(fout)], stdout=subprocess.DEVNULL)
    return np.frombuffer(fout.read_bytes(), dtype=np.int64).reshape(a.shape, order="F")


@pytest.mark.parametrize("T", [np.float32, np.float64, np.int32, np.int64])
def test_host_replay_network_and_long_path(host_check, tmp_path, T):
    """Both paths of K26, element code replayed: padding and both group shapes (inner == 1 and > 1), the fibre-id and global-index
    arithmetic and the long-fibre composition, for NaN payloads of both signs, +-0, +-Inf, integer extremes and heavy ties."""
    rng = np.random.default_rng(7)
    for ln in (1, 2, 3, 31, 32, 33, 100, 1000, L, L + 1):
        for shape, dim in (((ln, 5), 1), ((3, ln, 2), 2), ((2, 3, ln), 3), ((700, ln), 2)):
            if np.prod(shape) > 60000:
                continue
            for kind in ("specials", "repeated", "equal"):
                a = _data(T, int(np.prod(shape)), rng, kind).reshape(shape, order="F")
                want = model_perm(a, dim)
                for path in ("net", "long"):
                    assert np.array_equal(_replay(host_check, tmp_path, path, a, dim), want), (path, ln, shape, kind)


def test_host_replay_chunk_offsets(host_check, tmp_path):
    rng = np.random.default_rng(8)
    for N in range(2, 9):
        for dim in sorted({1, (N + 1) // 2, N}):
            shape = [int(x) for x in rng.integers(1, 4, N)]
            shape[dim - 1] = int(rng.integers(2, 50))
            lo = [0 if k == dim - 1 else int(rng.integers(1, 6)) for k in range(N)]
            gdims = [s if k == dim - 1 else s + lo[k] + int(rng.integers(0, 3)) for k, s in enumerate(shape)]
            a = _data(np.float64, int(np.prod(shape)), rng, "specials").reshape(shape, order="F")
            want = model_perm(a, dim, lo, gdims)
            for path in ("net", "long"):
                assert np.array_equal(_replay(host_check, tmp_path, path, a, dim, lo, gdims), want), (path, N, dim, shape)


LAYOUTS = [((40, 12), None), ((40, 12), "rows"), ((40, 12), "cols"), ((9, 7, 5), None), ((L + 5, 3), "rows"), ((3, L + 5), "cols")]


def _distribute(dab, a, how, nw):
    if how is None:
        return dab.distribute(a)
    dist = [nw, 1] if how == "rows" else [1, nw]
    return dab.distribute(a, procs=list(range(1, nw + 1)), dist=dist)


@pytest.mark.parametrize("nw", [1, 3, 8])
def test_host_flow(hostmem, dab, nw):
    """_sort.py's dims forms end to end on the host-memory ABI: split (redistribution) and whole dims, uneven chunk sizes (40 rows over 3
    workers, a 3-D array over 8), ``by``, and no device block outlives the calls."""
    sort_dims_hostmem.install_slices(hostmem)
    dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(50 + nw)
    for T in (np.float64, np.int32):
        for shape, how in LAYOUTS:
            a = _data(T, int(np.prod(shape)), rng, "repeated").reshape(shape, order="F")
            A = _distribute(dab, a, how, nw)
            for dim in range(1, a.ndim + 1):
                P = dab.sortperm(A, dims=dim)
                assert np.array_equal(dab.to_array(P), model_perm(a, dim))
                S = dab.sort(A, dims=dim)
                assert list(S.layout.indices) == list(P.layout.indices)
                Sb = dab.sort(A, dims=dim, by=abs)
                want = a.reshape(-1, order="F")[model_perm(np.abs(a), dim) - 1]
                assert np.array_equal(_bits(dab.to_array(Sb)), _bits(want)) and list(Sb.layout.indices) == list(P.layout.indices)
                for x in (P, S, Sb):
                    x.close()
            A.close()
    n0 = len(hostmem.blocks)
    A = dab.distribute(_data(np.float64, 600, rng).reshape((30, 20), order="F"))
    for by in (None, abs):
        dab.sortperm(A, dims=1, by=by).close()
        dab.sortperm(A, dims=2, by=by).close()
        dab.sort(A, dims=2, by=by).close()
    A.close()
    assert len(hostmem.blocks) == n0


def test_host_refusals_launch_nothing(hostmem, dab):
    dab.init(workers_per_rank=4, use_dist=False)
    rng = np.random.default_rng(9)
    A = dab.distribute(rng.standard_normal((8, 8)))
    Z = dab.distribute(rng.standard_normal((8, 8)).astype(np.complex128))
    H = dab.distribute(rng.standard_normal((8, 8)).astype(np.float16))
    n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
    for exc, f in [(dab.ArgumentError, lambda: dab.sortperm(A, dims=0)), (dab.ArgumentError, lambda: dab.sortperm(A, dims=np.bool_(True))),
                   (dab.ArgumentError, lambda: dab.sort(A, dims=2, sample=False)), (dab.ArgumentError, lambda: dab.sortperm(A, dims=1, rev=True)),
                   (TypeError, lambda: dab.sortperm(Z, dims=1)), (dab.UnsupportedError, lambda: dab.sort(Z, dims=1, by=abs)),
                   (dab.UnsupportedError, lambda: dab.sortperm(H, dims=2)), (dab.UnsupportedError, lambda: dab.sortperm(A[1:5, 2:4], dims=1))]:
        with pytest.raises(exc):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), exc
    assert dab.sortperm(A, dims=np.int64(2)).dims == (8, 8)


def test_gpu_sort_dims_module_against_the_host_memory_abi():
    """tests/test_gpu_sort_dims.py with the C ABI emulated over host memory: the host flow around K26 against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_sort_dims.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 25, tail
