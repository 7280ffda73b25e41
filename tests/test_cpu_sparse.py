"""CPU tier of sparse DArrays (row f9): the model of SparseArrays' loops (tests/sparse_oracle.py) against straightforward loops, the chunking
of ``distribute(S)`` against dense ``distribute`` over random layouts, the host canonicalisation, the K19 row-major order and the products
through the host-memory emulation of the C ABI (with tests/sparse_hostmem.py), the GPU module run against that emulation, and the no-spill compile of dab_sparse.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import sparse_hostmem
import sparse_oracle as so

sparse_hostmem.install()                                        # dab_spmv / dab_csc_to_csr for the host-memory emulation of the C ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _loop_fold(ptr, idx, val, x):
    out = np.zeros(len(ptr) - 1, dtype=val.dtype)
    with np.errstate(all="ignore"):
        for r in range(len(ptr) - 1):
            acc = val.dtype.type(0)
            for p in range(ptr[r], ptr[r + 1]):
                acc = acc + val[p] * x[idx[p]]
            out[r] = acc
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_vectorised_model_is_the_sequential_fold(dtype):
    rng = np.random.default_rng(1)
    lengths = rng.integers(0, 12, 200)
    lengths[::17] = 0
    ptr = np.concatenate(([0], np.cumsum(lengths))).astype(np.int64)
    idx = rng.integers(0, 50, int(ptr[-1])).astype(np.int32)
    if np.dtype(dtype).kind == "f":
        val = (rng.standard_normal(int(ptr[-1])) * 1e3).astype(dtype)
        x = rng.standard_normal(50).astype(dtype)
        val[::11], x[::13] = np.inf, -0.0
    else:
        hi = np.iinfo(dtype).max
        val, x = rng.integers(-hi, hi, int(ptr[-1])).astype(dtype), rng.integers(-hi, hi, 50).astype(dtype)
    assert so.same_bits(so.fold_rows(ptr, idx, val, x), _loop_fold(ptr, idx, val, x))


def test_float32_fold_rounds_every_step():
    """1 + 2^-24 + 2^-24 is 1 in Float32 folded left to right, 1 + 2^-23 summed in one go: the model must fold."""
    ptr = np.array([0, 3], dtype=np.int64)
    v = np.array([1, 2 ** -24, 2 ** -24], dtype=np.float32)
    got = so.fold_rows(ptr, np.array([0, 1, 2], dtype=np.int32), v, np.ones(3, dtype=np.float32))
    assert got[0] == np.float32(1)


def test_canonicalisation_of_unsorted_duplicates_and_stored_zeros():
    """A CSC with unsorted rows, duplicates and stored zeros: rows sorted, duplicates summed in storage order, zeros kept."""
    from darray_b200 import _sparse
    data = np.array([1.0, 0.0, 5.0, 2.0, -0.0, 3.0, 1e16, 1.0, -1e16])
    indices = np.array([3, 1, 3, 0, 2, 0, 4, 4, 4])
    indptr = np.array([0, 3, 5, 9])
    S = sp.csc_matrix((data, indices, indptr), shape=(5, 3))
    before = (S.data.copy(), S.indices.copy(), S.indptr.copy())
    shape, ip, rows, vals = _sparse.canonical_csc(S)
    assert shape == (5, 3) and list(ip) == [0, 2, 4, 6] and list(rows) == [1, 3, 0, 2, 0, 4]
    assert so.same_bits(vals, np.array([0.0, 6.0, 2.0, -0.0, 3.0, (1e16 + 1.0) + -1e16]))
    assert all(np.array_equal(a, b) for a, b in zip(before, (S.data, S.indices, S.indptr)))      # the input is not modified


def test_chunking_matches_dense_distribute_on_random_layouts(hostmem, dab):
    rng = np.random.default_rng(9)
    dab.init(workers_per_rank=8, use_dist=False)
    for trial in range(40):
        m, n = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        nw = int(rng.integers(1, 9))
        g0 = int(rng.choice([d for d in range(1, nw + 1) if nw % d == 0]))
        dist = (g0, nw // g0) if trial % 3 else None
        procs = list(rng.permutation(np.arange(1, 9))[:nw] + 0)
        S = sp.random(m, n, density=float(rng.uniform(0, 0.5)), random_state=rng, format="csc")
        S.data[::4] = 0.0
        try:
            D = dab.distribute(S.toarray(), procs=procs, dist=dist)
        except (dab.ArgumentError, ValueError):
            continue
        DS = dab.distribute(S, procs=procs, dist=dist)
        assert DS.layout.indices == D.layout.indices and list(DS.layout.pids) == list(D.layout.pids), (m, n, procs, dist)
        assert dab.nnz(DS) == S.nnz == sum(DS.chunk_nnz)
        r, c, v = so.canonical_triplets(S)
        for pid, ch in DS.chunks.items():
            shape, colptr, rowval, nzval = ch.to_host()
            tr, tc, tv = so.tile((r, c, v), DS.layout.localindices(pid))
            assert shape == D.chunks[pid].shape and colptr[-1] == tv.size
            assert np.array_equal(rowval, tr) and np.array_equal(np.repeat(np.arange(shape[1]), np.diff(colptr)), tc)
            assert so.same_bits(nzval, tv)
        dense = np.zeros((m, n))
        dense[r, c] = v
        assert so.same_bits(dab.to_array(DS), dense)
        DS.close()
        D.close()


def test_row_major_copy_order_and_products_on_the_host_memory_abi(hostmem, dab):
    """K19's composition (pack, K11 sort, unpack) gives rows ascending and columns ascending within a row; the distributed products
    through the real host runtime equal the model."""
    rng = np.random.default_rng(13)
    dab.init(workers_per_rank=8, use_dist=False)
    for dtype in (np.float32, np.int64):
        S = sp.random(90, 70, density=0.1, random_state=rng, format="csc").astype(dtype)
        if np.dtype(dtype).kind == "i":
            S.data = rng.integers(-2 ** 62, 2 ** 62, S.nnz).astype(dtype)
        DS = dab.distribute(S, dist=(4, 2))
        x = (rng.standard_normal(70) * 10).astype(dtype)
        y = dab.to_array(DS @ x)
        assert so.same_bits(y, so.mul_model(so.canonical_triplets(S), S.shape, DS.layout.cuts, x, False))
        for ch in DS.chunks.values():
            rowptr, colidx, val = (a.to_numpy() for a in ch.csr())
            _, colptr, rowval, nzval = ch.to_host()
            want = so.csc_to_csr(ch.shape[0], colptr, rowval, nzval)
            assert np.array_equal(rowptr, want[0]) and np.array_equal(colidx, want[1]) and so.same_bits(val, want[2])


def test_limits_and_types_refused_before_allocation(hostmem, dab):
    dab.init(workers_per_rank=2, use_dist=False)
    n0 = len(hostmem.blocks)

    class Huge:                                               # only shape and dtype are looked at before the refusal
        shape, dtype = (1 << 31, 4), np.dtype(np.float64)

        def tocsc(self):
            raise AssertionError("converted before the limit check")

    with pytest.raises(dab.UnsupportedError, match="2\\^31-1 rows"):
        dab.distribute(Huge(), procs=[1], dist=[1, 1])
    with pytest.raises(dab.UnsupportedError, match="complex"):
        dab.distribute(sp.random(4, 4, density=0.5, format="csc").astype(np.complex64))
    assert len(hostmem.blocks) == n0


def test_gpu_sparse_module_against_the_host_memory_abi():
    """tests/test_gpu_sparse.py with the C ABI emulated over host memory: the host runtime around K18 / K19 (layouts, chunk cuts, the mul!
    exchange and fold, the refusals, the launch and lifetime contracts) against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_sparse.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 30, tail


def test_dab_sparse_compiles_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_sparse.cu for sm_90a: no entry function uses a stack frame or spills."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_sparse.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "-Xptxas", "-v", "-c", src, "-o",
                        os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) >= 26 and len(frames) >= len(entries), r.stderr[-2000:]
    assert all(f == ("0", "0", "0") for f in frames), [e for e, f in zip(entries, frames) if f != ("0", "0", "0")]
