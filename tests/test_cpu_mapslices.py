"""CPU tier of ``mapslices`` (reference src/mapreduce.jl:191-208, test/darray.jl:804-841): the oracle's restatement of ``Base.mapslices``
on hand-checked cases, the slice kernels compiled for sm_90a, their per-element code replayed on the host (tools/slices_host_check.cu)
against ``std::sort`` / ``numpy.linalg.svd``, and the host runtime's whole ``mapslices`` flow over the host-memory emulation of the C ABI."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import mapslices_oracle as mo
from oracle import darray_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc")


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


# ---- the oracle -----------------------------------------------------------------------------------------------------------------------


def test_oracle_mapslices_issue_5177_shape_table():
    """test/darray.jl:823-836 on a host array: constant results of every shape over every pair of dims."""
    c = np.ones((2, 3, 4, 5))
    for const, dims, want in (((2, 3), [1, 2], (2, 3, 4, 5)), ((2, 4), [1, 3], (2, 3, 4, 5)), ((3, 4), [2, 3], (2, 3, 4, 5)),
                              ((6,), [1, 2], (6, 1, 4, 5)), ((6,), [1, 3], (6, 3, 1, 5)), ((6,), [2, 3], (2, 6, 1, 5)),
                              ((1, 6), [1, 2], (1, 6, 4, 5)), ((1, 6), [1, 3], (1, 3, 6, 5)), ((1, 6), [2, 3], (2, 1, 6, 5))):
        r = mo.jl_mapslices(lambda x, s=const: np.ones(s), c, dims)
        assert r.shape == want and np.all(r == 1)
    with pytest.raises(ValueError):                                # size(r1, 3) > 1 beyond the two slice dims
        mo.jl_mapslices(lambda x: np.ones((2, 3, 2)), c, [1, 2])


def test_oracle_mapslices_scalar_results_and_empty_dims():
    A = np.arange(24.0).reshape((2, 3, 4), order="F")
    B = mo.jl_mapslices(np.sum, A, [1, 2])                          # issue #3613: scalars collapse the slice dims to 1
    assert B.shape == (1, 1, 4) and list(B.ravel()) == [15.0, 51.0, 87.0, 123.0]
    assert mo.jl_mapslices(np.sum, A, [3]).shape == (2, 3, 1)
    assert np.array_equal(mo.jl_mapslices(np.sum, A, [3])[:, :, 0], A.sum(axis=2))
    C = mo.jl_mapslices(lambda x: np.max(-x), A, [])                # issue #5141: dims=[] is map(f, A)
    assert np.array_equal(C, -A)
    S = mo.jl_mapslices(np.sort, A[:, :, ::-1].copy(order="F"), [3])
    assert np.array_equal(S, A)
    V = mo.jl_mapslices(mo.svdvals_np, A, [1, 3])                   # svdvals of the 2x4 slices: a 2-vector along dim 1
    assert V.shape == (2, 3, 1) and np.allclose(V[:, 1, 0], np.linalg.svd(A[:, 1, :], compute_uv=False))


def test_oracle_darray_mapslices_layouts():
    """Redistribution grid and result layout of the reference's DArray-level mapslices."""
    A = np.arange(125.0).reshape((5, 5, 5), order="F")
    d = orc.distribute(A, procs=list(range(1, 9)), dist=[1, 1, 5])
    assert d.pids == [1, 2, 3, 4, 5]                                # procs(D): the five workers dist uses
    assert mo.redistribution_grid(d.dims, d.grid, [1, 2], 5) is None
    assert mo.redistribution_grid(d.dims, d.grid, [3], 5) == [1, 5, 1]     # defaultdist([5, 5], 5): the factor 5 to the last tie
    assert mo.redistribution_grid(d.dims, d.grid, [3], 8) == [2, 4, 1]     # defaultdist([5, 5], 8) = [2, 4]
    r = mo.darray_mapslices(np.sum, d, [1, 2])                     # local slice dims: same grid and pids, dims (1, 1, 5)
    assert r.dims == (1, 1, 5) and r.pids == d.pids and r.cuts == [[1, 2], [1, 2], d.cuts[2]]
    r = mo.darray_mapslices(np.sort, d, [3])                       # dim 3 is split: redistributed on the other two dims
    p = mo.redistribution_grid(d.dims, d.grid, [3], 5)
    assert list(r.grid) == p and r.dims == (5, 5, 5) and np.array_equal(orc.to_array(r), np.sort(A, axis=2))
    assert r.pids == list(range(1, int(np.prod(p)) + 1))


# ---- kernels: compile, and replay their element code on the host -----------------------------------------------------------------------


def test_slice_kernels_compile_for_sm90a(tmp_path):
    """dab_slices.cu builds for sm_90a (-fmad=false, like the library) without local-memory spills."""
    out = subprocess.run([_nvcc(), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                          "-Xptxas", "-v", "-c", os.path.join(CSRC, "dab_slices.cu"), "-o", str(tmp_path / "dab_slices.o")],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    log = out.stderr
    for kern in ("sort_slices_kernel", "svdvals_kernel"):
        assert kern in log
    assert "bytes spill stores" in log
    assert all(" 0 bytes spill stores" in ln for ln in log.splitlines() if "spill stores" in ln), log


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("slices") / "slices_host_check")
    subprocess.check_call([_nvcc(), "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", CSRC, "-o", exe,
                           os.path.join(ROOT, "tools", "slices_host_check.cu")])
    return exe


def test_sort_network_host_replay(host_check):
    """The bitonic network of sort_slices_kernel (padding, index map, directions) against std::sort, four dtypes, NaN payloads."""
    out = subprocess.run([host_check], capture_output=True, text=True)
    assert out.returncode == 0 and "slices_host_check: ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("shape", [(1, 1), (5, 5), (10, 10), (32, 32), (3, 17), (17, 3), (32, 128), (128, 32)])
def test_jacobi_host_replay_vs_numpy(host_check, tmp_path, shape):
    """The Jacobi sweeps of svdvals_kernel (pairing, rotation, tolerance, ranking) against numpy.linalg.svd in fp64."""
    m, n = shape
    k = min(m, n)
    rng = np.random.default_rng(m * 1000 + n)
    mats = [rng.standard_normal((m, n)), np.zeros((m, n)), np.eye(m, n)]
    r = max(1, k // 2)
    mats.append(rng.standard_normal((m, r)) @ rng.standard_normal((r, n)))          # rank-deficient
    U, _ = np.linalg.qr(rng.standard_normal((m, m)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    mats.append((U[:, :k] * np.logspace(0, -12, k)) @ V[:, :k].T)                   # condition number 1e12
    A = np.stack(mats, axis=2)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        np.array([m, n, A.shape[2]], dtype=np.int64).tofile(f)
        A.reshape(-1, order="F").tofile(f)
    subprocess.check_call([host_check, "svd", str(fin), str(fout)])
    got = np.fromfile(fout).reshape(A.shape[2], k)
    for b in range(A.shape[2]):
        want = np.linalg.svd(A[:, :, b], compute_uv=False)
        assert np.all(np.diff(got[b]) <= 0)
        assert np.max(np.abs(got[b] - want)) <= 1e-12 * max(want.max(), np.finfo(float).tiny), (shape, b)


@pytest.mark.parametrize("shape", [(5, 5), (32, 32), (3, 17), (128, 32)])
def test_jacobi_host_replay_extreme_magnitudes(host_check, tmp_path, shape):
    """Finite input far from 1 (sums of squares would overflow / underflow without the power-of-two scaling) against numpy, whose LAPACK
    scales its input too."""
    m, n = shape
    base = np.random.default_rng(m + 7 * n).standard_normal((m, n))
    scales = [1e160, 1e-170, 1e-160, 1e300, 1e-300, 1e-310]
    A = np.stack([base * s for s in scales], axis=2)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        np.array([m, n, A.shape[2]], dtype=np.int64).tofile(f)
        A.reshape(-1, order="F").tofile(f)
    subprocess.check_call([host_check, "svd", str(fin), str(fout)])
    got = np.fromfile(fout).reshape(A.shape[2], min(m, n))
    for b, s in enumerate(scales):
        want = np.linalg.svd(A[:, :, b], compute_uv=False)
        assert np.all(np.isfinite(got[b])) and np.max(np.abs(got[b] - want)) <= 1e-12 * want.max(), (shape, s)


# ---- the host runtime over the emulated C ABI -----------------------------------------------------------------------------------------


@pytest.fixture()
def rt8h(hostmem, dab):
    mo.install_hostmem(hostmem)
    return dab.init(workers_per_rank=8, use_dist=False)


def test_host_flow_reference_testset(rt8h, dab):
    mo.check_reference_testset(dab)


def test_host_flow_layouts(rt8h, dab):
    mo.check_layouts(dab)


def test_host_flow_errors_before_any_launch(rt8h, dab):
    mo.check_errors_before_launch(dab, rt8h)


def test_host_flow_svdvals_nonfinite_raises(rt8h, dab):
    A = np.random.default_rng(0).standard_normal((4, 4, 6))
    A[2, 1, 5] = np.nan
    D = dab.distribute(A, dist=[1, 1, 3])
    with pytest.raises(dab.ArgumentError, match="Infs or NaNs"):
        dab.mapslices(dab.svdvals, D, dims=(1, 2))
    A[2, 1, 5] = np.inf
    with pytest.raises(dab.ArgumentError, match="Infs or NaNs"):
        dab.mapslices(dab.svdvals, dab.distribute(A, dist=[1, 1, 3]), dims=(1, 2))
