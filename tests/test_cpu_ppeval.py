"""CPU tier of ``ppeval`` (reference src/mapreduce.jl:210-323, test/darray.jl:973-986): the oracle's restatement of ``_ppeval`` /
``ppeval`` / ``DArray(refs)`` on hand-worked cases, the batched kernels compiled for sm_90a without spills, the Jacobi element code of the
eigenvalue kernel replayed on the host (tools/ppeval_host_check.cu) against ``numpy.linalg.eigvalsh``, and the host runtime's whole
``ppeval`` flow over the host-memory emulation of the C ABI."""
import operator
import os
import shutil
import subprocess

import numpy as np
import pytest

import ppeval_oracle as po
from oracle import darray_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc")


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


# ---- the oracle -----------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("P", [1, 2, 3, 8])
def test_oracle_reference_testset_shapes(P):
    """test/darray.jl:974-981: A (10,10,P) and B (10,P) on P workers, one slice each; ppeval(*) is the per-slice product, on grid (1, P)."""
    rng = np.random.default_rng(P)
    A, B = rng.standard_normal((10, 10, P)), rng.standard_normal((10, P))
    pids = list(range(2, P + 2))
    oA, oB = orc.distribute(A, procs=pids, dist=[1, 1, P]), orc.distribute(B, procs=pids, dist=[1, P])
    R = po.darray_ppeval(operator.matmul, oA, oB)
    assert R.dims == (10, P) and R.grid == (1, P) and R.pids == pids
    assert R.indices == [((1, 10), (p, p)) for p in range(1, P + 1)]
    assert np.allclose(orc.to_array(R), np.stack([A[:, :, i] @ B[:, i] for i in range(P)], axis=1))
    S = A + A.transpose(1, 0, 2)
    E = po.darray_ppeval(lambda M: np.linalg.eigvalsh(M), orc.distribute(S, procs=pids, dist=[1, 1, P]))
    assert E.dims == (10, P) and np.isclose(orc.to_array(E).sum(), np.trace(S).sum())


def test_oracle_scalar_vector_matrix_results():
    """Chunks are (size(f(slice))..., nlocal): a scalar gives (nlocal,), a vector (n, nlocal), a matrix (m, n, nlocal); the grid
    (sd[1:nd-1]..., sd[end]) of procs grid (1, 1, 3) is (3,), (1, 3) and (1, 1, 3)."""
    A = np.arange(2.0 * 3 * 7).reshape((2, 3, 7), order="F")
    oA = orc.distribute(A, procs=[1, 2, 3], dist=[1, 1, 3])          # 3 + 2 + 2 slices
    s = po.darray_ppeval(np.sum, oA)
    assert s.dims == (7,) and s.grid == (3,) and [c.shape for c in s.chunks] == [(3,), (2,), (2,)]
    assert np.array_equal(orc.to_array(s), A.sum(axis=(0, 1)))
    v = po.darray_ppeval(lambda M: M[:, 0], oA)
    assert v.dims == (2, 7) and v.grid == (1, 3) and np.array_equal(orc.to_array(v), A[:, 0, :])
    m = po.darray_ppeval(lambda M: M.T, oA)
    assert m.dims == (3, 2, 7) and m.grid == (1, 1, 3) and np.array_equal(orc.to_array(m), A.transpose(1, 0, 2))


def test_oracle_dim_not_last():
    """Slicing along dimension 1 of a (4, 2, 3) array held on grid (2, 1, 1): chunks (2, 3, 2) on the grid (2, 1, 1) of procs, which
    stacks the two workers' results along dimension 1."""
    A = np.arange(24.0).reshape((4, 2, 3), order="F")
    oA = orc.distribute(A, procs=[1, 2], dist=[2, 1, 1])
    r = po.darray_ppeval(lambda M: M, oA, dim=(1,))
    assert [c.shape for c in r.chunks] == [(2, 3, 2), (2, 3, 2)] and r.grid == (2, 1, 1) and r.dims == (4, 3, 2)
    assert np.array_equal(r.chunks[0], np.moveaxis(A[:2], 0, -1)) and np.array_equal(r.chunks[1], np.moveaxis(A[2:], 0, -1))
    # slices are paired worker by worker: x (2, 3) sliced along 1 holds 1 slice per worker, M (2, 2, 3) sliced along 3 holds 2 and 1
    ox = orc.distribute(np.arange(6.0).reshape((2, 3), order="F"), procs=[1, 2], dist=[2, 1])
    oM = orc.distribute(np.ones((2, 2, 3)), procs=[1, 2], dist=[1, 1, 2])
    with pytest.raises(po.RefError) as e:
        po.darray_ppeval(lambda x, M: M @ x, ox, oM, dim=(1, 3))
    assert e.value.kind == "ArgumentError"


@pytest.mark.parametrize("case", ["dim_length", "distributed", "local_counts", "grid_prod", "grid_bounds", "inconsistent"])
def test_oracle_errors(case):
    o = orc.distribute(np.ones((10, 10, 4)), procs=[1, 2], dist=[1, 1, 2])
    if case == "dim_length":
        with pytest.raises(po.RefError, match="dim argument has wrong length. length\\(dim\\) = 1 but should be 2") as e:
            po.darray_ppeval(operator.matmul, o, o, dim=(3,))
    elif case == "distributed":
        with pytest.raises(po.RefError, match="dimension 1 is distributed. ppeval requires dimension 1") as e:
            po.darray_ppeval(np.sum, orc.distribute(np.ones((10, 4)), procs=[1, 2], dist=[2, 1]), dim=(2,))
    elif case == "local_counts":
        with pytest.raises(po.RefError, match="lengths of broadcast dimensions") as e:
            po.darray_ppeval(operator.matmul, o, orc.distribute(np.ones((10, 5)), procs=[1, 2], dist=[1, 2]))
    elif case == "grid_prod":                                       # (10, 4) on (1, 2), vector results: grid (1, 2) fits; on a DVector
        with pytest.raises(po.RefError) as e:                       # grid (2,) a vector result needs (2, 2)
            po.darray_ppeval(lambda x: np.ones(3), orc.distribute(np.ones(4), procs=[1, 2], dist=[2]))
        assert e.value.kind == "DimensionMismatch"
    elif case == "grid_bounds":                                     # matrix results of a DVector's slices: sd[1:2] of a 1-d grid
        with pytest.raises(po.RefError) as e:
            po.darray_ppeval(lambda x: np.ones((2, 2)), orc.distribute(np.ones(4), procs=[1, 2], dist=[2]))
        assert e.value.kind == "BoundsError"
    else:                                                           # grid (2, 1): 3 and 1 slices cannot share the one column
        with pytest.raises(po.RefError) as e:
            po.darray_ppeval(np.sum, orc.distribute(np.ones((4, 3)), procs=[1, 2], dist=[2, 1]), dim=(1,))
        assert e.value.kind in ("Inconsistent", "DimensionMismatch")


def test_oracle_exact_matmul_wraps():
    a = np.array([[2 ** 31 - 1, 2]], dtype=np.int32)
    b = np.array([[2], [2 ** 30]], dtype=np.int32)
    want = ((2 ** 31 - 1) * 2 + 2 * 2 ** 30) % 2 ** 32
    want = want - 2 ** 32 if want >= 2 ** 31 else want
    assert po.exact_matmul(a, b)[0, 0] == want
    assert po.exact_matmul(np.zeros((3, 0)), np.zeros((0, 2))).shape == (3, 2)


# ---- kernels: compile, and replay the eigenvalue element code on the host ----------------------------------------------------------------


def test_batched_kernels_compile_for_sm90a_without_spills(tmp_path):
    """dab_batched.cu builds for sm_90a with the library's flags; ptxas reports every kernel and 0 spill bytes for each."""
    out = subprocess.run([_nvcc(), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
                          "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "dab_batched.cu"), "-o",
                          str(tmp_path / "dab_batched.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    log = out.stderr
    for kern in ("bmm_small_kernel", "bmv_kernel", "bmm_tile_kernel", "eigvals_sym_kernel"):
        assert kern in log
    spills = [ln for ln in log.splitlines() if "spill stores" in ln]
    assert len(spills) == 14, log                                  # 3 product kernels x 4 dtypes + the eigenvalue kernel x 2
    assert all(" 0 bytes spill stores, 0 bytes spill loads" in ln for ln in spills), log


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("ppeval") / "ppeval_host_check")
    subprocess.check_call([_nvcc(), "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", CSRC, "-o", exe,
                           os.path.join(ROOT, "tools", "ppeval_host_check.cu")])
    return exe


def _replay(exe, tmp_path, A):
    n, batch = A.shape[0], A.shape[2]
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        np.array([n, batch], dtype=np.int64).tofile(f)
        A.reshape(-1, order="F").tofile(f)
    out = subprocess.run([exe, str(fin), str(fout)], capture_output=True, text=True)
    assert out.returncode == 0 and "ppeval_host_check: ok" in out.stdout, out.stdout + out.stderr
    r = np.fromfile(fout).reshape(batch, n + 1)
    return r[:, :n], r[:, n]


@pytest.mark.parametrize("n", [1, 2, 10, 33, 64])
def test_jacobi_host_replay_vs_eigvalsh(host_check, tmp_path, n):
    """Random symmetric, diagonal, zero, repeated-eigenvalue and rank-deficient matrices, and entries scaled to 1e+-300 and 1e-310:
    |lambda - lambda_ref| <= 64 n 2^-52 max|lambda_ref|, ascending, within the sweep limit."""
    rng = np.random.default_rng(n)
    X = rng.standard_normal((n, n))
    Sym = X + X.T
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    r = max(1, n // 2)
    Y = rng.standard_normal((n, r))
    mats = [Sym, np.diag(rng.standard_normal(n)), np.zeros((n, n)), (Q * np.resize([1.0, -2.0, 1.0], n)) @ Q.T, Y @ Y.T,
            Sym * 1e300, Sym * 1e-300, Sym * 1e-310]
    A = np.stack(mats, axis=2)
    got, sweeps = _replay(host_check, tmp_path, A)
    for b in range(A.shape[2]):
        want = np.linalg.eigvalsh(A[:, :, b])
        assert np.all(np.isfinite(got[b])) and np.all(np.diff(got[b]) >= 0), (n, b)
        assert np.max(np.abs(got[b] - want)) <= 64 * n * 2.0 ** -52 * np.max(np.abs(want)), (n, b)
        assert 1 <= sweeps[b] <= 40


# ---- the host runtime over the emulated C ABI -----------------------------------------------------------------------------------------


@pytest.fixture()
def rt8h(hostmem, dab):
    po.install_hostmem(hostmem)
    return dab.init(workers_per_rank=8, use_dist=False)


def test_host_flow_reference_testset(rt8h, dab):
    po.check_reference_testset(dab)


def test_host_flow_layouts(rt8h, dab):
    po.check_layouts(dab)


def test_host_flow_errors_before_any_launch(rt8h, dab):
    po.check_errors_before_launch(dab, rt8h)


def test_host_flow_status_errors(rt8h, dab):
    po.check_status_errors(dab)


def test_host_flow_packing_strides(rt8h, dab, hostmem):
    """What the runtime hands dab_matmul_batched: slice strides m*k / k*n for packed operands and 0 for a broadcast host operand, the
    batch a worker's slice count; no temporaries survive the call."""
    calls = []
    real = hostmem.dab_matmul_batched

    def spy(*a):
        calls.append([int(v.value if hasattr(v, "value") else v or 0) for v in a[1:]])
        return real(*a)

    hostmem.dab_matmul_batched = spy
    pids = list(dab.workers())
    A = np.random.default_rng(2).standard_normal((3, 4, 16))
    H = np.ones((4, 2))
    D = dab.distribute(A, procs=pids, dist=[1, 1, 8])
    reg0 = dab.registry_size()
    R = dab.ppeval(lambda a, h: a @ h, D, H)
    assert [(c[1], c[2], c[3], c[5], c[7], c[9]) for c in calls] == [(3, 2, 4, 12, 0, 2)] * 8
    assert np.allclose(dab.to_array(R), np.einsum("ikb,kj->ijb", A, H))
    R.close()
    assert dab.registry_size() == reg0
    A2 = np.ascontiguousarray(A.transpose(2, 0, 1))                # (16, 3, 4) sliced along 1: every chunk is packed to (3, 4, 2) first
    D2 = dab.distribute(A2, procs=pids, dist=[8, 1, 1])
    calls.clear()
    R2 = dab.ppeval(lambda a, h: a @ h, D2, H, dim=(1, 0))
    assert [(c[1], c[2], c[3], c[5], c[7], c[9]) for c in calls] == [(3, 2, 4, 12, 0, 2)] * 8
    want = po.darray_ppeval(lambda a, h: a @ h, orc.distribute(A2, procs=pids, dist=[8, 1, 1]), H, dim=(1, 0))
    po.assert_same_layout(R2, want)
    assert R2.dims == (24, 2, 2) and np.allclose(dab.to_array(R2), orc.to_array(want))
    R2.close()
    D.close()
    D2.close()
    assert dab.registry_size() == reg0 - 1                          # D is gone; nothing else was left behind
