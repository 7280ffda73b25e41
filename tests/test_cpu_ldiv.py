"""CPU tier of ``ldiv`` / ``det`` of slices (row f17, K27): the kernels compiled for sm_90a with no stack frame and no spills, the element
code of dab_lu_core.cuh replayed on the host (tools/lu_host_check.cu) against NumPy and SciPy, the host flow of ppeval / mapslices through
the host-memory model of K27 (tests/ldiv_hostmem.py) on 1, 3 and 8 workers, and the GPU module run against that model."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg as sla

import ldiv_hostmem as lh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc")
PATHS = {0: "lu", 1: "lower", 2: "upper", 3: "diag"}


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


def test_limit_matches_the_header():
    from darray_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dab200.h")).read()
    assert int(re.search(r"#define DAB_LU_MAX_N (\d+)", hdr).group(1)) == lh.LU_MAX_N == _lib.LU_MAX_N


def test_k27_compiles_without_stack_or_spills():
    """``nvcc -fmad=false -Xptxas -v`` of dab_lu_batched.cu for sm_90a: 20 kernels (4 group widths and the block kernel, x 2 dtypes x
    ldiv / det), none with a stack frame or a spill."""
    r = subprocess.run([_nvcc(), "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c", os.path.join(CSRC, "dab_lu_batched.cu"), "-o", os.devnull],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 20 and len(frames) == len(entries), r.stderr[-2000:]
    assert all(f == ("0", "0", "0") for f in frames), r.stderr[-2000:]


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("lu") / "lu_host_check")
    subprocess.check_call([_nvcc(), "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", CSRC, "-o", exe,
                           os.path.join(ROOT, "tools", "lu_host_check.cu")])
    return exe


def _replay(exe, tmp_path, mats):
    n = mats[0].shape[0]
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(np.array([n, len(mats)], dtype=np.int64).tobytes()
                    + b"".join(np.asarray(M, dtype=np.float64).reshape(-1, order="F").tobytes() for M in mats))
    out = subprocess.run([exe, str(fin), str(fout)], capture_output=True, text=True)
    assert out.returncode == 0 and "lu_host_check: ok" in out.stdout, out.stdout + out.stderr
    return np.fromfile(fout).reshape(len(mats), n + 3)


@pytest.mark.parametrize("n", list(range(1, 17)) + [31, 32, 33, 47, 63, 64])
def test_host_replay_vs_numpy_scipy(host_check, tmp_path, n):
    """Path, pivot sequence (against lu_factor's piv on matrices without ties), info on every path -- a lower-triangular singular slice
    included, where LU pivoting would report another index -- and det's sign and value."""
    rng = np.random.default_rng(n)
    dense = [rng.standard_normal((n, n)) for _ in range(4)]
    mats = dense + [np.diag(rng.standard_normal(n)), np.tril(dense[0]), np.triu(dense[1])]
    if n > 1:
        L = np.tril(dense[2])
        L[0, 0] = 0.0
        U = np.triu(dense[3])
        U[n - 1, n - 1] = -0.0
        Z = dense[0].copy()
        Z[:, n // 2] = 0.0
        N = dense[1].copy()
        N[n - 1, 0] = np.nan
        D = np.diag(rng.standard_normal(n))
        D[n // 2, n // 2] = 0.0
        mats += [L, U, Z, N, D]
    got = _replay(host_check, tmp_path, mats)
    for M, row in zip(mats, got):
        path, info, det, piv = PATHS[int(row[0])], row[1], row[2], row[3:].astype(int)
        assert path == lh.path_of(M)
        x, fail = lh.jl_ldiv(M, np.ones(n))
        want_info = 0 if fail is None else (-1 if fail[0] == "nonfinite" else fail[1])
        assert info == want_info, (n, path, info, want_info)
        if path == "lu" and np.all(np.isfinite(M)):
            _, wpiv, _ = lh.lu_factor(M)
            assert np.array_equal(piv, wpiv), (n, piv, wpiv)
        wd = lh.jl_det(M)
        if np.isnan(wd):
            assert np.isnan(det)
        else:
            assert np.signbit(det) == np.signbit(wd) and abs(det - wd) <= 64 * n * 2.0 ** -52 * abs(wd), (n, path, det, wd)
        if path == "lu" and fail is None:
            assert abs(det - np.linalg.det(M)) <= 64 * n * 2.0 ** -52 * abs(np.linalg.det(M))
    if n > 1:                                                      # the lower singular slice: substitution says 1, LU pivoting another
        lu, piv, linfo = lh.lu_factor(mats[7])
        assert got[7][1] == 1 and linfo != 1


@pytest.fixture()
def k27(hostmem):
    return lh.install(hostmem)


@pytest.mark.parametrize("nw", [1, 3, 8])
def test_host_flow(k27, dab, nw):
    """ppeval(ldiv) / ppeval(det) / mapslices(det) end to end on the host-memory ABI: layouts and values against the oracle's ppeval with
    numpy.linalg.solve / det, Int32 / Int64, broadcast operands, dim not last, and the status errors on every worker count."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    lh.check_forms(dab)
    lh.check_status_errors(dab)
    lh.check_errors_before_launch(dab, rt)


def test_ldiv_and_det_outside_ppeval_raise(dab):
    for f in (lambda: dab.ldiv(np.eye(2), np.ones(2)), lambda: dab.det(np.eye(2))):
        with pytest.raises(dab.UnsupportedError, match="ppeval"):
            f()
    e = dab.SingularException(3)
    assert isinstance(e, dab.DabError) and e.info == 3 and str(e) == "SingularException(3)"


def test_gpu_ldiv_module_against_the_host_memory_abi():
    """tests/test_gpu_ldiv.py with the C ABI emulated over host memory: the host flow around K27 against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_ldiv.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 39, tail
