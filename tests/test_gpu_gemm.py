"""GPU parity tests for K12 (dab_gemm): the tile product of the matrix-matrix mul! (reference src/linalg.jl:189-257).

Float32 goes through the wgmma 3xTF32 kernel (TMA operands, register accumulators) when bases / leading dimensions are 16-byte aligned and
through the SIMT tile kernel otherwise; Float64 / Int32 / Int64 through the SIMT kernel.  Integers are exact (wrap-around like Julia);
floats are compared with an fp64 product: |R - R64| <= tol * (|A| @ |B|) elementwise (the forward-error form of every GEMM bound),
tol = 2e-6 for Float32 (BLAS sgemm itself only guarantees k * eps), 1e-14 * k for Float64."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
F32 = np.float32


def gemm(dab, rt, A, B, transA=False, lda=None, ldb=None):
    from darray_b200 import _lib
    A, B = np.asfortranarray(A), np.asfortranarray(B)
    k, n = B.shape
    m = A.shape[1] if transA else A.shape[0]
    assert (A.shape[0] if transA else A.shape[1]) == k
    ra = A.shape[0]
    lda = lda or ra
    ldb = ldb or k
    dA = dab.B200Array.empty(rt, (lda, A.shape[1]), A.dtype)
    dB = dab.B200Array.empty(rt, (ldb, n), A.dtype)
    hA = np.zeros((lda, A.shape[1]), dtype=A.dtype, order="F")
    hA[:ra] = A
    hB = np.zeros((ldb, n), dtype=A.dtype, order="F")
    hB[:k] = B
    dA.copy_from_host(hA)
    dB.copy_from_host(hB)
    dC = dab.B200Array.empty(rt, (m, n), A.dtype)
    _lib.call("dab_gemm", rt.ctx, dab.dab_dtype(A.dtype), 1 if transA else 0, m, n, k, C.c_void_p(dA.ptr), lda, C.c_void_p(dB.ptr), ldb,
              C.c_void_p(dC.ptr), m)
    out = dC.to_numpy()
    for x in (dA, dB, dC):
        x.free()
    return out


def check_float(R, A, B, transA, tol):
    A64 = (A.T if transA else A).astype(np.float64)
    want = A64 @ B.astype(np.float64)
    bound = np.abs(A64) @ np.abs(B.astype(np.float64))
    err = np.abs(R.astype(np.float64) - want)
    worst = float((err / np.maximum(bound, 1e-300)).max())
    assert worst <= tol, worst
    return worst


SHAPES = [(128, 128, 32), (128, 128, 256), (256, 384, 512), (100, 60, 44), (37, 36, 1000), (1, 1, 1), (129, 257, 33), (512, 8, 2048),
          (4, 640, 4), (1024, 1024, 1024)]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("transA", [False, True])
def test_gemm_f32_tma_and_simt_kernels(dab, rt1, m, n, k, transA):
    rng = np.random.default_rng(m * 7 + n * 3 + k)
    for kind in ("uniform", "normal"):
        A = (rng.random((k, m) if transA else (m, k)) if kind == "uniform" else rng.standard_normal((k, m) if transA else (m, k))).astype(F32)
        B = (rng.random((k, n)) if kind == "uniform" else rng.standard_normal((k, n))).astype(F32)
        # exact leading dimensions (aligned only when the row count is a multiple of 4) and padded-to-4 leading dimensions (TMA path)
        for pad in (False, True):
            ra = A.shape[0]
            lda = (ra + 3) // 4 * 4 if pad else ra
            ldb = (k + 3) // 4 * 4 if pad else k
            R = gemm(dab, rt1, A, B, transA, lda, ldb)
            check_float(R, A, B, transA, 2e-6)
    # the SIMT kernel on the same data: a leading dimension of A that is not a multiple of 4 is one TMA cannot address
    ra = A.shape[0]
    R2 = gemm(dab, rt1, A, B, transA, ra if ra % 4 else ra + 1)
    check_float(R2, A, B, transA, 2e-6 * max(1.0, k / 512))


def test_gemm_f32_relative_1e6_on_positive_data(dab, rt1):
    """Uniform [0,1) data (the bench's distribution): every entry of the tensor-core product within 1e-6 RELATIVE of the fp64 product,
    for a long contraction, thanks to the two-level accumulation (register partials of 64 k, fp32 round-to-nearest between them)."""
    rng = np.random.default_rng(5)
    m, n, k = 256, 256, 8192
    A, B = rng.random((m, k)).astype(F32), rng.random((k, n)).astype(F32)
    want = A.astype(np.float64) @ B.astype(np.float64)
    R = gemm(dab, rt1, A, B)
    rel = float(np.abs(R.astype(np.float64) - want).max() / np.abs(want).min())
    assert rel <= 1e-6, rel


@pytest.mark.parametrize("dtype", [np.float64, np.int32, np.int64])
@pytest.mark.parametrize("transA", [False, True])
def test_gemm_other_types(dab, rt1, dtype, transA):
    rng = np.random.default_rng(11)
    for m, n, k in [(65, 130, 77), (128, 64, 256), (3, 5, 1000)]:
        if np.dtype(dtype).kind == "f":
            A, B = rng.standard_normal((k, m) if transA else (m, k)), rng.standard_normal((k, n))
            R = gemm(dab, rt1, A, B, transA)
            check_float(R, A, B, transA, 1e-15 * k)
        else:
            hi = 2 ** 20 if dtype == np.int32 else 2 ** 40            # products overflow and wrap, like Julia's machine integers
            A = rng.integers(-hi, hi, (k, m) if transA else (m, k)).astype(dtype)
            B = rng.integers(-hi, hi, (k, n)).astype(dtype)
            R = gemm(dab, rt1, A, B, transA)
            with np.errstate(over="ignore"):
                want = (A.T if transA else A) @ B                       # NumPy integer matmul wraps too
            assert R.dtype == np.dtype(dtype) and np.array_equal(R, want)

