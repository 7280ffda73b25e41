"""GPU parity tests for the Level-2 widening: K9 dab_gemv / mul! / A*x / A'*x (reference src/linalg.jl:78-167, 280-311; tests
test/darray.jl:933-941), K10 copy(transpose/adjoint) (src/linalg.jl:1-17; test/darray.jl:713-733) and Diagonal lmul!/rmul!
(src/linalg.jl:169-187; test/darray.jl:270-282).  Integer results and every data movement are bit-exact against the oracle;
Float results obey the 1e-6 (Float32) relative bound against an fp64 truth, scaled by sum |a||x| as for any dot product."""
import ctypes as C

import numpy as np
import pytest

from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu


def _gemv(dab, rt, A, x, trans):
    from darray_b200 import _lib
    dA = dab.B200Array.from_numpy(rt, np.asfortranarray(A))
    dx = dab.B200Array.from_numpy(rt, x) if x.size else dab.B200Array.empty(rt, (0,), A.dtype)
    nout = A.shape[1] if trans else A.shape[0]
    dr = dab.B200Array.empty(rt, (nout,), A.dtype)
    _lib.call("dab_gemv", rt.ctx, dab.dab_dtype(A.dtype), int(trans), C.c_void_p(dA.ptr), A.shape[0], A.shape[1], C.c_void_p(dx.ptr),
              C.c_void_p(dr.ptr))
    out = dr.to_numpy()
    for b in (dA, dx, dr):
        b.free()
    return out


def _check_matvec(got, A, x, trans):
    M = A.T if trans else A
    if A.dtype.kind == "f":
        want = M.astype(np.float64) @ x.astype(np.float64)
        scale = np.abs(M.astype(np.float64)) @ np.abs(x.astype(np.float64))
        tol = 1e-6 if A.dtype == np.float32 else 1e-14
        assert got.dtype == A.dtype and np.all(np.abs(got - want) <= tol * scale + 1e-300)
        if A.dtype == np.float32:
            # and it agrees with the oracle's restatement (fp64 accumulate, one rounding) to the last bit or one ulp
            o = orc._tile_matvec(np.asfortranarray(A), x, trans)
            assert np.all(np.abs(got - o) <= np.maximum(np.spacing(np.abs(o)), 1e-12 * scale))
    else:
        o = orc._tile_matvec(np.asfortranarray(A), x, trans)
        assert got.dtype == A.dtype and np.array_equal(got, o)


SHAPES = [(1, 1), (7, 5), (64, 64), (1000, 3), (3, 1000), (4096, 257), (257, 4096), (1, 100003), (100003, 1), (33, 2049), (2048, 2048),
          (5, 0), (0, 5), (12, 16), (1028, 515), (4100, 1030)]


@pytest.mark.parametrize("trans", [0, 1])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_gemv_kernel_all_shapes(dab, rt1, dtype, trans):
    rng = np.random.default_rng(31 + trans)
    for (m, n) in SHAPES:
        k = m if trans else n
        if np.dtype(dtype).kind == "f":
            A = rng.standard_normal((m, n)).astype(dtype)
            x = rng.standard_normal(k).astype(dtype)
        else:
            hi = 2 ** 28 if dtype == np.int32 else 2 ** 60                   # products overflow: the wrap-around is part of the contract
            A = rng.integers(-hi, hi, (m, n)).astype(dtype)
            x = rng.integers(-hi, hi, k).astype(dtype)
        _check_matvec(_gemv(dab, rt1, A, x, trans), A, x, trans)


def _gemv_offset(dab, rt, A, x, off, trans=0, xoff=0):
    """A * x (or A' * x) with the matrix placed `off` elements and x `xoff` elements past a 256-byte aligned allocation (every phase
    of the 16-byte words)."""
    from darray_b200 import _lib
    m, n = A.shape
    flat = np.zeros(m * n + off, dtype=A.dtype)
    flat[off:] = np.asfortranarray(A).reshape(-1, order="F")
    xf = np.zeros(x.size + xoff, dtype=A.dtype)
    xf[xoff:] = x
    dA = dab.B200Array.from_numpy(rt, flat)
    dx = dab.B200Array.from_numpy(rt, xf)
    dr = dab.B200Array.empty(rt, (n if trans else m,), A.dtype)
    isz = A.dtype.itemsize
    _lib.call("dab_gemv", rt.ctx, dab.dab_dtype(A.dtype), int(trans), C.c_void_p(dA.ptr + off * isz), m, n, C.c_void_p(dx.ptr + xoff * isz),
              C.c_void_p(dr.ptr))
    out = dr.to_numpy()
    for b in (dA, dx, dr):
        b.free()
    return out


@pytest.mark.parametrize("trans", [0, 1])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_gemv_misaligned_columns_every_phase(dab, rt1, dtype, trans):
    """A*x and A'*x when the columns do not start on 16-byte boundaries (leading dimension not a multiple of 16 bytes and / or a
    misaligned base, x misaligned too): the phase-class kernels against the oracle, for every phase of the base pointer."""
    rng = np.random.default_rng(77 + trans)
    # the phase-class kernels take m >= 256 and n >= 64; the smaller shapes reach the unit-wise kernels
    for (m, n) in [(65, 17), (257, 64), (257, 4096), (1001, 515), (1023, 4097), (4099, 67), (32769, 77), (259, 1000), (1026, 130), (66, 35)]:
        k = m if trans else n
        if np.dtype(dtype).kind == "f":
            A = rng.standard_normal((m, n)).astype(dtype)
            x = rng.standard_normal(k).astype(dtype)
        else:
            hi = 2 ** 28 if dtype == np.int32 else 2 ** 60
            A = rng.integers(-hi, hi, (m, n)).astype(dtype)
            x = rng.integers(-hi, hi, k).astype(dtype)
        nph = 16 // np.dtype(dtype).itemsize
        for off in range(nph):
            xoff = (off * 3 + 1) % nph if trans else 0
            _check_matvec(_gemv_offset(dab, rt1, A, x, off, trans=trans, xoff=xoff), A, x, trans)


def test_gemv_large_chunk_bandwidth_shape(dab, rt1):
    """A 512 MiB Float32 chunk (the column-block shape of config C4 scaled to fit the test budget), both orientations; values on a
    2^-24 grid in [0,1) so the fp64-accumulated result is the correctly rounded exact answer."""
    m, n = 16384, 8192
    A = orc.rand_u01(7, 0, m * n).reshape((m, n), order="F")
    for trans in (0, 1):
        x = orc.rand_u01(8 + trans, 0, m if trans else n)
        got = _gemv(dab, rt1, A, x, trans)
        M = A.T if trans else A
        want = (M.astype(np.float64) @ x.astype(np.float64))
        assert np.all(np.abs(got - want) <= 1e-6 * want)
        w32 = want.astype(np.float32)                                        # exact products, fp64 sums: one rounding to Float32
        assert np.all(np.abs(got - w32) <= np.spacing(w32)) and np.mean(got == w32) > 0.999


@pytest.mark.parametrize("dist", [(1, 1), (2, 1), (1, 2), (2, 4), (4, 2), (8, 1), (1, 8)])
def test_matvec_darray(dab, rt8, dist):
    rng = np.random.default_rng(37)
    for dtype in (np.float64, np.float32, np.int64):
        shape = (203, 157)
        if np.dtype(dtype).kind == "f":
            A = rng.standard_normal(shape).astype(dtype)
            mk = lambda k: rng.standard_normal(k).astype(dtype)                                  # noqa: E731
        else:
            A = rng.integers(-1000, 1000, shape).astype(dtype)
            mk = lambda k: rng.integers(-1000, 1000, k).astype(dtype)                            # noqa: E731
        nw = dist[0] * dist[1]
        procs = list(range(1, nw + 1))
        DA = dab.distribute(A, procs=procs, dist=dist)
        oA = orc.distribute(A, procs=procs, dist=list(dist))
        for trans in (False, True):
            x = mk(shape[0] if trans else shape[1])
            W = dab.transpose(DA) if trans else DA
            y = W @ x                                                                           # A*x / transpose(A)*x
            oy = orc.darray_matvec(oA, x, trans)
            assert y.layout.grid == tuple(oy.grid) and list(y.layout.pids) == oy.pids and list(y.layout.indices) == oy.indices
            got, want = dab.to_array(y), orc.to_array(oy)
            if np.dtype(dtype).kind == "f":
                M = A.T if trans else A
                scale = np.abs(M.astype(np.float64)) @ np.abs(x.astype(np.float64))
                assert np.all(np.abs(got - want) <= (2e-6 if dtype == np.float32 else 1e-14) * scale)
            else:
                assert np.array_equal(got, want)
            # x as a DVector with its own (default) layout: blocks are halo-fetched (x[A.cuts[2][j]:...], src/linalg.jl:91)
            y2 = W @ dab.distribute(x)
            assert np.array_equal(dab.to_array(y2), got)
            # mul!(y, A, x, alpha, beta) on an existing y
            y0 = mk(len(want))
            Y = dab.distribute(y0, procs=oy.pids, dist=[len(oy.pids)])
            oY = orc.distribute(y0, procs=oy.pids, dist=[len(oy.pids)])
            dab.mul_(Y, dab.adjoint(DA) if trans else DA, x, 3, 2)
            wantY = orc.to_array(orc.darray_mul_vec(oY, oA, x, 3, 2, trans))
            if np.dtype(dtype).kind == "f":
                assert np.all(np.abs(dab.to_array(Y) - wantY) <= (4e-6 if dtype == np.float32 else 1e-13) * (3 * scale + 2 * np.abs(y0)))
            else:
                assert np.array_equal(dab.to_array(Y), wantY)
            dab.mul_(Y, W, x, 1, 1)                                                              # alpha == beta == 1: plain accumulate
            if np.dtype(dtype).kind != "f":
                assert np.array_equal(dab.to_array(Y), wantY + orc.to_array(oy))


def test_matvec_errors_and_reference_dot_test(dab, rt8):
    rng = np.random.default_rng(41)
    A = rng.standard_normal((20, 20))
    b = rng.standard_normal(20)
    DA, Db = dab.distribute(A), dab.distribute(b)
    c = DA @ Db                                                               # test/darray.jl:933-941
    assert np.isclose(float(dab.dot(c, Db)), np.dot(dab.to_array(c), b), rtol=1e-12)
    assert np.allclose(dab.to_array(c), A @ b, rtol=1e-13, atol=1e-13)
    with pytest.raises(dab.DimensionMismatch):
        DA @ np.zeros(21)
    y_bad = dab.distribute(np.zeros(20), procs=[1, 2, 3], dist=[3])
    if list(y_bad.layout.cuts[0]) != list(DA.layout.cuts[0]):
        with pytest.raises(dab.ArgumentError):
            dab.mul_(y_bad, DA, b)
    with pytest.raises(dab.DimensionMismatch):
        DA @ np.zeros((21, 3))                                                # matrix-matrix: contracted sizes differ


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int64, np.int32])
@pytest.mark.parametrize("grid", [None, (8, 1), (1, 8), (2, 4), (4, 2)])
def test_matmatmul(dab, rt8, dtype, grid):
    """``A*B``, ``A'*B``, ``transpose(A)*B`` and ``mul!(C, A, B, alpha, beta)`` (reference src/linalg.jl:189-311; reference tests
    test/darray.jl:915-931, 996-1012): layout of the result (owners, grid, cuts) equals the oracle's, integer results exactly, float
    results within the forward-error bound of the tile products (K12: wgmma 3xTF32 for aligned Float32 tiles, SIMT otherwise)."""
    rng = np.random.default_rng(47)
    m, kdim, n = 96, 130, 72                               # 130 / 8 -> 17,17,16,... column blocks: unaligned leading dimensions too
    mk = (lambda *s: rng.integers(-9, 9, s).astype(dtype)) if np.dtype(dtype).kind != "f" else (lambda *s: rng.standard_normal(s).astype(dtype))
    A, At, B = mk(m, kdim), mk(kdim, m), mk(kdim, n)
    tol = 4e-6 if dtype == np.float32 else 1e-13
    for trans in (False, True):
        H = At if trans else A
        DA = dab.distribute(H, dist=grid)
        oA = orc.distribute(H, nworkers=8) if grid is None else orc.distribute(H, procs=list(range(1, 9)), dist=list(grid))
        for bgrid in (None, (1, 8), (8, 1)):
            DB = dab.distribute(B, dist=bgrid)
            oB = orc.distribute(B, nworkers=8) if bgrid is None else orc.distribute(B, procs=list(range(1, 9)), dist=list(bgrid))
            W = dab.transpose(DA) if trans else DA
            Cd = W @ DB
            oC = orc.darray_matmat(oA, oB, trans)
            assert Cd.layout.grid == tuple(oC.grid) and list(Cd.layout.pids) == oC.pids and list(Cd.layout.indices) == oC.indices
            got, want = dab.to_array(Cd), orc.to_array(oC)
            M = H.T if trans else H
            if np.dtype(dtype).kind == "f":
                bound = np.abs(M.astype(np.float64)) @ np.abs(B.astype(np.float64))
                assert np.all(np.abs(got.astype(np.float64) - M.astype(np.float64) @ B.astype(np.float64)) <= tol * bound)
                assert np.all(np.abs(got.astype(np.float64) - want) <= 2 * tol * bound)
            else:
                assert np.array_equal(got, want)
        # mul!(C, A, B, alpha, beta) on an existing C with the layout of A*B; B as a host matrix
        C0 = mk(M.shape[0], n)
        Cd = dab.distribute(C0, procs=oC.pids, dist=list(oC.grid))
        oC0 = orc.distribute(C0, procs=oC.pids, dist=list(oC.grid))
        dab.mul_(Cd, dab.adjoint(DA) if trans else DA, B, 3, 2)
        wantC = orc.to_array(orc.darray_mul_mat(oC0, oA, B, 3, 2, trans))
        if np.dtype(dtype).kind == "f":
            assert np.all(np.abs(dab.to_array(Cd) - wantC) <= 2 * tol * (3 * bound + 2 * np.abs(C0)))
        else:
            assert np.array_equal(dab.to_array(Cd), wantC)


def test_matmatmul_reference_tests_and_errors(dab, rt8):
    rng = np.random.default_rng(53)
    A, B = rng.standard_normal((30, 30)), rng.standard_normal((30, 20))       # test/darray.jl:996-1012
    DA, DB = dab.distribute(A), dab.distribute(B)
    for W, want in ((DA, A @ B), (dab.transpose(DA), A.T @ B), (dab.adjoint(DA), A.T @ B)):
        assert np.allclose(dab.to_array(W @ DB), want, rtol=1e-12, atol=1e-12)
    A2 = rng.standard_normal((20, 20))                                        # test/darray.jl:915-931
    B2 = rng.standard_normal((20, 20))
    D2, E2 = dab.distribute(A2), dab.distribute(B2)
    assert np.abs(dab.to_array(D2 @ E2) - A2 @ B2).max() < np.sqrt(np.finfo(np.float64).eps)
    assert np.abs(dab.to_array(D2.T @ E2) - A2.T @ B2).max() < np.sqrt(np.finfo(np.float64).eps)
    Cd = dab.dzeros((30, 20), procs=list(DA.layout.pids)[:DA.layout.grid[0]], dist=[DA.layout.grid[0], 1])
    with pytest.raises(dab.DimensionMismatch):
        dab.mul_(Cd, DA, np.zeros((31, 20)))
    with pytest.raises(dab.DimensionMismatch):
        dab.mul_(Cd, DA, np.zeros((30, 21)))
    bad = dab.dzeros((30, 20), procs=[1, 2, 3], dist=[3, 1])
    if list(bad.layout.cuts[0]) != list(DA.layout.cuts[0]):
        with pytest.raises(dab.ArgumentError):
            dab.mul_(bad, DA, B)


def test_matmatmul_float32_tensor_core_tiles(dab, rt2):
    """Chunks big and aligned enough for the wgmma path (2 workers -> 512 x 256 column blocks): 1e-6 relative on positive data."""
    rng = np.random.default_rng(59)
    A, B = rng.random((512, 512)).astype(np.float32), rng.random((512, 384)).astype(np.float32)
    DA, DB = dab.distribute(A), dab.distribute(B)
    want = A.astype(np.float64) @ B.astype(np.float64)
    got = dab.to_array(DA @ DB)
    assert got.dtype == np.float32 and float(np.abs(got - want).max() / np.abs(want).min()) <= 1e-6
    gt = dab.to_array(DA.T @ DB)
    wt = A.T.astype(np.float64) @ B.astype(np.float64)
    assert float(np.abs(gt - wt).max() / np.abs(wt).min()) <= 1e-6


@pytest.mark.parametrize("shape", [(100, 200), (200, 100), (7, 3), (1, 9), (64, 64), (257, 1031), (3, 1)])
def test_transpose_copy(dab, rt8, shape):
    """test/darray.jl:713-733: copy(transpose(A)) == transpose(Array(A)), copy(adjoint(A)) == adjoint(Array(A)) (real eltypes)."""
    rng = np.random.default_rng(43)
    for dtype in (np.float64, np.float32, np.int64, np.bool_):
        A = (rng.standard_normal(shape) * 100).astype(dtype)
        DA = dab.distribute(A)
        oT = orc.darray_transpose(orc.distribute(A, nworkers=8))
        for T in (dab.transpose(DA).copy(), dab.adjoint(DA).copy(), DA.T.copy()):
            assert T.dims == (shape[1], shape[0]) and T.layout.grid == tuple(oT.grid) and list(T.layout.indices) == oT.indices
            assert list(T.layout.pids) == oT.pids
            assert np.array_equal(dab.to_array(T), A.T)
            for pid, ch in T.chunks.items():
                assert np.array_equal(ch.to_numpy(), oT.chunks[oT.pids.index(pid)])
    # a non-default source layout (row blocks): each result chunk gathers pieces from several owners
    A = rng.standard_normal((130, 70))
    DA = dab.distribute(A, dist=(8, 1))
    assert np.array_equal(dab.to_array(DA.T.copy()), A.T)


def test_transpose_large(dab, rt2):
    m, n = 8192 + 3, 4096 + 5
    A = orc.rand_u01(11, 0, m * n).reshape((m, n), order="F")
    DA = dab.distribute(A)
    assert np.array_equal(dab.to_array(DA.T.copy()), A.T)


def test_diagonal_scaling(dab, rt8):
    """test/darray.jl:270-282: lmul!(D, DA) and rmul!(DA, D) equal the dense results exactly."""
    rng = np.random.default_rng(47)
    for dtype in (np.float64, np.float32):
        A = rng.standard_normal((100, 100)).astype(dtype)
        b = rng.standard_normal(100).astype(dtype)
        DA = dab.distribute(A)
        assert dab.lmul_diag(b, DA) is DA
        assert np.array_equal(dab.to_array(DA), b[:, None] * A)
        want = orc.darray_scale_diag(orc.distribute(A, nworkers=8), b, "l")
        for pid, ch in DA.chunks.items():
            assert np.array_equal(ch.to_numpy(), want.chunks[want.pids.index(pid)])
        DB = dab.distribute(A)
        dab.rmul_diag(DB, b)
        assert np.array_equal(dab.to_array(DB), A * b[None, :])
        with pytest.raises(dab.DimensionMismatch):
            dab.lmul_diag(b[:-1], DA)
