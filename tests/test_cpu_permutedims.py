"""CPU tier of ``permutedims`` (row f18): ``permute_plan`` against a NumPy model of Julia's ``permutedims``, the collapse rule and
the mover each piece gets, the public forms through the host-memory emulation of the C ABI (with tests/permute_hostmem.py), the
refusals, the GPU module run against that emulation, and the no-spill compile of dab_permute.cu."""
import itertools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import permute_hostmem

permute_hostmem.install()                                       # dab_permute_box for the host-memory emulation of the C ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128, np.float16]


def model(a, perm):
    """Julia's ``permutedims(A, perm)`` for a 1-based ``perm``."""
    return np.transpose(a, [p - 1 for p in perm])


def _values(T, shape, rng):
    T = np.dtype(T)
    n = int(np.prod(shape))
    if T == np.bool_:
        a = rng.random(n) > 0.5
    elif T.kind == "i":
        a = rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T)
    elif T.kind == "c":
        a = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(T)
    else:
        a = rng.standard_normal(n).astype(T)
        a[::7] = -0.0
        if n > 3:                                                # a NaN with a payload
            U = {2: np.uint16, 4: np.uint32, 8: np.uint64}[T.itemsize]
            a[3] = np.array({2: 0x7E05, 4: 0x7FC00123, 8: 0x7FF8000000000123}[T.itemsize], dtype=U).view(T)
    return a.reshape(shape, order="F")


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def run_plan(plan, src_layout, dst_layout, a):
    """Executes ``plan`` on host buffers (one flat array per chunk), element by element from each piece's offsets, strides and extents;
    returns the assembled destination and how often each destination element was written."""
    from darray_b200.layout import shape_of
    src = {c: np.asfortranarray(a[tuple(slice(r[0] - 1, r[1]) for r in I)]).ravel(order="F") for c, I in enumerate(src_layout.indices)}
    dst = {c: np.zeros(int(np.prod(shape_of(I))), dtype=a.dtype) for c, I in enumerate(dst_layout.indices)}
    hits = {c: np.zeros(v.size, dtype=np.int64) for c, v in dst.items()}
    for p in plan:
        do = np.zeros((), dtype=np.int64)
        so = np.zeros((), dtype=np.int64)
        for e, ds, ss in zip(p.extent, p.dst_strides, p.src_strides):
            do = do[..., None] + np.arange(e, dtype=np.int64) * ds
            so = so[..., None] + np.arange(e, dtype=np.int64) * ss
        do, so = do.reshape(-1) + p.dst_offset, so.reshape(-1) + p.src_offset
        dst[p.dst_chunk][do] = src[p.src_chunk][so]
        np.add.at(hits[p.dst_chunk], do, 1)
    out = np.zeros(dst_layout.dims, dtype=a.dtype, order="F")
    cover = np.zeros(dst_layout.dims, dtype=np.int64, order="F")
    for c, I in enumerate(dst_layout.indices):
        sl = tuple(slice(r[0] - 1, r[1]) for r in I)
        out[sl] = dst[c].reshape(shape_of(I), order="F")
        cover[sl] = hits[c].reshape(shape_of(I), order="F")
    return out, cover


def _random_dist(rng, dims, nw):
    """An irregular grid for up to nw workers (a dimension may be cut more ways than it is long: empty chunks)."""
    grid = [1] * len(dims)
    left = nw
    while left > 1:
        k = int(rng.integers(len(dims)))
        f = 2 if left % 2 == 0 else left
        grid[k] *= f
        left //= f
    return grid


def _plan_cases():
    rng = np.random.default_rng(18)
    cases = []
    for N in (3, 4):                                             # every permutation of 3 and 4 dims
        for perm in itertools.permutations(range(1, N + 1)):
            cases.append((tuple(int(v) for v in rng.integers(1, 6, N)), perm, int(rng.choice([1, 2, 8])), int(rng.integers(1 << 30))))
    for N in range(1, 9):                                        # random shapes of 1..8 dims
        for _ in range(4):
            dims = tuple(int(v) for v in rng.integers(1, {1: 40, 2: 12, 3: 7, 4: 5, 5: 4, 6: 3, 7: 3, 8: 2}[N] + 1, N))
            cases.append((dims, tuple(int(v) + 1 for v in rng.permutation(N)), int(rng.choice([1, 2, 8])), int(rng.integers(1 << 30))))
    return cases


@pytest.mark.parametrize("dims,perm,nw,seed", _plan_cases())
def test_plan_matches_the_model(dims, perm, nw, seed):
    """Source and destination in default, irregular and foreign layouts (empty chunks included) on 1, 2 and 8 workers: executing the
    plan writes every destination element exactly once and gives ``permutedims(A, perm)``; the plan is a pure function of the layouts
    (same plan twice) and every piece's extents multiply to the elements it moves."""
    from darray_b200._permute import permute_plan
    from darray_b200.layout import make_layout
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(dims)
    pd = tuple(dims[p - 1] for p in perm)
    pids = list(range(1, nw + 1))
    srcs = [make_layout(dims, pids), make_layout(dims, pids, _random_dist(rng, dims, nw))]
    dsts = [make_layout(pd, pids), make_layout(pd, list(reversed(pids)), _random_dist(rng, pd, nw))]
    for sl in srcs:
        for dl in dsts:
            plan = permute_plan(sl, dl, perm, 8)
            assert plan == permute_plan(sl, dl, perm, 8)
            out, cover = run_plan(plan, sl, dl, a)
            assert (cover == 1).all(), (sl.grid, dl.grid)
            _same(out, model(a, perm))
            for p in plan:
                assert len(p.extent) == len(p.dst_strides) == len(p.src_strides) and min(p.extent) >= 1
                small = len(p.extent) > 1 and 1 in p.src_strides[1:] and (p.extent[0] * p.extent[p.src_strides.index(1, 1)] < 512
                                                                           or min(p.extent[0], p.extent[p.src_strides.index(1, 1)]) < 2)
                assert p.mover == ("gather" if p.src_strides[0] == 1 or len(p.extent) == 1 or p.dst_strides[0] != 1 or 1 not in p.src_strides[1:]
                                   or small else "permute")


def test_collapse_rule_and_mover_selection():
    """Extent-1 dims go, destination-adjacent dims contiguous on both sides merge, and the mover is the gather exactly when the source's
    unit-stride dim is the destination's dim 0 after collapsing, a side has no unit stride, or the plane is below the measured size."""
    from darray_b200._permute import collapse, permute_plan, select_mover
    from darray_b200.layout import make_layout
    assert collapse((4, 1, 5), (1, 4, 4), (5, 20, 1)) == ((4, 5), (1, 4), (5, 1))
    assert collapse((3, 4, 5), (1, 3, 12), (1, 3, 12)) == ((60,), (1,), (1,))
    assert collapse((1, 1), (1, 1), (1, 3)) == ((1,), (1,), (1,))
    assert collapse((6, 7, 2), (1, 6, 42), (7, 1, 42)) == ((6, 7, 2), (1, 6, 42), (7, 1, 42))
    assert collapse((6, 7, 2), (1, 6, 42), (14, 1, 7)) == ((6, 14), (1, 6), (14, 1))       # dims 1, 2 merge on both sides
    assert select_mover((60,), (1,), (1,), 4) == "gather"
    assert select_mover((40, 30), (1, 40), (30, 1), 4) == "permute"
    assert select_mover((40, 30), (1, 40), (1, 40), 4) == "gather"
    assert select_mover((40, 30), (1, 40), (30, 3), 4) == "gather"                       # no unit stride in the source
    # the measured plane threshold: 1024 elements for 4-byte elements, 512 for 2- and 8-byte ones; sides of at least 16 bytes
    assert select_mover((32, 32, 99), (1, 32, 1024), (32, 1, 1024), 4) == "permute"
    assert select_mover((24, 24, 99), (1, 24, 576), (24, 1, 576), 4) == "gather"
    assert select_mover((24, 24, 99), (1, 24, 576), (24, 1, 576), 8) == "permute"
    assert select_mover((16, 16, 99), (1, 16, 256), (16, 1, 256), 8) == "gather"
    assert select_mover((8, 64, 99), (1, 8, 512), (64, 1, 512), 2) == "permute"
    assert select_mover((1024, 4, 99), (1, 1024, 4096), (4, 1, 4096), 4) == "permute"
    assert select_mover((1024, 4, 99), (1, 1024, 4096), (4, 1, 4096), 2) == "gather"

    def movers(dims, perm, es=4):
        L = make_layout(dims, [1])
        return [p.mover for p in permute_plan(L, make_layout(tuple(dims[p - 1] for p in perm), [1]), perm, es)]

    assert movers((50, 60, 7), (1, 3, 2)) == ["gather"]           # dim 1 stays in place: runs of 50
    assert movers((50, 60, 7), (2, 1, 3)) == ["permute"]
    assert movers((50, 60, 7), (3, 2, 1)) == ["gather"]           # a 7 x 60 plane: too small
    assert movers((50, 60, 70), (3, 2, 1)) == ["permute"]
    assert movers((10, 10, 1000), (2, 1, 3)) == ["gather"]        # the batched per-slice transpose of small slices
    assert movers((1, 60, 70), (2, 1, 3)) == ["gather"]           # the unit dim goes, nothing moves: one contiguous run
    assert movers((50, 1, 70), (3, 2, 1)) == ["permute"]
    p = permute_plan(make_layout((4, 5, 6), [1]), make_layout((5, 6, 4), [1]), (2, 3, 1), 4)[0]
    assert (p.extent, p.dst_strides, p.src_strides) == ((30, 4), (1, 30), (4, 1))          # (2, 3, 1) is a 2-D transpose of (4, 30)


def _launch_plan(dab, A, dims, perm):
    from darray_b200._permute import permute_plan
    B = dab.similar(A, dims=dims)
    n = len(permute_plan(A.layout, B.layout, perm, A.dtype.itemsize))
    B.close()
    return n


@pytest.mark.parametrize("T", ELTYPES)
def test_host_public_forms_every_element_type(hostmem, dab, T):
    """``permutedims`` of 3- to 6-d arrays in irregular layouts on 8 workers, ``permutedims_`` into a destination with another grid,
    ``permutedims(v)`` and ``permutedims(M)`` (= ``copy(transpose(M))``, the same launches): byte for byte against ``np.transpose``;
    the launch count equals the plan's piece count; nothing is left registered."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    rng = np.random.default_rng(np.dtype(T).itemsize * 7 + len(np.dtype(T).str))
    r0 = dab.registry_size()
    for dims, perm, dist in [((5, 6, 7), (3, 1, 2), [2, 1, 3]), ((4, 3, 5, 2), (2, 4, 1, 3), [1, 4, 1, 2]),
                             ((3, 2, 4, 2, 3), (5, 3, 1, 4, 2), None), ((2, 3, 2, 2, 3, 2), (6, 1, 5, 2, 4, 3), [1, 1, 2, 1, 2, 2])]:
        a = _values(T, dims, rng)
        A = dab.distribute(a, procs=list(range(1, 9)), dist=dist)
        l0 = hostmem.launches
        B = dab.permutedims(A, perm)
        assert hostmem.launches - l0 == _launch_plan(dab, A, B.dims, perm)
        _same(dab.to_array(B), model(a, perm))
        S = dab.similar(A, dims=B.dims)
        assert B.layout.same_as(S.layout)
        pd = B.dims
        D = dab.distribute(np.zeros(pd, dtype=T), procs=list(range(8, 0, -1))[:6], dist=[1] * (len(pd) - 1) + [min(6, pd[-1])])
        assert dab.permutedims_(D, A, list(np.array(perm))) is D
        _same(dab.to_array(D), model(a, perm))
        for x in (A, B, S, D):
            x.close()
    v = _values(T, (37,), rng)
    V = dab.distribute(v)
    R = dab.permutedims(V)
    assert R.dims == (1, 37)
    _same(dab.to_array(R), v.reshape(1, 37))
    m = _values(T, (13, 9), rng)
    M = dab.distribute(m, dist=[4, 2])
    l0 = hostmem.launches
    P = dab.permutedims(M)
    l1 = hostmem.launches
    Q = dab.copy_transposed(dab.transpose(M))
    assert l1 - l0 == hostmem.launches - l1
    _same(dab.to_array(P), m.T)
    _same(dab.to_array(P), dab.to_array(Q))
    _same(dab.to_array(dab.permutedims(M, (2, 1))), m.T)
    for x in (V, R, M, P, Q):
        x.close()
    assert dab.registry_size() == r0
    rt.shutdown()


def test_host_permutedims_matrix_into_a_foreign_layout_and_empty(hostmem, dab):
    """``permutedims_`` of a matrix into any layout, identity permutations, and empty arrays and chunks (no launch for those)."""
    rt = dab.init(workers_per_rank=3, use_dist=False)
    rng = np.random.default_rng(5)
    m = rng.standard_normal((7, 11))
    M = dab.distribute(m)
    D = dab.dzeros((11, 7), procs=[3, 1, 2], dist=[1, 3])
    _same(dab.to_array(dab.permutedims_(D, M, (2, 1))), m.T)
    a = rng.standard_normal((2, 4, 3))
    _same(dab.to_array(dab.permutedims(dab.distribute(a), (1, 2, 3))), a)
    E = dab.distribute(np.zeros((0, 3, 2)))
    l0 = hostmem.launches
    R = dab.permutedims(E, (3, 1, 2))
    assert R.dims == (2, 0, 3) and hostmem.launches == l0
    s = rng.standard_normal((2, 1, 2))
    small = dab.distribute(s, procs=[1, 2, 3], dist=[1, 1, 3])     # 2 x 1 x 2 cut 3 ways along dim 3, and into 3 along dim 1
    X = dab.dzeros((2, 1, 2), procs=[1, 2, 3], dist=[3, 1, 1])
    assert sum(1 for L in (small.layout, X.layout) for I in L.indices if any(r[1] < r[0] for r in I)) == 2
    l0 = hostmem.launches
    _same(dab.to_array(dab.permutedims_(X, small, (3, 2, 1))), model(s, (3, 2, 1)))
    from darray_b200._permute import permute_plan
    assert hostmem.launches - l0 == len(permute_plan(small.layout, X.layout, (3, 2, 1), 8)) == 2
    rt.shutdown()


def test_host_refusals_before_any_launch(hostmem, dab):
    """Every error of the contract is raised before any allocation or launch and leaves the registry as it was."""
    import scipy.sparse as sp
    rt = dab.init(workers_per_rank=4, use_dist=False)
    A = dab.distribute(np.arange(24.0).reshape(2, 3, 4))
    D = dab.dzeros((4, 2, 3))
    D32 = dab.dzeros((4, 2, 3), dtype=np.float32)
    D2 = dab.dzeros((4, 6))
    S = dab.distribute(sp.random(8, 8, density=0.3, format="csc", random_state=1))
    A9 = dab.distribute(np.zeros((1,) * 9))
    cases = [(dab.ArgumentError, "expected permutation of size 3, but length\\(perm\\)=2", lambda: dab.permutedims(A, (1, 2))),
             (dab.ArgumentError, "not a permutation", lambda: dab.permutedims(A, (1, 1, 2))),
             (dab.ArgumentError, "not a permutation", lambda: dab.permutedims(A, (0, 1, 2))),
             (dab.ArgumentError, "not a permutation", lambda: dab.permutedims(A, (1.0, 2, 3))),
             (dab.ArgumentError, "not a permutation", lambda: dab.permutedims(A, (True, 2, 3))),
             (dab.ArgumentError, "size 3", lambda: dab.permutedims_(D, A, (3, 1))),
             (dab.ArgumentError, "not a permutation", lambda: dab.permutedims_(D, A, (3, 3, 2))),
             (dab.DimensionMismatch, "destination tensor of incorrect size", lambda: dab.permutedims_(D, A, (1, 2, 3))),
             (dab.DimensionMismatch, "incorrect size", lambda: dab.permutedims_(D2, A, (3, 1, 2))),
             (dab.ArgumentError, "share storage", lambda: dab.permutedims_(A, A, (1, 2, 3))),
             (dab.UnsupportedError, "float32", lambda: dab.permutedims_(D32, A, (3, 1, 2))),
             (dab.UnsupportedError, "sparse", lambda: dab.permutedims(S, (2, 1))),
             (dab.UnsupportedError, "sparse", lambda: dab.permutedims_(D, S, (2, 1))),
             (dab.UnsupportedError, r"to_darray\(\)", lambda: dab.permutedims(A[0:2, :, :], (3, 1, 2))),
             (dab.UnsupportedError, r"to_darray\(\)", lambda: dab.permutedims_(D, A[:, :, :], (3, 1, 2))),
             (dab.UnsupportedError, "9 dimensions", lambda: dab.permutedims(A9, tuple(range(9, 0, -1)))),
             (TypeError, "MethodError", lambda: dab.permutedims(A))]
    for exc, msg, f in cases:
        n0, l0, r0 = len(hostmem.blocks), hostmem.launches, dab.registry_size()
        with pytest.raises(exc, match=msg):
            f()
        assert (len(hostmem.blocks), hostmem.launches, dab.registry_size()) == (n0, l0, r0), msg
    rt.shutdown()


def test_hostmem_model_refuses_what_the_kernel_refuses(hostmem, dab):
    """The emulation's preconditions are the kernel's: DAB_ERR_ARG without a launch."""
    import ctypes as C
    L = sys.modules["darray_b200._lib"]
    rt = dab.init(workers_per_rank=1, use_dist=False)
    buf = rt.alloc(4096)
    LL = C.c_longlong * 9

    def call(es, nd, ds, ss, ext):
        return L.call("dab_permute_box", rt.ctx, es, nd, C.c_void_p(buf), LL(*ds), C.c_void_p(buf + 2048), LL(*ss), (C.c_size_t * 9)(*ext))

    ok = ([1, 4] + [16] * 7, [4, 1] + [16] * 7, [4, 4] + [1] * 7)
    for es, nd, ds, ss, ext in [(3, 2) + ok, (4, 1) + ok, (4, 9) + ok, (4, 2, [2, 4] + [0] * 7, ok[1], ok[2]),
                                (4, 2, ok[0], [1, 4] + [0] * 7, ok[2]), (4, 3, [1, 4, 16] + [0] * 6, [4, 1, 1] + [0] * 6, [4, 4, 1] + [0] * 6)]:
        l0 = hostmem.launches
        with pytest.raises(dab.ArgumentError):
            call(es, nd, ds, ss, ext)
        assert hostmem.launches == l0
    l0 = hostmem.launches
    call(4, 2, ok[0], ok[1], [4, 0] + [1] * 7)
    assert hostmem.launches == l0
    rt.free(buf)
    rt.shutdown()


def test_gpu_permutedims_module_against_the_host_memory_abi():
    """tests/test_gpu_permutedims.py with the C ABI emulated over host memory: the host flow around K28 (plans, layouts, launch counts,
    refusal contracts) against the same models."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_permutedims.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 10, tail


def test_permute_instances_compile_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_permute.cu for sm_90a: all 9 instances (1 / 2 / 4 / 8-byte elements with 16-byte and one-element
    accesses, 16-byte elements) use no stack frame and spill nothing."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_permute.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) == 9 and all("permute_box_kernel" in e for e in entries), entries
    assert len(frames) == len(entries) and all(f == ("0", "0", "0") for f in frames), list(zip(entries, frames))
