"""CPU tier of findmax / findmin / argmax / argmin (K20): the model of Julia's loops (tests/findmax_oracle.py) against the literal sequential
loops, the host runtime over random 1-8 worker layouts through the host-memory emulation of the C ABI, the GPU module run against that
emulation, and the no-spill compile of dab_findminmax.cu."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import findmax_oracle as fo

fo.install()                                                    # dab_findminmax / _dim / dab_combine_findminmax for the emulated C ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _specials(rng, dtype, n):
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return rng.random(n) < 0.5
    if dt.kind == "f":
        pool = np.array([0.0, -0.0, 1.0, -1.0, 2.5, np.inf, -np.inf, np.nan, -np.nan], dtype=dt)
    else:
        info = np.iinfo(dt)
        pool = np.array([0, 1, -1, 7, info.min, info.max, info.min + 1], dtype=dt)
    return rng.choice(pool, n)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64, np.bool_])
def test_vectorised_model_is_the_sequential_loop(dtype):
    rng = np.random.default_rng(2)
    maps = [None] if np.dtype(dtype) == np.bool_ else [None, np.abs, lambda x: x * x]
    for trial in range(300):
        a = _specials(rng, dtype, int(rng.integers(1, 12)))
        for which in (fo.FINDMAX, fo.FINDMIN):
            for f in maps:
                v, i = fo.find(which, a, f)
                sv, si = fo.seq_find(which, a, f)
                assert i == si and fo.same_bits(np.asarray([v]), np.asarray([sv])), (which, a, v, i, sv, si)


def test_julia_rules_on_literal_cases():
    f32 = np.float32
    nan = np.float32(np.nan)
    assert fo.seq_find(fo.FINDMAX, np.array([1, nan, 3, nan], dtype=f32))[1] == 1             # NaN wins, the first one is kept
    assert fo.seq_find(fo.FINDMIN, np.array([1, nan, -3, nan], dtype=f32))[1] == 1
    assert fo.seq_find(fo.FINDMAX, np.array([-0.0, 0.0], dtype=f32))[1] == 1                   # findmax prefers +0.0
    assert fo.seq_find(fo.FINDMIN, np.array([0.0, -0.0], dtype=f32))[1] == 1                   # findmin prefers -0.0
    assert fo.seq_find(fo.FINDMAX, np.array([2, 5, 5], dtype=np.int32))[1] == 1                # ties keep the earlier index
    assert fo.seq_find(fo.FINDMAX, np.array([-2 ** 31, 3], dtype=np.int32), np.abs)[1] == 1    # abs(typemin) == typemin wraps


def test_dims_model_is_the_sequential_loop_per_slice():
    rng = np.random.default_rng(4)
    A = _specials(rng, np.float64, 4 * 5 * 3).reshape((4, 5, 3), order="F")
    for dims in (1, 2, 3, (1, 3), (2, 3), (1, 2, 3), 4):
        for which in (fo.FINDMAX, fo.FINDMIN):
            v, i = fo.find_dims(which, A, dims)
            ds = {dims} if isinstance(dims, int) else set(dims)
            for out in np.ndindex(*v.shape):
                sel = tuple(slice(None) if k + 1 in ds else slice(out[k], out[k] + 1) for k in range(3))
                g = np.arange(A.size).reshape(A.shape, order="F")[sel].ravel(order="F")
                sv, si = fo.seq_find(which, A[sel])
                assert fo.same_bits(np.asarray([v[out]]), np.asarray([sv])) and i[out] == g[si] + 1, (dims, out)


def test_host_runtime_on_random_layouts(hostmem, dab):
    """The whole-array and dims forms through the real host runtime (chunk results made global, the fold, plan_reducedim, the slab
    exchange with indices) on random 1-8 worker layouts, against the model."""
    rng = np.random.default_rng(9)
    dab.init(workers_per_rank=8, use_dist=False)
    done = 0
    for trial in range(60):
        shape = tuple(int(s) for s in rng.integers(1, 9, int(rng.integers(1, 4))))
        nw = int(rng.integers(1, 9))
        procs = [int(p) for p in rng.permutation(np.arange(1, 9))[:nw]]
        dtype = [np.float32, np.float64, np.int32, np.int64, np.bool_][trial % 5]
        A = _specials(rng, dtype, int(np.prod(shape))).reshape(shape, order="F")
        try:
            d = dab.distribute(A, procs=procs)
        except (dab.ArgumentError, ValueError):
            continue
        for which, fn in ((fo.FINDMAX, dab.findmax), (fo.FINDMIN, dab.findmin)):
            v, i = fn(d)
            wv, wi = fo.find(which, A)
            assert fo.same_bits(np.asarray([v]), np.asarray([wv])) and i == fo.julia_index(shape, wi), (shape, procs, which)
            dims = tuple(sorted(set(int(k) for k in rng.integers(1, len(shape) + 2, int(rng.integers(1, 3))))))
            V, I = fn(d, dims=dims)
            wv, wi = fo.find_dims(which, A, dims)
            assert fo.same_bits(dab.to_array(V), wv) and np.array_equal(dab.to_array(I), wi), (shape, procs, dims, which)
            V.close()
            I.close()
        d.close()
        done += 1
    assert done >= 30


def test_index_geometry_merges_whole_dims_and_maps_positions_exactly():
    """The (chunk dims, offsets, global dims) handed to dab_findminmax_dim, with whole lower dims merged, give every chunk position its
    global linear index; a layout cut along more than 8 groups of dims is refused before anything runs."""
    from darray_b200 import _findmax
    from darray_b200.layout import make_layout, shape_of
    rng = np.random.default_rng(21)
    for trial in range(200):
        N = int(rng.integers(1, 10))
        dims = tuple(int(s) for s in rng.integers(1, 5, N))
        grid = tuple(int(rng.integers(1, min(s, 2) + 1)) for s in dims)
        L = make_layout(dims, list(range(1, int(np.prod(grid)) + 1)), grid)
        for pid in L.pids:
            cd, off, gd = _findmax._index_geometry(L, pid)
            assert int(np.prod(gd)) == int(np.prod(dims)) and len(cd) <= 1 + sum(g > 1 for g in grid)
            shape = shape_of(L.localindices(pid))
            n = int(np.prod(shape))
            for pos in rng.integers(0, n, min(n, 5)):
                c = np.unravel_index(int(pos), cd, order="F")
                g = int(np.ravel_multi_index(tuple(int(a) + o for a, o in zip(c, off)), gd, order="F"))
                assert g == _findmax._global0(L, pid, int(pos)), (dims, grid, pid, pos)
    L9 = make_layout((2,) * 9, list(range(1, 513)), (2,) * 9)
    with pytest.raises(_findmax._lib.UnsupportedError, match="more than 8"):
        _findmax._check_index_geometry(L9)
    _findmax._check_index_geometry(make_layout((2,) * 9, list(range(1, 257)), (1,) + (2,) * 8))   # a whole first dim merges: 8 groups


def test_gpu_findmax_module_against_the_host_memory_abi():
    """tests/test_gpu_findmax.py with the C ABI emulated over host memory: the host runtime around K20 (layouts, the global indices, the
    slab exchange, views, the refusals and their launch contract) against the same model."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_findmax.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 30, tail


def test_gpu_findmax_paths_module_against_the_host_memory_abi():
    """tests/test_gpu_findmax_paths.py with the C ABI emulated over host memory: its case designs, premises, guard bands and refusal
    statuses against the same model (the 2 GiB cases skip)."""
    env = dict(os.environ, DAB_HOSTMEM="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_findmax_paths.py", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 130, tail


@pytest.mark.parametrize("sm_count", [132, 114, 16, fo.MIN_SM_COUNT])
def test_case_table_reaches_every_label_from_the_minimum_sm_count(sm_count):
    """The launch model reaches every label from the case table of tests/test_gpu_findmax_paths.py at the SM counts of the H100 SXM (132)
    and PCIe (114), of a 16-SM partition and at the table's minimum; each case reaches the label it is named for, and Bool never takes the
    16-byte kernel."""
    seen = set()
    for case in fo.case_table(sm_count):
        for dt in (np.float32, np.float64, np.int32, np.int64, np.bool_):
            labels = fo.case_labels(case, dt, sm_count)
            want = "bool_vec_shape" if dt == np.bool_ and case[1] in ("vec", "vec_split") else case[1]
            assert want in labels, (case[0], np.dtype(dt).name, labels)
            assert dt != np.bool_ or not any(l.startswith("vec") for l in labels)
            seen |= labels
    assert seen == fo.ALL_LABELS, fo.ALL_LABELS ^ seen


def test_no_pass_leaves_a_split_empty_below_the_minimum_sm_count():
    """Below fo.MIN_SM_COUNT SMs a pass gets at most 256 splits of at least 256 elements, so none is empty: the case table refuses to be
    built there, rather than claim a label it cannot reach."""
    sm = fo.MIN_SM_COUNT - 1
    with pytest.raises(ValueError):
        fo.case_table(sm)
    for inner in (1, 2, 5, 300):
        for red in list(range(256, 256 * 300, 37)) + [256 * 256 + k for k in range(-3, 4)]:
            assert not fo.fmdim_plan(np.float32, inner, red, 1, 0, False, sm)["empty"], (inner, red)
    assert fo.fmdim_plan(np.float32, 2, 256 * 288 + 1, 1, 0, False, fo.MIN_SM_COUNT)["empty"]


def test_launch_model_on_literal_plans():
    """fmdim_plan on hand-worked plans: the split count and bounds, an empty split, the launch count and the grid that loops."""
    p = fo.fmdim_plan(np.float32, 2, 306200, 1, 0, False, 132)        # 1024 splits of 300: the last three are empty
    assert p["kernel"] == "strided" and p["nsplit"] == 1024 and p["bounds"][1020] == (306000, 306200) and p["empty"]
    assert [hi <= lo for lo, hi in p["bounds"]].count(True) == 3 and p["launches"] == 2
    p = fo.fmdim_plan(np.float32, 1, 12293, 3, 0, False, 132)          # lead32: 6 splits of 2049, the last 2048
    assert (p["kernel"], p["G"], p["nsplit"], p["bounds"][-1]) == ("lead", 32, 6, (10245, 12293))
    assert fo.fmdim_plan(np.float32, 1, 65536, 1, 0, False, 132)["launches"] == 2
    assert fo.fmdim_plan(np.float32, 1, 65536, 1, 0, True, 132)["kernel"] == "lead"   # never the whole-chunk kernel with an index input
    assert fo.fmdim_plan(np.float64, 16384, 3, 1, 0, False, 132)["vec"]
    assert not fo.fmdim_plan(np.float64, 16384, 3, 1, 8, False, 132)["vec"]          # one element off 16 bytes
    assert fo.fmdim_plan(np.int32, 1, 5, 132 * 8 * 64 + 1, 0, False, 132)["loops"]
    assert not fo.fmdim_plan(np.int32, 1, 5, 132 * 8 * 64, 0, False, 132)["loops"]
    g = fo.flat_grid(np.float32, 8, 2 + 3 * 4096 + 5 * 4 + 3)
    assert (g["head"], g["tiles"], g["grid"], g["tiles_per_cta"], g["rem_vecs"], g["tail"]) == (2, 3, 2, 2, 5, 3)


def test_emulated_index_input_pass_is_the_sequential_loop():
    """The emulated dab_findminmax_dim with an index input (a later pass, or the fold on the owner) against ``seq_find`` over the whole
    original run: the earlier pass's (value, 1-based index) of random groups of positions, in random order, with "no element" entries (-1)
    mixed in, for every dtype and both functions."""
    import ctypes as C
    import hostmem_abi as hm
    rng = np.random.default_rng(31)
    emu = hm.HostMemABI()
    codes = {np.float32: hm.F32, np.float64: hm.F64, np.int32: hm.I32, np.int64: hm.I64, np.bool_: hm.U8}
    for trial in range(300):
        dtype = list(codes)[trial % 5]
        which = (fo.FINDMAX, fo.FINDMIN)[(trial // 5) % 2]
        inner, n = int(rng.integers(1, 4)), int(rng.integers(1, 30))
        ngroups = int(rng.integers(1, n + 1))
        red = ngroups + int(rng.integers(0, 3))
        X = np.empty((inner, red, 1), dtype=dtype)
        II = np.full((inner, red, 1), -1, dtype=np.int64)
        wants = []
        for i in range(inner):
            A = _specials(rng, dtype, n)
            g = rng.integers(0, ngroups, n)
            g[:ngroups] = np.arange(ngroups)                     # no group is empty
            slots = rng.permutation(red)[:ngroups]               # the pass's entries in an order of their own; the rest are -1
            X[i, :, 0] = A[0]
            for k in range(ngroups):
                members = np.nonzero(g == k)[0]
                v, j = fo.seq_find(which, A[members])
                X[i, slots[k], 0], II[i, slots[k], 0] = v, members[j] + 1
            wants.append(fo.seq_find(which, A))
        ov, oi = np.zeros(inner, dtype=dtype), np.zeros(inner, dtype=np.int64)
        vp = lambda a: C.c_void_p(a.ctypes.data)
        xs, iis = np.asfortranarray(X), np.asfortranarray(II)
        st = fo.dab_findminmax_dim(emu, None, codes[dtype], which, 0, vp(xs), vp(iis), inner, red, 1, 0, None, None, None, vp(ov), vp(oi))
        assert st == 0
        for i, (v, j) in enumerate(wants):
            assert fo.same_bits(ov[i:i + 1], np.asarray([v])) and oi[i] == j + 1, (trial, i, ov[i], oi[i], v, j)


def test_dab_findminmax_compiles_without_stack_or_spills():
    """``nvcc -Xptxas -v`` of dab_findminmax.cu for sm_90a: no entry function uses a stack frame or spills."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_findminmax.cu")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "-Xptxas", "-v", "-c", src, "-o",
                        os.devnull], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(entries) >= 100 and len(frames) >= len(entries), r.stderr[-2000:]
    assert all(f == ("0", "0", "0") for f in frames), [e for e, f in zip(entries, frames) if f != ("0", "0", "0")]
