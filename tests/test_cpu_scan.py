"""CPU tier of the scans (``cumsum`` / ``cumprod`` / ``accumulate`` and their ``!`` forms): the result-type table, every error, the
``dims > ndims`` / ``init`` quirk and empty inputs, the host runtime's whole flow over the host-memory emulation of the C ABI
(tests/scan_oracle.py) for layouts on 1 to 8 workers, the scan kernels compiled for sm_90a without spills, and the carry plan checked
pairwise and executed over gloo on two ranks."""
import os
import re
import shutil
import socket
import subprocess
import sys
import traceback

import numpy as np
import pytest

import scan_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = (np.float32, np.float64, np.int32, np.int64, np.bool_)


# ---- the model ------------------------------------------------------------------------------------------------------------------------


def test_model_result_types_and_reduce_first():
    """The issue's table, and Julia's fold on hand-worked cases."""
    table = {np.float32: ("f4",) * 5, np.float64: ("f8",) * 5, np.int32: ("i8", "i8", "i4", "i4", "i4"), np.int64: ("i8",) * 5,
             np.bool_: ("i8", "?", "i8", "?", "?")}
    for dt, want in table.items():
        got = (so.result_type(dt, "+", True), so.result_type(dt, "*", True), so.result_type(dt, "+", False), so.result_type(dt, "*", False),
               so.result_type(dt, "max", False))
        assert tuple(g.str[1:] if g != np.dtype(bool) else "?" for g in got) == want, dt
    assert so.jl_accumulate("+", np.array([-0.0, -0.0]), 1).tolist() == [-0.0, -0.0] and np.signbit(so.jl_accumulate("+", np.array([-0.0]), 1))[0]
    assert np.signbit(so.jl_accumulate("+", np.array([-0.0]), 1, init=0.0))[0] == False  # noqa: E712 -- op(init, x1) = 0.0 + -0.0
    assert so.jl_accumulate("+", np.array([2 ** 31 - 1, 1], dtype=np.int32), 1).tolist() == [2 ** 31 - 1, -2 ** 31]
    assert so.jl_accumulate("+", np.array([2 ** 31 - 1, 1], dtype=np.int32), 1, cum=True).tolist() == [2 ** 31 - 1, 2 ** 31]
    assert so.jl_accumulate("+", np.array([True, True]), 1).tolist() == [1, 2]
    assert so.jl_accumulate("*", np.array([True, False, True]), 1).tolist() == [True, False, False]
    mx = so.jl_accumulate("max", np.array([-0.0, 0.0, -1.0, np.nan, 5.0]), 1)
    assert not np.signbit(mx[1]) and mx[2] == 0.0 and np.isnan(mx[3]) and np.isnan(mx[4])
    assert np.signbit(so.jl_accumulate("min", np.array([0.0, -0.0, 0.0]), 1)[2])
    assert np.isinf(so.jl_accumulate("+", np.array([3e38, 3e38, -3e38], dtype=np.float32), 1)[2])      # Julia's Float32 fold stays Inf


# ---- host flow over the emulation -----------------------------------------------------------------------------------------------------


@pytest.fixture()
def scan_rt(hostmem, dab, request):
    so.install_hostmem(hostmem)
    return lambda wpr: dab.init(workers_per_rank=wpr, use_dist=False)


def _data(dt, shape, rng):
    if dt == np.bool_:
        return rng.random(shape) < 0.5
    if np.dtype(dt).kind == "i":
        return rng.integers(-50, 50, shape).astype(dt)
    return (rng.integers(-8, 9, shape) * 2.0 ** -10).astype(dt)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


@pytest.mark.parametrize("wpr", [1, 2, 3, 8])
def test_host_flow_layouts(scan_rt, dab, wpr):
    rt = scan_rt(wpr)
    rng = np.random.default_rng(wpr)
    pids = dab.workers()
    P = len(pids)
    for shape in [(37,), (13, 11), (5, 6, 7)]:
        for dt in DTYPES:
            A = _data(dt, shape, rng)
            dists = [None] + [g for g in ([1] * (len(shape) - 1) + [P], [P] + [1] * (len(shape) - 1))
                              if len(shape) > 1 and P > 1 and all(e >= n for e, n in zip(shape, g))]
            for dist in dists:
                d = dab.distribute(A, procs=pids, dist=dist)
                for dims in range(1, len(shape) + 2):
                    for fn, op in ((dab.cumsum, "+"), (dab.cumprod, "*")):
                        r = fn(d, dims=dims)
                        assert _same(dab.to_array(r), so.jl_accumulate(op, A, dims, cum=True)), (wpr, shape, dt, dist, dims, op)
                        assert r.layout.same_as(dab.similar(d, r.dtype).layout)
                        r.close()
                    for op in ("max", "min", "+", "*"):
                        init = 1 if op in ("+", "*") else None
                        r = dab.accumulate(op, d, dims=dims, init=init)
                        want = so.jl_accumulate(op, A, dims, init=init if dims <= len(shape) else None)
                        assert _same(dab.to_array(r), want), (wpr, shape, dt, dist, dims, op)
                        r.close()
                d.close()
    assert rt.launches() > 0


def test_host_flow_inplace_other_layout_views(scan_rt, dab):
    scan_rt(8)
    rng = np.random.default_rng(5)
    A = _data(np.float64, (24, 10), rng)
    d = dab.distribute(A, procs=dab.workers(), dist=[4, 2])
    dab.cumsum_(d, d, dims=1)                                     # dest is src, dims split over 4 workers
    assert _same(dab.to_array(d), so.jl_accumulate("+", A, 1, cum=True))
    src = dab.distribute(A, procs=dab.workers(), dist=[8, 1])
    dest = dab.distribute(np.zeros((24, 10)), procs=dab.workers(), dist=[1, 8])   # dest's own layout, src read through the halo path
    dab.accumulate_("max", dest, src, dims=2)
    assert _same(dab.to_array(dest), so.jl_accumulate("max", A, 2))
    assert dest.layout.grid == (1, 8)
    v = src[3:20, 2:9]                                            # SubDArray source
    assert _same(dab.to_array(dab.cumsum(v, dims=1)), so.jl_accumulate("+", A[3:20, 2:9], 1, cum=True))
    I = dab.distribute(_data(np.int32, (24, 10), rng), procs=dab.workers(), dist=[8, 1])
    out = dab.similar(I, np.int64)
    dab.cumprod_(out, I, dims=1)
    assert _same(dab.to_array(out), so.jl_accumulate("*", dab.to_array(I), 1, cum=True))


def test_init_and_dims_beyond_ndims(scan_rt, dab):
    """init is op(init, x1); dims > ndims is copyto!(B, A) and ignores init, even one that could not be represented."""
    scan_rt(2)
    A = np.array([1.5, 2.0, -3.0], dtype=np.float32)
    d = dab.distribute(A)
    assert _same(dab.to_array(dab.accumulate("+", d, init=2)), np.array([3.5, 5.5, 2.5], dtype=np.float32))
    assert _same(dab.to_array(dab.accumulate("max", d, init=1.75)), np.array([1.75, 2.0, 2.0], dtype=np.float32))
    assert _same(dab.to_array(dab.accumulate("+", d, dims=2, init=0.1)), A)
    B = dab.distribute(np.array([True, False, True]))
    assert _same(dab.to_array(dab.cumsum(B, dims=2)), np.array([1, 0, 1]))
    assert _same(dab.to_array(dab.accumulate("*", B, dims=3, init=7)), np.array([True, False, True]))
    with pytest.raises(dab.UnsupportedError, match="init=0.1"):
        dab.accumulate("+", d, init=0.1)
    with pytest.raises(dab.UnsupportedError, match="init=2"):
        dab.accumulate("max", B, init=2)
    with pytest.raises(dab.UnsupportedError, match="init"):
        dab.accumulate("+", dab.distribute(np.array([1], dtype=np.int32)), init=2 ** 31)


def test_empty_inputs(scan_rt, dab):
    scan_rt(3)
    for shape, dims in (((4, 0), 1), ((0, 5), 2), ((3, 0, 2), 3), ((3, 0, 2), 1)):
        d = dab.distribute(np.zeros(shape, dtype=np.int32))
        r = dab.cumsum(d, dims=dims)
        assert r.dims == shape and r.dtype == np.dtype(np.int64)
        dab.cumsum_(r, d, dims=dims)


def test_errors(scan_rt, dab):
    rt = scan_rt(2)
    d = dab.distribute(np.ones((4, 3), dtype=np.float32))
    v = dab.distribute(np.ones(6, dtype=np.float32))
    n0 = rt.launches()
    reg = dab.registry_size()
    cases = [
        (lambda: dab.cumsum(d, dims=0), dab.ArgumentError, "dims must be a positive integer"),
        (lambda: dab.accumulate("+", d, dims=-1), dab.ArgumentError, "dims must be a positive integer"),
        (lambda: dab.cumsum(d), TypeError, "UndefKeywordError: keyword argument `dims` not assigned"),
        (lambda: dab.cumprod(d), TypeError, "UndefKeywordError"),
        (lambda: dab.cumsum_(dab.similar(d), d), TypeError, "UndefKeywordError"),
        (lambda: dab.accumulate("+", d), dab.UnsupportedError, "without dims"),
        (lambda: dab.accumulate_("+", dab.similar(d), d), dab.ArgumentError, "dims must be provided"),
        (lambda: dab.cumsum_(v, d, dims=1), dab.DimensionMismatch, "shape of B must match A"),
        (lambda: dab.cumsum_(dab.similar(d, np.float64), d, dims=1), dab.UnsupportedError, "destination"),
        (lambda: dab.accumulate(lambda a, b: a - b, v), dab.UnsupportedError, "not served"),
        (lambda: dab.accumulate("-", v), dab.UnsupportedError, "not served"),
        (lambda: dab.cumsum(dab.distribute(np.ones(3, dtype=np.complex64))), dab.UnsupportedError, "complex64"),
        (lambda: dab.cumsum(v, dims=0), dab.ArgumentError, "positive"),
    ]
    for call, exc, text in cases:
        with pytest.raises(exc, match=re.escape(text)):
            call()
    assert rt.launches() == n0
    dab.d_closeall()
    assert dab.registry_size() <= reg


def test_op_vocabulary(scan_rt, dab):
    import builtins
    import operator
    scan_rt(1)
    v = dab.distribute(np.array([3, -1, 4, 1], dtype=np.int64))
    for op, want in ((operator.add, [3, 2, 6, 7]), (np.multiply, [3, -3, -12, -12]), (builtins.max, [3, 3, 4, 4]), (np.minimum, [3, -1, -1, -1]),
                     ("min", [3, -1, -1, -1])):
        assert dab.to_array(dab.accumulate(op, v)).tolist() == want


# ---- the kernels compile without spills -----------------------------------------------------------------------------------------------


def test_scan_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "distributedarrays.jl_b200", "csrc", "dab_scan.cu")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "-Xptxas", "-v",
                          "--expt-relaxed-constexpr", "-c", src, "-o", str(tmp_path / "s.o")], capture_output=True, text=True, check=True)
    log = out.stderr
    assert log.count("Compiling entry function") >= 80
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert props and all(p == ("0", "0", "0") for p in props)


# ---- the carry plan over gloo ---------------------------------------------------------------------------------------------------------


def test_carry_plan_pure_and_pairwise():
    import darray_b200 as dab
    from darray_b200._mapreduce import exchange_plan
    from darray_b200._scan import carry_plan
    L = dab.make_layout((12, 10, 6), list(range(1, 9)), [2, 2, 2])
    f = carry_plan(L, 2)
    assert f[0] == [] and f[2] == [0] and f[3] == [1] and f[6] == [4]
    f3 = carry_plan(L, 3)
    assert f3[4] == [0] and f3[7] == [3]
    for wpr in (1, 2, 4):
        plans = [exchange_plan(L, L, f, lambda p: (p - 1) // wpr, r) for r in range(8 // wpr)]
        for r, xp in enumerate(plans):
            for peer, other in enumerate(plans):
                if peer != r:
                    assert [(mp, rl) for mp, dst, rl in xp["sends"] if dst == peer] == [(mp, rl) for rl, s, mp, src in other["recvs"] if src == r]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, wpr, q):
    """Every rank holds its own workers' chunk totals (from the model); executing the plan over gloo and folding each stack in grid order
    must give every chunk the carry of the whole array's scan at its first row."""
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import torch
        import torch.distributed as dist

        import darray_b200 as dab
        import scan_oracle as so_
        from darray_b200._mapreduce import exchange_plan
        from darray_b200._scan import carry_plan
        from darray_b200.layout import shape_of

        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
        P = world * wpr
        rank_of = lambda pid: (pid - 1) // wpr                    # noqa: E731
        rng = np.random.default_rng(11)
        for shape, grid, dims in (((16, 9), (P, 1), 1), ((6, 20), (1, P), 2), ((8, 6, 4), (2, 1, P // 2), 3), ((8, 6, 4), (2, 1, P // 2), 1)):
            A = rng.integers(-9, 9, shape).astype(np.int64)
            L = dab.make_layout(shape, list(range(1, P + 1)), list(grid))
            k = dims - 1
            fib = carry_plan(L, dims)
            xp = exchange_plan(L, L, fib, rank_of, rank)
            chunk = lambda rl: A[tuple(slice(lo - 1, hi) for lo, hi in L.indices[rl])]   # noqa: E731
            mine = {L.pids[rl]: chunk(rl).sum(axis=k).ravel(order="F") for rl in range(len(L.pids)) if rank_of(L.pids[rl]) == rank}
            stacks = {rl: [None] * len(fib[rl]) for rl in xp["owned"]}
            for rl, slot, mp in xp["local"]:
                stacks[rl][slot] = mine[mp]
            reqs = [dist.isend(torch.from_numpy(np.ascontiguousarray(mine[mp])), dst) for mp, dst, rl in xp["sends"]]
            for rl, slot, mp, src in xp["recvs"]:
                buf = torch.empty(mine_len := int(np.prod([s for j, s in enumerate(shape_of(L.indices[rl])) if j != k])), dtype=torch.int64)
                dist.recv(buf, src)
                stacks[rl][slot] = buf.numpy().copy()
                del mine_len
            for r in reqs:
                r.wait()
            full = so_.jl_accumulate("+", A, dims, cum=True)
            for rl, parts in stacks.items():
                lo = L.indices[rl][k][0]
                if not parts:
                    continue
                carry = np.sum(parts, axis=0)
                idx = [slice(a - 1, b) for a, b in L.indices[rl]]
                idx[k] = slice(lo - 2, lo - 1)                     # the row before the chunk: the carry it must start from
                assert np.array_equal(carry, full[tuple(idx)].ravel(order="F")), (shape, grid, dims, rl)
            dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:
        q.put((rank, traceback.format_exc()))


@pytest.mark.parametrize("wpr", [1, 2])
def test_world2_carry_plan_over_gloo(wpr):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, wpr, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    for rank, msg in results:
        assert msg == "ok", f"rank {rank}:\n{msg}"
