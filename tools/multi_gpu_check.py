#!/usr/bin/env python
"""Multi-GPU parity + bandwidth check, one process per GPU:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29517 tools/multi_gpu_check.py

Checks, against the CPU oracle regenerated on every rank: sum / maximum with the NCCL all-gather + ordered left fold,
mapreducedim with the grouped send/recv between-phase, findmax / findmin with dims and cumsum / accumulate along a dim cut
across ranks, sort and sortperm of a DVector, one-sided halo reads over CUDA IPC peer mappings, broadcast across mismatched layouts; then times the C5 halo
read (256 MiB slab from the next rank) and prints one JSON line per metric (rank 0).
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402
from oracle import darray_oracle as orc  # noqa: E402

F32 = np.float32


def main():
    rt = dab.init(workers_per_rank=1)
    P, r = rt.world, rt.rank
    assert P >= 2, "run under torchrun with >= 2 ranks"
    log = (lambda *a: print(*a, flush=True)) if r == 0 else (lambda *a: None)

    # ---- C3-style: 1-D Float32, sum / maximum / minimum with the cross-worker combine
    n = (1 << 20) + 7
    N = n * P + 3
    x = dab.drand((N,), dtype=F32, seed=99)
    hx = orc.rand_u01(99, 0, N)
    od = orc.distribute(hx, nworkers=P)
    assert x.indices == od.indices and x.layout.grid == tuple(od.grid) == (P,)
    s, parts = dab.mapreduce(None, "+", x, _partials=True)
    fold = parts[0]
    for p in parts[1:]:
        fold = F32(fold + p)
    exact = orc.rand_u01_ksum(99, 0, N) * 2.0 ** -24
    ref, _ = orc.darray_mapreduce(None, "+", od)
    assert s == fold and abs(float(s) - exact) <= 1e-6 * exact and abs(float(s) - float(ref)) <= 1e-6 * exact, (s, fold, exact, ref)
    s2 = dab.sum(x)  # fused single-call path (dab_mapreduce_all)
    assert s2 == s, (s2, s)
    assert dab.maximum(x) == hx.max() and dab.minimum(x) == hx.min()
    assert dab.count(x, lambda v: v > 0.5) == int((hx > 0.5).sum())
    y = dab.similar(x)
    dab.broadcast_into(y, lambda v: F32(1.5) * v + F32(0.25), x)
    assert np.array_equal(dab.to_array(y), F32(1.5) * hx + F32(0.25))
    log("ok: 1-D sum/max/min/count/broadcast on", P, "GPUs; sum =", float(s), "exact =", exact)

    # ---- C4-style: 2-D, mapreducedim over every region, default grid
    R, Cc = 96, 40 * P
    A = orc.rand_u01(5, 0, R * Cc).reshape((R, Cc), order="F")
    dA = dab.distribute(A)
    oA = orc.distribute(A, nworkers=P)
    assert dA.layout.grid == tuple(oA.grid) and dA.indices == oA.indices
    A64 = A.astype(np.float64)
    for dims, ax in ((1, 0), (2, 1), ((1, 2), (0, 1))):
        Rd = dab.sum(dA, dims=dims)
        oR = orc.darray_mapreducedim(None, "+", oA, (dims,) if isinstance(dims, int) else dims)
        assert Rd.layout.pids == oR.pids and Rd.indices == oR.indices
        got = dab.to_array(Rd)
        assert np.allclose(got, A64.sum(axis=ax, keepdims=True), rtol=1e-6) and np.allclose(got, orc.to_array(oR), rtol=1e-6)
        assert np.array_equal(dab.to_array(dab.maximum(dA, dims=dims)), A.max(axis=ax, keepdims=True))
    for grid in ((P, 1), (1, P)):
        dB = dab.distribute(A, dist=grid)
        for dims, ax in ((1, 0), (2, 1)):
            assert np.allclose(dab.to_array(dab.sum(dB, dims=dims)), A64.sum(axis=ax, keepdims=True), rtol=1e-6)
    Ai = (A * 1000).astype(np.int64)
    dI = dab.distribute(Ai, dist=(P, 1))
    assert np.array_equal(dab.to_array(dab.mapreduce(lambda t: t * t, "+", dI, dims=1)), (Ai * Ai).sum(axis=0, keepdims=True))
    log("ok: mapreducedim with cross-rank between-phase")

    # ---- findmax / findmin with dims, and scans, along a dim cut across ranks: (value, index) slabs and scan carries travel between ranks
    rows, cols = np.indices(A.shape)
    lin = rows + cols * R + 1                                           # Julia's 1-based column-major linear index
    for grid in ((P, 1), (1, P)):
        dB, dI = dab.distribute(A, dist=grid), dab.distribute(Ai, dist=grid)
        for dims, ax in ((1, 0), (2, 1)):
            for find, arg in ((dab.findmax, np.argmax), (dab.findmin, np.argmin)):     # NumPy's first index of the extreme is Julia's
                v, i = find(dB, dims=dims)
                k = np.expand_dims(arg(A, axis=ax), ax)
                assert np.array_equal(dab.to_array(v), np.take_along_axis(A, k, ax)), (grid, dims)
                assert np.array_equal(dab.to_array(i), np.take_along_axis(lin, k, ax)), (grid, dims)
            assert np.array_equal(dab.to_array(dab.cumsum(dI, dims=dims)), np.cumsum(Ai, axis=ax)), (grid, dims)
            assert np.allclose(dab.to_array(dab.cumsum(dB, dims=dims)), np.cumsum(A64, axis=ax), rtol=1e-6), (grid, dims)
            got = dab.to_array(dab.accumulate("max", dB, dims=dims, init=F32(0.25)))
            assert np.array_equal(got, np.maximum(np.maximum.accumulate(A, axis=ax), F32(0.25))), (grid, dims)
    log("ok: findmax / findmin with dims, cumsum and accumulate along dims cut across ranks")

    # ---- halo reads: one-sided peer loads over CUDA IPC
    dA.share()
    x.share()
    rt.barrier()
    assert np.array_equal(np.asarray(dA[3:90, 5:Cc - 3]), A[3:90, 5:Cc - 3])
    nxt = (r + 1) % P
    lo, hi = x.indices[nxt][0]
    assert np.array_equal(np.asarray(x[lo - 1 + 11:lo - 1 + 11 + 5000]), hx[lo - 1 + 11:lo - 1 + 11 + 5000])
    assert np.array_equal(np.asarray(x[lo - 1 - 100:lo - 1 + 100]), hx[lo - 1 - 100:lo - 1 + 100])   # spans two owners
    # broadcast with mismatched layouts -> makelocal halo fetch inside the broadcast
    dB = dab.distribute(A, dist=(P, 1))
    dC = dab.distribute(A, dist=(1, P))
    Z = dab.broadcast(lambda u, v: u * v + 1, dB, dC)
    # the sources are overwritten right after the op returns: the op's trailing fence guarantees that no other rank's one-sided
    # copy kernel is still reading them (a missing fence shows up as NaNs in Z)
    dab.fill_(dB, np.nan)
    dab.fill_(dC, np.nan)
    assert np.array_equal(dab.to_array(Z), A * A + 1)
    dD = dab.distribute(A, dist=(P, 1))
    dE = dab.dzeros(A.shape, dist=(1, P), dtype=F32)
    dab.map_inplace(lambda u: 2 * u, dE, dD)                    # map! across layouts, then clobber the source at once
    dab.fill_(dD, np.nan)
    assert np.array_equal(dab.to_array(dE), 2 * A)
    rt.barrier()
    log("ok: halo getindex / makelocal over peer memory")

    # ---- Level-2: A*x, A'*x (tile products + NCCL send/recv to the owners of y), mul! with a DVector x, copy(transpose(A))
    for grid in (None, (P, 1), (1, P)):
        Mx = orc.rand_u01(21, 0, 203 * 157).reshape((203, 157), order="F")
        dM = dab.distribute(Mx, dist=grid)
        oM = orc.distribute(Mx, nworkers=P) if grid is None else orc.distribute(Mx, procs=list(range(1, P + 1)), dist=list(grid))
        for trans in (False, True):
            xv = orc.rand_u01(22 + trans, 0, 203 if trans else 157)
            W = dM.T if trans else dM
            yv = W @ xv
            oy = orc.darray_matvec(oM, xv, trans)
            assert list(yv.layout.pids) == oy.pids and list(yv.layout.indices) == oy.indices
            want = (Mx.T if trans else Mx).astype(np.float64) @ xv.astype(np.float64)
            got = dab.to_array(yv)
            assert np.all(np.abs(got - want) <= 1e-6 * want) and np.all(np.abs(got - orc.to_array(oy)) <= 1e-6 * want)
            y2 = W @ dab.distribute(xv)                         # x as a DVector: blocks halo-fetched from their owners
            assert np.array_equal(dab.to_array(y2), got)
            dab.mul_(yv, W, xv, 2, 1)                           # y = 2*A*x + y
            assert np.all(np.abs(dab.to_array(yv) - 3 * want) <= 3e-6 * want)
        # matrix-matrix: A*B, A'*B with B a DMatrix (blocks halo-fetched), mul!(C, A, B, 2, 1)
        Bx = orc.rand_u01(31, 0, 157 * 64).reshape((157, 64), order="F")
        Bt = orc.rand_u01(32, 0, 203 * 64).reshape((203, 64), order="F")
        for trans, Bh in ((False, Bx), (True, Bt)):
            W = dM.T if trans else dM
            dBm = dab.distribute(Bh)
            Cm = W @ dBm
            oBm = orc.distribute(Bh, nworkers=P)
            oCm = orc.darray_matmat(oM, oBm, trans)
            assert list(Cm.layout.pids) == oCm.pids and list(Cm.layout.indices) == oCm.indices and Cm.layout.grid == tuple(oCm.grid)
            wantm = (Mx.T if trans else Mx).astype(np.float64) @ Bh.astype(np.float64)
            gotm = dab.to_array(Cm)
            assert np.all(np.abs(gotm - wantm) <= 2e-6 * wantm), float(np.abs(gotm / wantm - 1).max())
            dab.mul_(Cm, W, Bh, 2, 1)
            assert np.all(np.abs(dab.to_array(Cm) - 3 * wantm) <= 6e-6 * wantm)
        Tm = dM.T.copy()
        oT = orc.darray_transpose(oM)
        assert list(Tm.layout.indices) == oT.indices and np.array_equal(dab.to_array(Tm), Mx.T)
    rt.barrier()
    log("ok: A*x, A'*x, mul!, copy(transpose(A)) across ranks")

    # ---- ComplexF64: sum (allgather + ordered complex fold, every rank) and copy(adjoint(A)) with pieces pulled from peers
    Z = dab.drand((203, 157), dtype=np.complex128, seed=41)
    hz = dab.to_array(Z)
    k = 2.0 ** 24
    ex = complex(np.round(hz.real * k).astype(np.int64).sum() / k, np.round(hz.imag * k).astype(np.int64).sum() / k)
    s = complex(dab.sum(Z))
    assert abs(s.real - ex.real) <= 1e-13 * ex.real and abs(s.imag - ex.imag) <= 1e-13 * ex.imag, (s, ex)
    H = dab.to_array(dab.adjoint(Z).copy())
    assert np.array_equal(H.real, hz.T.real) and np.array_equal(H.imag, -hz.T.imag)
    rt.barrier()
    log("ok: ComplexF64 sum and copy(adjoint(A)) across ranks")

    # ---- sparse chunks: A*x and A'*x with the tile products on every rank, bit for bit against the model of SparseArrays' loops
    import scipy.sparse as sps
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import sparse_oracle as so
    rs = np.random.default_rng(83)
    Sh = sps.random(203, 157, density=0.1, random_state=rs, data_rvs=rs.standard_normal, format="csc")   # same seed on every rank
    DS = dab.distribute(Sh)
    trip = so.canonical_triplets(Sh)
    for trans, xs in ((False, rs.standard_normal(157)), (True, rs.standard_normal(203))):
        y = dab.to_array((DS.T if trans else DS) @ dab.distribute(xs))
        assert so.same_bits(y, so.mul_model(trip, Sh.shape, DS.layout.cuts, xs, trans)), trans
    assert dab.nnz(DS) == Sh.nnz
    DS.close()
    rt.barrier()
    log("ok: sparse A*x and A'*x across ranks")

    # ---- samplesort across ranks: pieces travel by grouped NCCL send/recv; layout and boundaries equal the oracle's
    for T in (np.int64, np.float64):
        rs = np.random.default_rng(77)
        av = rs.integers(-10 ** 12, 10 ** 12, 300007).astype(T) if T is np.int64 else rs.standard_normal(300007)
        dv = dab.distribute(av)
        ov = orc.distribute(av, nworkers=P)
        for sample in (True, False, av[:400]):
            d2, bnd = dab.sort_with_boundaries(dv, sample=sample)
            o2, ob = orc.darray_sort(ov, sample)
            assert np.array_equal(bnd, ob) and list(d2.layout.pids) == o2.pids and list(d2.layout.indices) == o2.indices
            assert np.array_equal(dab.to_array(d2), np.sort(av))
            d2.close()
    rt.barrier()
    log("ok: sort(d::DVector) across ranks")

    # ---- sortperm across ranks: keys and the Int64 index plane travel by the same grouped send/recv; exact against the model
    for T in (np.int64, np.float64):
        rs = np.random.default_rng(78)
        av = rs.integers(-50, 50, 300007).astype(T)                    # heavy ties: stability across ranks is the whole answer
        dv = dab.distribute(av)
        for sample in (True, False, av[:400]):
            p = dab.sortperm(dv, sample=sample)
            s = dab.sort(dv, sample=sample)
            assert np.array_equal(dab.to_array(p), orc.jl_sortperm_stable(av) + 1)
            assert list(p.layout.pids) == list(s.layout.pids) and list(p.layout.indices) == list(s.layout.indices)
            p.close()
            s.close()
    rt.barrier()
    log("ok: sortperm(d::DVector) across ranks")

    # ---- C5: 256 MiB slab owned by the next rank, contiguous and 2-D strided, bandwidth vs NVLink
    m = 1 << 26
    big = dab.drand((P * (1 << 28),), dtype=F32, seed=3)      # 1 GiB chunk per GPU
    big.share()
    rt.barrier()
    lo = big.indices[nxt][0][0]
    sub = big[lo - 1 + 12345:lo - 1 + 12345 + m]
    results = {}
    dst = dab.B200Array.empty(rt, (m,), F32)
    sub.copy_to(dst)                                                   # warm-up (opens the IPC mapping)
    e0, e1 = rt.event(), rt.event()
    rt.barrier()
    rt.record(e0)
    reps = 10
    for _ in range(reps):
        sub.copy_to(dst)
    rt.record(e1)
    ms = rt.elapsed_ms(e0, e1) / reps
    rt.barrier()
    results["contiguous"] = 4.0 * m / ms / 1e6
    dst.free()
    dev = sub.to_device()
    w = np.empty(4096, dtype=F32)
    _lib.call("dab_d2h", rt.ctx, C.c_void_p(w.ctypes.data), C.c_void_p(dev.ptr + 4 * 777), 4 * 4096)
    rt.sync()
    assert np.array_equal(w, orc.rand_u01(3, lo - 1 + 12345 + 777, 4096))
    dev.free()
    # 2-D strided: row block of a column-major matrix chunk held by the next rank
    M = dab.drand((16384, 8192 * P), dtype=F32, seed=4, dist=(1, P))   # chunk 16384 x 8192 = 512 MiB per GPU
    M.share()
    rt.barrier()
    c0 = M.indices[nxt][1][0] - 1
    subm = M[1024:1024 + 8192, c0:c0 + 8192]                           # 8192 x 8192 = 256 MiB, row-range => strided
    dst = dab.B200Array.empty(rt, (8192, 8192), F32)
    subm.copy_to(dst)
    e0, e1 = rt.event(), rt.event()
    rt.barrier()
    rt.record(e0)
    for _ in range(10):
        subm.copy_to(dst)
    rt.record(e1)
    ms = rt.elapsed_ms(e0, e1) / 10
    rt.barrier()
    dst.free()
    results["strided_2d"] = 4.0 * 8192 * 8192 / ms / 1e6
    dev = subm.to_device()
    col = np.empty(8192, dtype=F32)
    _lib.call("dab_d2h", rt.ctx, C.c_void_p(col.ctypes.data), C.c_void_p(dev.ptr + 4 * 8192 * 5), 4 * 8192)
    rt.sync()
    g0 = (c0 + 5) * 16384 + 1024
    assert np.array_equal(col, orc.rand_u01(4, g0, 8192))
    dev.free()
    allr = rt.allgather_object(results)
    if r == 0:
        worst = {k: min(a[k] for a in allr) for k in results}
        print(json.dumps({"metric": "halo getindex GB/s per reader (all ranks read from their right neighbour concurrently)", "n_gpus": P,
                          "slab_bytes": 4 * m, "GBs_min_over_ranks": worst, "nvlink_peer_copy_peak_GBs": 770.0,
                          "frac_of_peak": {k: v / 770.0 for k, v in worst.items()}}), flush=True)
    dab.d_closeall()
    rt.barrier()
    log("multi-gpu check passed on", P, "GPUs")
    rt.shutdown()


if __name__ == "__main__":
    main()
