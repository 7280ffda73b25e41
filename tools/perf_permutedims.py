#!/usr/bin/env python
"""Single-GPU rates of permutedims (row f18): K28 dab_permute_box against the untiled dab_gather_box on the same pieces, the whole
permutedims call, and copy(transpose(M)) (K10) and copy(A) on the same bytes.

Workloads, 1 GiB each, one chunk on one worker: Float32 (4096, 4096, 64) with perm (2, 1, 3) and (3, 2, 1), Float32 (1024, 1024, 256)
with (2, 3, 1), Float64 (4096, 2048, 16) with (3, 1, 2), ComplexF64 (2048, 2048, 16) with (2, 1, 3), a short leading dimension
Float32 (8, 4096, 8192) with (2, 1, 3) (an 8-element tile side), Float32 (64, 4096, 1024) with (1, 3, 2), which keeps dim 1 in place
and so takes the gather path (its pieces are batches of contiguous runs), odd extents (one-element accesses), Float16 and Bool, and
batched transposes of small planes on each side of the plan's plane threshold (PERMUTE_MIN_PLANE) for every element size.  K28 is
timed on every piece it can take, including those the plan sends to the gather.  Rates are 2 x bytes over the time: one read and one write of
every element.  CUDA events on the ctx stream, every shape warmed up, medians of 7 rounds of 5 calls.  The permute and gather outputs
are compared bit for bit at the timed sizes.  Prints the card's name, power limit and max SM clock, read in the same run."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402
from darray_b200._permute import permute_box_applies, permute_plan  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)

MIB = 1 << 20
WORKLOADS = [(np.float32, (4096, 4096, 64), (2, 1, 3)), (np.float32, (4096, 4096, 64), (3, 2, 1)),
             (np.float32, (1024, 1024, 256), (2, 3, 1)), (np.float64, (4096, 2048, 16), (3, 1, 2)),
             (np.complex128, (2048, 2048, 16), (2, 1, 3)), (np.float32, (8, 4096, 8192), (2, 1, 3)),
             (np.float32, (64, 4096, 1024), (1, 3, 2)),
             # one-element accesses (odd extents), and 2- and 1-byte elements
             (np.float32, (4097, 4095, 16), (2, 1, 3)), (np.float16, (8192, 8192, 8), (2, 1, 3)), (np.bool_, (16384, 16384, 4), (2, 1, 3)),
             # batched transposes of small planes, on each side of PERMUTE_MIN_PLANE for every element size
             (np.float32, (8, 8, 1 << 24), (2, 1, 3)), (np.float32, (24, 24, 1024 * MIB // 2304), (2, 1, 3)),
             (np.float32, (32, 32, 1 << 20), (2, 1, 3)), (np.float64, (16, 16, 1 << 22), (2, 1, 3)),
             (np.float64, (24, 24, 1024 * MIB // 4608), (2, 1, 3)), (np.float16, (16, 16, 1 << 22), (2, 1, 3)),
             (np.float16, (24, 24, 1024 * MIB // 1152), (2, 1, 3)), (np.bool_, (24, 24, 1024 * MIB // 576), (2, 1, 3)),
             (np.bool_, (32, 32, 1 << 20), (2, 1, 3)), (np.complex128, (16, 16, 1 << 18), (2, 1, 3)),
             (np.complex128, (24, 24, 1024 * MIB // 9216), (2, 1, 3)), (np.bool_, (40, 40, 1024 * MIB // 1600), (2, 1, 3)),
             (np.bool_, (64, 64, 1 << 18), (2, 1, 3)), (np.complex128, (16, 32, 1 << 17), (2, 1, 3))]


def timed(rt, fn, reps=5, rounds=7):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(rounds):
        e0, e1 = rt.event(), rt.event()
        rt.sync()
        rt.record(e0)
        for _ in range(reps):
            fn()
        rt.record(e1)
        rt.sync()
        ts.append(rt.elapsed_ms(e0, e1) / reps)
        rt.event_destroy(e0)
        rt.event_destroy(e1)
    return float(np.median(ts))


def piece_call(rt, entry, es, p, dst, src):
    nd = len(p.extent)
    LL = C.c_longlong * nd
    d, s, ext = C.c_void_p(dst + p.dst_offset * es), C.c_void_p(src + p.src_offset * es), (C.c_size_t * nd)(*p.extent)
    if entry == "dab_permute_box":
        return lambda: _lib.call(entry, rt.ctx, es, nd, d, LL(*p.dst_strides), s, LL(*p.src_strides), ext)
    return lambda: _lib.call(entry, rt.ctx, es, nd, d, LL(*p.dst_strides), None, s, LL(*p.src_strides), None, ext)


def main():
    rt = dab.init(workers_per_rank=1, use_dist=False)
    for T, dims, perm in WORKLOADS:
        T = np.dtype(T)
        es = T.itemsize
        nbytes = int(np.prod(dims)) * es
        A = dab.drand(dims, procs=[1], dtype=T) if T.kind in "fc" else dab.dfill(1, dims, procs=[1], dtype=T)
        pd = tuple(dims[k - 1] for k in perm)
        B = dab.similar(A, dims=pd)
        G = dab.similar(A, dims=pd)
        plan = permute_plan(A.layout, B.layout, perm, es)
        assert len(plan) == 1
        p = plan[0]
        src, bptr, gptr = A.chunks[1].ptr, B.chunks[1].ptr, G.chunks[1].ptr
        row = dict(dtype=T.name, dims=dims, perm=perm, mover=p.mover, extent=p.extent)
        rate = lambda ms: round(2 * nbytes / ms / 1e6, 1)  # noqa: E731
        k28 = permute_box_applies(p.extent, p.dst_strides, p.src_strides)    # timed on both sides of the plan's threshold
        if k28:
            ms = timed(rt, piece_call(rt, "dab_permute_box", es, p, bptr, src))
            row["permute_box_ms"], row["permute_box_GBps"] = round(ms, 3), rate(ms)
        ms = timed(rt, piece_call(rt, "dab_gather_box", es, p, gptr, src))
        row["gather_box_ms"], row["gather_box_GBps"] = round(ms, 3), rate(ms)
        if k28:
            pb = piece_call(rt, "dab_permute_box", es, p, bptr, src)
            pb()
            rt.sync()
            row["outputs_equal"] = bool(np.array_equal(B.chunks[1].to_numpy().reshape(-1, order="F").view(np.uint8),
                                                         G.chunks[1].to_numpy().reshape(-1, order="F").view(np.uint8)))

        def api():
            dab.permutedims(A, perm).close()

        ms = timed(rt, api, reps=3)
        row["permutedims_ms"], row["permutedims_GBps"] = round(ms, 3), rate(ms)
        n = int(np.prod(dims))
        m = 1 << ((n.bit_length() - 1) // 2)                    # a matrix of the same bytes, as square as a power of two allows
        M = dab.similar(A, dims=(m, n // m))
        Mt = dab.similar(M, dims=(n // m, m))
        ms = timed(rt, lambda: _lib.call("dab_transpose_box", rt.ctx, es, C.c_void_p(Mt.chunks[1].ptr), n // m, C.c_void_p(M.chunks[1].ptr), m,
                                         m, n // m))
        row["transpose_box_ms"], row["transpose_box_GBps"] = round(ms, 3), rate(ms)
        ms = timed(rt, lambda: dab.copy_transposed(dab.transpose(M)).close(), reps=3)
        row["copy_transpose_ms"], row["copy_transpose_GBps"] = round(ms, 3), rate(ms)
        ms = timed(rt, lambda: dab.copy(A).close(), reps=3)
        row["copy_ms"], row["copy_GBps"] = round(ms, 3), rate(ms)
        for x in (A, B, G, M, Mt):
            x.close()
        print(json.dumps(row), flush=True)
    dab.d_closeall()
    rt.shutdown()


if __name__ == "__main__":
    main()
