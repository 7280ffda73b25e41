#!/usr/bin/env python
"""permutedims across GPUs, one process per GPU:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29528 tools/multi_gpu_permute.py

Checks, against np.transpose computed on the host on every rank: a 3-d array split across ranks permuted into the default layout and,
with permutedims!, into a destination cut along another dimension in reversed rank order (most source pieces are peer reads over CUDA
IPC), a matrix through copy_transposed, and the same refusal on every rank with nothing left registered; then times permutedims of a
Float32 (2048, 2048, 64) array split along its last dimension with perm (3, 2, 1), whose pieces are almost all peer reads, and prints
one JSON line (rank 0).
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402


def main():
    rt = dab.init(workers_per_rank=1)
    P, r = rt.world, rt.rank
    assert P >= 2, "run under torchrun with >= 2 ranks"
    log = (lambda *a: print(*a, flush=True)) if r == 0 else (lambda *a: None)
    rng = np.random.default_rng(28)                                      # the same host data on every rank

    h = rng.standard_normal((37, 11 * P, 23))
    A = dab.distribute(h, dist=[1, P, 1])
    for perm in [(3, 1, 2), (2, 3, 1), (1, 3, 2)]:
        want = np.transpose(h, [p - 1 for p in perm])
        B = dab.permutedims(A, perm)
        assert np.array_equal(dab.to_array(B).view(np.uint64), want.view(np.uint64)), perm
        D = dab.dzeros(want.shape, procs=list(reversed(rt.workers())), dist=[P, 1, 1])
        dab.permutedims_(D, A, perm)
        assert np.array_equal(dab.to_array(D).view(np.uint64), want.view(np.uint64)), perm
    log("ok: 3-d array across", P, "ranks, default and foreign destinations")

    m = rng.standard_normal((301, 17 * P))
    M = dab.distribute(m)
    assert np.array_equal(dab.to_array(dab.permutedims(M)), m.T)
    log("ok: permutedims(M) across ranks")

    r0 = dab.registry_size()
    msg = None
    try:
        dab.permutedims_(A, A, (1, 2, 3))
    except dab.ArgumentError as e:
        msg = str(e)
    msgs = rt.allgather_object(msg)
    assert msg is not None and all(x == msg for x in msgs), msgs
    assert dab.registry_size() == r0
    log("ok: the same refusal on every rank:", msg)

    big = dab.drand((2048, 2048, 64), dtype=np.float32)
    dab.permutedims(big, (3, 2, 1)).close()
    ts = []
    for _ in range(5):
        rt.barrier()
        t0 = time.perf_counter()
        out = dab.permutedims(big, (3, 2, 1))
        rt.sync()
        ts.append((time.perf_counter() - t0) * 1e3)
        out.close()
    nbytes = 2048 * 2048 * 64 * 4
    log(json.dumps({"metric": "permutedims_f32_2048x2048x64_(3,2,1)_ms", "ranks": P, "median_ms": round(float(np.median(ts)), 3),
                    "GBps_2x_bytes": round(2 * nbytes / float(np.median(ts)) / 1e6, 1)}))
    dab.d_closeall()
    log("multi-gpu permutedims passed")
    rt.shutdown()


if __name__ == "__main__":
    main()
