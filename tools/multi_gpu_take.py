#!/usr/bin/env python
"""d[I::DArray] across GPUs, one process per GPU:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29518 tools/multi_gpu_take.py

Checks, against Julia's A[I] computed on the host on every rank: a 2-d d split across ranks indexed by an I in a different layout (its
blocks are halo reads, the source elements peer loads over CUDA IPC), v[sortperm(v)] across ranks, and the same BoundsError on every
rank with nothing left registered; then times v[p] for 2^26 Float64 with p a random permutation (most reads are peer reads over NVLink)
and prints one JSON line (rank 0).
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402
from oracle import darray_oracle as orc  # noqa: E402


def model(a, I):
    return np.asarray(a).ravel(order="F")[np.asarray(I) - 1].reshape(np.shape(I), order="F")


def main():
    rt = dab.init(workers_per_rank=1)
    P, r = rt.world, rt.rank
    assert P >= 2, "run under torchrun with >= 2 ranks"
    log = (lambda *a: print(*a, flush=True)) if r == 0 else (lambda *a: None)
    rng = np.random.default_rng(7)                                       # the same host data on every rank

    h = rng.standard_normal((301, 17 * P))
    d = dab.distribute(h)
    Ih = rng.integers(1, h.size + 1, (1000, 3))
    I = dab.distribute(Ih, procs=list(reversed(rt.workers())), dist=[P, 1])
    R = d[I]
    assert not I.layout.same_as(R.layout)
    assert np.array_equal(dab.to_array(R).view(np.uint64), model(h, Ih).view(np.uint64))
    I32 = dab.distribute(Ih.astype(np.int32))
    assert np.array_equal(dab.to_array(d[I32]), model(h, Ih))
    log("ok: 2-d d across", P, "ranks, I in another layout, Int64 and Int32")

    vh = np.round(rng.standard_normal(200003), 2)
    vh[rng.integers(0, vh.size, 1000)] = np.nan
    v = dab.distribute(vh)
    w = v[dab.sortperm(v)]
    assert np.array_equal(dab.to_array(w).view(np.uint64), vh[orc.jl_sortperm_stable(vh)].view(np.uint64))
    log("ok: v[sortperm(v)] across ranks")

    bad = Ih.copy()
    bad[990, 2] = h.size + 9                                             # in the last rank's part of R only
    bad[999, 2] = 0
    B = dab.distribute(bad)
    r0 = dab.registry_size()
    msg = None
    try:
        d[B]
    except IndexError as e:
        msg = str(e)
    msgs = rt.allgather_object(msg)
    assert msg is not None and all(m == msg for m in msgs) and f"[{h.size + 9}]" in msg, msgs
    assert dab.registry_size() == r0
    assert np.array_equal(dab.to_array(d[I]), model(h, Ih))
    log("ok: the same BoundsError on every rank:", msg)

    n = 1 << 26
    big = dab.distribute(rng.standard_normal(n))
    p = dab.distribute((rng.permutation(n) + 1).astype(np.int64))
    big[p].close()
    ts = []
    for _ in range(5):
        rt.barrier()
        t0 = time.perf_counter()
        out = big[p]
        rt.sync()
        ts.append((time.perf_counter() - t0) * 1e3)
        out.close()
    log(json.dumps({"metric": "take_2^26_f64_random_permutation_ms", "ranks": P, "median_ms": round(float(np.median(ts)), 3),
                    "useful_GBps": round(n * 24 / float(np.median(ts)) / 1e6, 1)}))
    dab.d_closeall()
    log("multi-gpu take passed")
    rt.shutdown()


if __name__ == "__main__":
    main()
