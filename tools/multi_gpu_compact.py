#!/usr/bin/env python
"""d[mask], findall and filter across GPUs, one process per GPU:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29519 tools/multi_gpu_compact.py

Checks, against Julia's logical indexing computed on the host on every rank: a 2-d d split along dim 1 across ranks (its runs
interleave the ranks in the global order) with the mask in a different layout (halo reads of the mask), results whose chunks live on
other ranks (peer stores over CUDA IPC), findall and filter with a predicate, and an all-false mask; then times d[m] for 2^26 Float64
at density 0.5 and prints one JSON line (rank 0).
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402


def model(a, m):
    return np.asarray(a).ravel(order="F")[np.asarray(m).ravel(order="F")]


def main():
    rt = dab.init(workers_per_rank=1)
    P, r = rt.world, rt.rank
    assert P >= 2, "run under torchrun with >= 2 ranks"
    log = (lambda *a: print(*a, flush=True)) if r == 0 else (lambda *a: None)
    rng = np.random.default_rng(7)                                       # the same host data on every rank

    h = rng.standard_normal((301, 37))
    mh = rng.random(h.shape) < 0.4
    d = dab.distribute(h, dist=[P, 1])
    m = dab.distribute(mh, procs=list(reversed(rt.workers())), dist=[1, P])
    assert not m.layout.same_as(d.layout)
    R = d[m]
    assert np.array_equal(dab.to_array(R).view(np.uint64), model(h, mh).view(np.uint64))
    F = dab.findall(m)
    assert np.array_equal(dab.to_array(F), np.flatnonzero(mh.ravel(order="F")) + 1)
    assert np.array_equal(dab.to_array(d[F]).view(np.uint64), dab.to_array(R).view(np.uint64))
    log("ok: d split along dim 1 across", P, "ranks, the mask in another layout, findall and d[findall(m)]")

    assert np.array_equal(dab.to_array(dab.filter(lambda x: x > 0.5, d)), model(h, h > 0.5))
    assert np.array_equal(dab.to_array(dab.findall(lambda x: x < 0, d)), np.flatnonzero((h < 0).ravel(order="F")) + 1)
    E = d[dab.distribute(np.zeros(h.shape, dtype=bool))]
    assert E.dims == (0,)
    log("ok: filter and findall with predicates, an all-false mask")

    n = 1 << 26
    big = dab.distribute(rng.standard_normal(n))
    bm = dab.broadcast(lambda x: x > 0, big)
    big[bm].close()
    ts = []
    for _ in range(5):
        rt.barrier()
        t0 = time.perf_counter()
        out = big[bm]
        rt.sync()
        ts.append((time.perf_counter() - t0) * 1e3)
        out.close()
    log(json.dumps({"metric": "compact_2^26_f64_density_0.5_ms", "ranks": P, "median_ms": round(float(np.median(ts)), 3)}))
    dab.d_closeall()
    log("multi-gpu compact passed")
    rt.shutdown()


if __name__ == "__main__":
    main()
