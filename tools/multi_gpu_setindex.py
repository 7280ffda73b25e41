#!/usr/bin/env python
"""d[key] = v across GPUs, one process per GPU:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29519 tools/multi_gpu_setindex.py

Checks, against Julia's sequential setindex! computed on the host on every rank: a 2-d d split across ranks written through an I in
another layout with duplicates that cross ranks (peer atomics into other ranks' bitmaps and winner tables, peer stores into their chunks),
with a DArray value in a third layout; a mask in another layout with a DArray value (peer reads of the values); a strided view written
from a view of another DArray; and the same BoundsError on every rank with d unchanged and nothing left registered.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402


def model_take(a, I, v):
    out = a.copy()
    flat = out.reshape(-1, order="F")
    g = np.asarray(I, dtype=np.int64).reshape(-1, order="F") - 1
    vals = np.asarray(v).reshape(-1, order="F")
    _, last_rev = np.unique(g[::-1], return_index=True)
    last = g.size - 1 - last_rev
    flat[g[last]] = vals[last]
    return flat.reshape(a.shape, order="F")


def main():
    rt = dab.init(workers_per_rank=1)
    P, r = rt.world, rt.rank
    assert P >= 2, "run under torchrun with >= 2 ranks"
    rng = np.random.default_rng(11)                                      # the same host data on every rank
    h = rng.standard_normal((301, 17 * P))
    d = dab.distribute(h)
    Ih = rng.integers(1, h.size + 1, (4000, 3))
    Ih[:50] = Ih[-50:]                                                   # duplicates whose occurrences live on different ranks
    I = dab.distribute(Ih, procs=list(reversed(rt.workers())), dist=[P, 1])
    vh = rng.standard_normal(Ih.shape)
    v = dab.distribute(vh, procs=list(reversed(rt.workers())), dist=[1, min(P, 3)])
    d[I] = v
    want = model_take(h, Ih, vh)
    assert np.array_equal(dab.to_array(d).view(np.uint64), want.view(np.uint64)), "d[I] = v"

    mh = rng.random(h.shape) < 0.4
    m = dab.distribute(mh, procs=list(reversed(rt.workers())))
    w = rng.standard_normal(int(mh.sum()))
    d[m] = dab.distribute(w)
    f = want.reshape(-1, order="F")
    f[mh.reshape(-1, order="F")] = w
    want = f.reshape(h.shape, order="F")
    assert np.array_equal(dab.to_array(d).view(np.uint64), want.view(np.uint64)), "d[m] = v"

    E = rng.standard_normal((100, 40))
    e = dab.distribute(E, procs=list(reversed(rt.workers())))
    d[3:250:3, 1:9] = e[10:93, 30:38]
    want[3:250:3, 1:9] = E[10:93, 30:38]
    assert np.array_equal(dab.to_array(d).view(np.uint64), want.view(np.uint64)), "view write"

    bad = Ih.copy()
    bad[3999, 2] = h.size + 1
    B = dab.distribute(bad, procs=list(reversed(rt.workers())), dist=[P, 1])
    r0 = dab.registry_size()
    try:
        d[B] = 0.0
        raise AssertionError("no BoundsError")
    except IndexError as e:
        assert f"[{h.size + 1}]" in str(e), str(e)
    assert dab.registry_size() == r0
    assert np.array_equal(dab.to_array(d).view(np.uint64), want.view(np.uint64)), "d changed by a failed call"
    dab.d_closeall()
    if r == 0:
        print("multi-gpu setindex passed", flush=True)
    rt.shutdown()


if __name__ == "__main__":
    main()
