#!/usr/bin/env python
"""Single-GPU rates of findmax (K20; CUDA events, algorithmic bytes over the call's time, warmed up, medians of repeats) against maximum on
the same chunk in the same run: findmax(d) and maximum(d) of one 2^30-element Float32 chunk and one Float64 chunk (sizeof(T) bytes per
element), and findmax(d; dims) / maximum(d; dims) for dims = 1 and 2 of a 32768 x 16384 Float32 chunk (findmax: 4 bytes per element read,
4 + 8 per output written; maximum: 4 read, 4 written).  Each result is checked against the host.  Prints the card's name, power limit and
max SM clock, read in the same run."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)


def timed(rt, fn, reps=10, rounds=5):
    for _ in range(3):
        fn()
    out = []
    for _ in range(rounds):
        e0, e1 = rt.event(), rt.event()
        rt.sync()
        rt.record(e0)
        for _ in range(reps):
            fn()
        rt.record(e1)
        rt.sync()
        out.append(rt.elapsed_ms(e0, e1) / reps)
        rt.event_destroy(e0)
        rt.event_destroy(e1)
    return float(np.median(out))


def report(name, ms, nbytes):
    gbs = nbytes / ms / 1e6
    print(f"{name:52s} {ms:9.4f} ms {gbs:9.1f} GB/s", flush=True)
    return gbs


def close_all(*arrays):
    for a in arrays:
        a.close()


rt = dab.init(workers_per_rank=1, use_dist=False)
n = 1 << 30
for dt in (np.float32, np.float64):
    x = dab.drand((n,), dtype=dt, seed=1)
    isz = np.dtype(dt).itemsize
    rm = report(f"maximum(d) {np.dtype(dt).name} 2^30", timed(rt, lambda: dab.maximum(x)), isz * n)
    rf = report(f"findmax(d) {np.dtype(dt).name} 2^30", timed(rt, lambda: dab.findmax(x)), isz * n)
    print(f"  findmax / maximum rate: {rf / rm:.3f}", flush=True)
    v, i = dab.findmax(x)
    host = dab.to_array(x)
    assert v == host.max() and i == int(np.argmax(host)) + 1, (v, i)
    del host
    x.close()

A = dab.drand((32768, 16384), dtype=np.float32, seed=2)
m = A.size
for dims, nout in ((1, 16384), (2, 32768)):
    rm = report(f"maximum(d; dims={dims}) Float32 32768x16384", timed(rt, lambda: close_all(dab.maximum(A, dims=dims)), reps=5), 4 * m + 4 * nout)
    rf = report(f"findmax(d; dims={dims}) Float32 32768x16384", timed(rt, lambda: close_all(*dab.findmax(A, dims=dims)), reps=5),
                4 * m + 12 * nout)
    print(f"  findmax / maximum rate: {rf / rm:.3f}", flush=True)
    V, I = dab.findmax(A, dims=dims)
    v, i = dab.to_array(V).ravel(order="F"), dab.to_array(I).ravel(order="F")
    for k in (0, nout // 2, nout - 1):                                           # a sample of slices against the host
        sl = np.asarray(A[:, k:k + 1] if dims == 1 else A[k:k + 1, :]).ravel(order="F")
        j = int(np.argmax(sl))
        want = (j + 1 + 32768 * k) if dims == 1 else (k + 1 + 32768 * j)
        assert v[k] == sl[j] and i[k] == want, (dims, k, v[k], i[k], sl[j], want)
    close_all(V, I)
A.close()
dab.d_closeall()
print("perf_findmax: results checked", flush=True)
