#!/usr/bin/env python
"""Single-GPU rates of the scans (K17; CUDA events, algorithmic bytes over kernel time, warmed up, medians of repeats): cumsum! of a 2^30
Float32 vector, cumsum!(B, A; dims=1) of 4096 x 2^18 and 10 x 10^8, dims=2 of 32768 x 32768 and 3 x 10^8, and the vector with dims split
over 8 workers on the one GPU.  Bytes are in + out per element, plus one more read per element where the length is split (the strided
path's segments, or the chunk totals of a split dims).  Yardsticks in the same run: the package's identity broadcast y .= x on the same
bytes and torch.cumsum on the same tensor.  Prints the card's name, power limit and max SM clock, read in the same run."""
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
        out.append(rt.elapsed_ms(e0, e1) / reps)
        rt.event_destroy(e0)
        rt.event_destroy(e1)
    return float(np.median(out))


def report(name, ms, nbytes):
    print(f"{name:52s} {ms:9.4f} ms {nbytes / ms / 1e6:9.1f} GB/s", flush=True)


rt = dab.init(workers_per_rank=1, use_dist=False)
n = 1 << 30
x = dab.drand((n,), dtype=np.float32, seed=1)
y = dab.similar(x)
report("y .= x (identity broadcast) Float32 2^30", timed(rt, lambda: dab.broadcast_into(y, lambda v: v, x)), 8 * n)
report("cumsum!(y, x) Float32 2^30", timed(rt, lambda: dab.cumsum_(y, x)), 8 * n)
x.close()
y.close()
for shape, dims, extra in (((4096, 1 << 18), 1, 0), ((10, 10 ** 8), 1, 0), ((32768, 32768), 2, 4), ((3, 10 ** 8), 2, 4)):
    A = dab.drand(shape, dtype=np.float32, seed=2)
    B = dab.similar(A)
    m = A.size
    report(f"cumsum!(B, A; dims={dims}) Float32 {shape[0]}x{shape[1]}", timed(rt, lambda: dab.cumsum_(B, A, dims=dims), reps=5), (8 + extra) * m)
    A.close()
    B.close()
dab.d_closeall()

rt8 = dab.init(workers_per_rank=8, use_dist=False)
x = dab.drand((n,), dtype=np.float32, seed=3)
y = dab.similar(x)
# 7 of the 8 chunks are read once more for their totals
report("cumsum!(y, x) Float32 2^30, dims split over 8 workers", timed(rt8, lambda: dab.cumsum_(y, x), reps=5), 8 * n + 4 * n * 7 // 8)
dab.d_closeall()

try:
    import torch
    t = torch.rand(n, dtype=torch.float32, device="cuda")
    o = torch.empty_like(t)

    def ttimed(fn, reps=10, rounds=5):
        for _ in range(3):
            fn()
        out = []
        for _ in range(rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            e1.synchronize()
            out.append(e0.elapsed_time(e1) / reps)
        return float(np.median(out))

    report("torch.cumsum(float32 2^30, out=)", ttimed(lambda: torch.cumsum(t, 0, out=o)), 8 * n)
except Exception as e:  # the yardstick is optional: the numbers above stand on their own
    print("torch yardstick not measured:", repr(e)[:200])
