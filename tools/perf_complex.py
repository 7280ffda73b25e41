#!/usr/bin/env python
"""Single-GPU rates of the complex element types (CUDA events, algorithmic bytes over kernel time, warmed up, medians of repeats):
sum of 2^28 ComplexF64 and 2^29 ComplexF32 beside the Float64 sum of the same bytes, copy(adjoint(A)) against copy(transpose(A)) of the
same ComplexF64 matrix, z .* w for ComplexF32, and torch's complex sum / conj().T.contiguous() as yardsticks.  Prints the card's name and
power limit, read in the same run."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
rt = dab.init(use_dist=False)


def timed(fn, reps=10, rounds=5):
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
    return float(np.median(out))


def report(name, ms, nbytes):
    print(f"{name:48s} {ms:9.4f} ms {nbytes / ms / 1e6:9.1f} GB/s", flush=True)


GiB4 = 1 << 32
z128 = dab.drand((1 << 28,), dtype=np.complex128, seed=1)
report("sum(z) ComplexF64 2^28            (4 GiB)", timed(lambda: dab.sum(z128)), GiB4)
z128.close()
z64 = dab.drand((1 << 29,), dtype=np.complex64, seed=2)
report("sum(z) ComplexF32 2^29            (4 GiB)", timed(lambda: dab.sum(z64)), GiB4)
z64.close()
x64 = dab.drand((1 << 29,), dtype=np.float64, seed=3)
report("sum(x) Float64 2^29               (4 GiB)", timed(lambda: dab.sum(x64)), GiB4)
x64.close()

A = dab.drand((16384, 8192), dtype=np.complex128, seed=4)                    # 2 GiB
nb = 2 * A.size * 16
report("copy(adjoint(A)) ComplexF64 16384x8192", timed(lambda: dab.adjoint(A).copy().close(), reps=5), nb)
report("copy(transpose(A)) ComplexF64 16384x8192", timed(lambda: dab.transpose(A).copy().close(), reps=5), nb)
A.close()

n = 1 << 28
z = dab.drand((n,), dtype=np.complex64, seed=5)
w = dab.drand((n,), dtype=np.complex64, seed=6)
out = dab.similar(z)
report("out .= z .* w ComplexF32 2^28     (24 B/elem)", timed(lambda: dab.broadcast_into(out, lambda a, b: a * b, z, w)), 24 * n)
for d in (z, w, out):
    d.close()

try:
    import torch
    t = torch.complex(torch.rand(1 << 28, dtype=torch.float64, device="cuda"), torch.rand(1 << 28, dtype=torch.float64, device="cuda"))
    M = torch.complex(torch.rand(16384, 8192, dtype=torch.float64, device="cuda"), torch.rand(16384, 8192, dtype=torch.float64, device="cuda"))

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

    report("torch.sum(complex128 2^28)        (4 GiB)", ttimed(lambda: t.sum()), GiB4)
    report("torch M.conj().T.contiguous() c128 16384x8192", ttimed(lambda: M.conj().T.contiguous(), reps=5), 2 * M.numel() * 16)
except Exception as e:  # the yardstick is optional: the numbers above stand on their own
    print("torch yardstick not measured:", repr(e)[:200])
dab.d_closeall()
