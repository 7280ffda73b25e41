#!/usr/bin/env python
"""Single-GPU rates of Float16 against Float32 through the same public calls (CUDA events, HBM bytes moved over time, warmed up,
medians of repeats): the flagship step y .= a.*x .+ b; sum(y) at 2^31 Float16 and 2^30 Float32 elements (the same bytes), sum(d) and
sum(A, dims=1) and dot(x, y) (the fused map-reduce kernel) of the same bytes, with torch's half-precision a*x+b, torch.sum and torch.sum(dim=0) on the same memory as yardsticks.
Prints the card's name and power limit, read in the same run, and each rate's share of 3.35 TB/s."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402

PEAK = 3.35e12
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
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


rates = {}


def report(key, name, ms, nbytes):
    gbs = nbytes / ms / 1e6
    rates[key] = (ms, gbs)
    print(f"{name:52s} {ms:9.4f} ms {gbs:9.1f} GB/s {100 * gbs * 1e9 / PEAK:6.1f} % of 3.35 TB/s", flush=True)


def flagship(dt, n, key):
    x = dab.drand((n,), dtype=dt, seed=1)
    y = dab.similar(x)
    a, b = dt(0.5), dt(0.25)

    def step():
        dab.broadcast_into(y, lambda v: a * v + b, x)
        return dab.sum(y)

    es = np.dtype(dt).itemsize
    # HBM bytes each path moves: Float32 runs the step as ONE fused map-store-reduce kernel (reads x, writes y); Float16 trees take the
    # NVRTC broadcast and then the reduce kernel (reads x, writes y, reads y)
    passes = 2 if np.dtype(dt) == np.dtype(np.float32) else 3
    report(key, f"y .= a.*x .+ b; sum(y)  {np.dtype(dt).name} n={n}", timed(step), passes * es * n)
    report(key + "_sum", f"sum(d)                  {np.dtype(dt).name} n={n}", timed(lambda: dab.sum(x)), es * n)
    report(key + "_dot", f"dot(x, y)               {np.dtype(dt).name} n={n}", timed(lambda: dab.dot(x, y)), 2 * es * n)   # fused map-reduce kernel
    x.close()
    y.close()


def sum_dims(dt, rows, cols, key):
    A = dab.drand((rows, cols), dtype=dt, seed=2)
    es = np.dtype(dt).itemsize
    report(key, f"sum(A, dims=1)          {np.dtype(dt).name} {rows}x{cols}", timed(lambda: dab.sum(A, dims=1).close(), reps=5), es * A.size)
    A.close()


flagship(np.float16, 1 << 31, "f16")
flagship(np.float32, 1 << 30, "f32")
sum_dims(np.float16, 1 << 15, 1 << 15, "f16_dims")
sum_dims(np.float32, 1 << 15, 1 << 14, "f32_dims")
for k in ("", "_sum"):
    print(f"Float16 / Float32 bytes per second{k or ' (flagship)':>12s}: {rates['f16' + k][1] / rates['f32' + k][1]:.3f}")
print(f"Float16 / Float32 bytes per second (dot):    {rates['f16_dot'][1] / rates['f32_dot'][1]:.3f}")
print(f"Float16 / Float32 bytes per second (dims=1): {rates['f16_dims'][1] / rates['f32_dims'][1]:.3f}")

try:
    import torch

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

    n = 1 << 31
    t = torch.rand(n, dtype=torch.float16, device="cuda")
    u = torch.empty_like(t)

    def tstep():
        torch.add(torch.mul(t, 0.5, out=u), 0.25, out=u)
        return u.sum()

    ms = ttimed(tstep)
    print(f"torch half a*x+b; sum  n=2^31: {ms:.4f} ms; Float16 DArray step takes {rates['f16'][0] / ms:.2f}x its time")
    ms = ttimed(lambda: t.sum())
    print(f"torch.sum half n=2^31:         {ms:.4f} ms; Float16 DArray sum takes {rates['f16_sum'][0] / ms:.2f}x its time")
    del t, u
    M = torch.rand(1 << 15, 1 << 15, dtype=torch.float16, device="cuda")
    ms = ttimed(lambda: M.sum(dim=1), reps=5)                # column-major A's dims=1 is row-major M's last dim
    print(f"torch.sum(dim) half 32768^2:   {ms:.4f} ms; Float16 DArray sum(A, dims=1) takes {rates['f16_dims'][0] / ms:.2f}x its time")
except Exception as e:  # the yardstick is optional: the numbers above stand on their own
    print("torch yardstick not measured:", repr(e)[:200])
dab.d_closeall()
