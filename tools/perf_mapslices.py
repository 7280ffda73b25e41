#!/usr/bin/env python
"""Rates of the two mapslices kernels on one GPU, with CUDA events after a warm-up, and the card's name and power limit read in the same run.

  dab_sort_slices      GB/s on 2 x element bytes per element (one read, one write: its HBM roofline) and the share of the 3.35 TB/s
                       H100 SXM data sheet; 2^28 elements as columns of 32 / 1024 / 4096 (dim 1, inner = 1) and as rows of the same
                       lengths (dim 2, inner > 1).  Yardsticks in the same run: torch.sort along the same dim (NaN-free data without
                       signed zeros, where its order is isless), and a per-fibre dab_sort loop at one mid size.
  dab_svdvals_batched  matrices/s for 2^16 random matrices of 5x5, 10x10, 32x32.  No FLOP/s figure: the number of Jacobi sweeps (and
                       of rotations) a matrix takes is data-dependent and not reported by the kernel, so an operation count would be a
                       guess, not a measurement.
Run: python tools/perf_mapslices.py  (needs a GPU; prints one line per measurement)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402

HBM = 3.35e12
rt = dab.init(workers_per_rank=1, use_dist=False)


def card():
    out = subprocess.run(["nvidia-smi", "-i", str(rt.device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return out


def timed(fn, reps=5):
    for _ in range(2):
        fn()
    e0, e1 = rt.event(), rt.event()
    rt.sync()
    rt.record(e0)
    for _ in range(reps):
        fn()
    rt.record(e1)
    return rt.elapsed_ms(e0, e1) / reps


print("card:", card(), flush=True)
import torch  # noqa: E402

rng = np.random.default_rng(1)
N = 1 << 28
for T in (np.float32, np.float64):
    es = np.dtype(T).itemsize
    a = (rng.random(N, dtype=np.float64) + 0.5).astype(T)        # NaN-free, no signed zeros: torch.sort's order is isless here
    x = dab.B200Array.from_numpy(rt, a)
    y = dab.B200Array.empty(rt, (N,), T)
    xt = torch.from_numpy(a).to("cuda")
    code = dab.dab_dtype(np.dtype(T))
    for ln in (32, 1024, 4096):
        for dim in (1, 2):
            inner, outer = (1, N // ln) if dim == 1 else (N // ln, 1)
            fn = lambda: _lib.call("dab_sort_slices", rt.ctx, code, C.c_void_p(x.ptr), C.c_void_p(y.ptr), inner, ln, outer)  # noqa: E731
            ms = timed(fn)
            gbs = 2 * es * N / ms / 1e6
            # torch: the same fibres, column-major (inner, len, outer) == row-major (outer, len, inner)
            tv = xt.view(outer, ln, inner)
            torch.sort(tv, dim=1)
            torch.cuda.synchronize()
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(5):
                torch.sort(tv, dim=1)
            s1.record()
            torch.cuda.synchronize()
            tms = s0.elapsed_time(s1) / 5
            print(f"sort_slices {np.dtype(T).name} len={ln:5d} dim={dim} inner={inner:9d} outer={outer:9d}: {ms:8.3f} ms {gbs:7.0f} GB/s "
                  f"({gbs * 1e9 / HBM:5.1%} of 3.35 TB/s); torch.sort {tms:8.3f} ms -> torch/ours {tms / ms:5.2f}", flush=True)
    # per-fibre K11 loop at one mid size (1024): the path the in-shared-memory kernel replaces
    ln, nf = 1024, 2048
    tmp = dab.B200Array.empty(rt, (ln,), T)

    def loop():
        for f in range(nf):
            _lib.call("dab_sort", rt.ctx, code, C.c_void_p(x.ptr + f * ln * es), C.c_void_p(y.ptr + f * ln * es), C.c_void_p(tmp.ptr), ln)

    ms_loop = timed(loop, reps=2)
    ms_ss = timed(lambda: _lib.call("dab_sort_slices", rt.ctx, code, C.c_void_p(x.ptr), C.c_void_p(y.ptr), 1, ln, nf))
    print(f"sort_slices {np.dtype(T).name} {nf} fibres of {ln}: {ms_ss:8.3f} ms; per-fibre dab_sort loop {ms_loop:8.3f} ms -> "
          f"{ms_loop / ms_ss:6.1f}x", flush=True)
    for b in (x, y, tmp):
        b.free()
    del xt
    torch.cuda.empty_cache()

B = 1 << 16
for n in (5, 10, 32):
    A = rng.standard_normal(n * n * B)
    dA = dab.B200Array.from_numpy(rt, A)
    S = dab.B200Array.empty(rt, (n * B,), np.float64)
    st = dab.B200Array.empty(rt, (1,), np.int32)
    ms = timed(lambda: _lib.call("dab_svdvals_batched", rt.ctx, _lib.F64, C.c_void_p(dA.ptr), n, n, B, C.c_void_p(S.ptr), C.c_void_p(st.ptr)))
    print(f"svdvals_batched Float64 {B} x {n}x{n}: {ms:8.3f} ms {B / ms * 1e3:12.0f} matrices/s", flush=True)
    for b in (dA, S, st):
        b.free()
dab.d_closeall()
rt.shutdown()
