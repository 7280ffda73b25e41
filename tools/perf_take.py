#!/usr/bin/env python
"""Single-GPU rates of the indexed gather K22 (dab_index_gather, the step under d[I::DArray]) against torch.index_select on the same
tensors, then whole d[p] calls on 8 workers against the host composition d[np.asarray(p) - 1].to_darray().

Kernel cases: one chunk on one worker, n = 2^26 and 2^28 Int64 indices into a Float32 or Float64 source of n elements, four index
patterns: identity, a uniform random permutation, sortperm of uniform data (dab.sortperm: a random permutation produced the way users
get one) and a block-local permutation (shuffled within 64 KiB windows of the source).  Useful bytes per element: 8 + 2 * elem (read the
index, read the element, write the element); index_select moves the same bytes.  Both outputs are compared bit for bit in the same
run.  CUDA events, every shape warmed up, the two kernels alternated, medians of repeats.

Whole calls: v[p] for 2^26 Float64 on 8 workers with p = sortperm(v), host clock to a device synchronise.  With two or more GPUs the
same call is repeated under torchrun by tools/multi_gpu_take.py (peer reads over NVLink).  Prints the card's name, power limit and max
SM clock, read in the same run."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)


def timed_pair(rt, fa, fb, reps=5, rounds=7):
    """Median ms of fa (dab events on the ctx stream) and fb (torch events), alternated round by round."""
    for _ in range(2):
        fa()
        fb()
    ta, tb = [], []
    for _ in range(rounds):
        e0, e1 = rt.event(), rt.event()
        rt.sync()
        torch.cuda.synchronize()
        rt.record(e0)
        for _ in range(reps):
            fa()
        rt.record(e1)
        rt.sync()
        ta.append(rt.elapsed_ms(e0, e1) / reps)
        rt.event_destroy(e0)
        rt.event_destroy(e1)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            fb()
        t1.record()
        torch.cuda.synchronize()
        tb.append(t0.elapsed_time(t1) / reps)
    return float(np.median(ta)), float(np.median(tb))


def timed_wall(rt, fn, rounds=5):
    fn().close()
    out = []
    for _ in range(rounds):
        rt.sync()
        t0 = time.perf_counter()
        r = fn()
        rt.sync()
        out.append((time.perf_counter() - t0) * 1e3)
        r.close()
    return float(np.median(out))


def kernel_cases(rt):
    print(f"{'case':44s} {'K22 ms':>9s} {'GB/s':>8s} {'index_select ms':>16s} {'GB/s':>8s} {'K22/torch':>10s}", flush=True)
    dev = torch.device("cuda", rt.device)
    for n in (1 << 26, 1 << 28):
        g = torch.Generator(device=dev)
        g.manual_seed(n)
        for T, tt in ((np.float32, torch.float32), (np.float64, torch.float64)):
            es = np.dtype(T).itemsize
            src = torch.rand(n, device=dev, generator=g, dtype=torch.float64).to(tt)
            out = torch.empty_like(src)
            bad = torch.full((1,), -1, dtype=torch.int64, device=dev)
            w = 65536 // es
            pats = {"identity": lambda: torch.arange(n, device=dev),
                    "random permutation": lambda: torch.randperm(n, device=dev, generator=g),
                    "sortperm(uniform)": None,
                    "shuffled in 64 KiB windows": lambda: torch.argsort(torch.arange(n, device=dev) // w
                                                                        + torch.rand(n, device=dev, generator=g, dtype=torch.float64) * 0.5)}
            for name, make in pats.items():
                if make is None:
                    v = dab.drand((n,), procs=[1], seed=n)
                    p = dab.sortperm(v)
                    idx1 = torch.from_numpy(dab.to_array(p)).to(dev)
                    v.close()
                    p.close()
                    idx0 = idx1 - 1
                else:
                    idx0 = make().to(torch.int64)
                    idx1 = idx0 + 1
                torch.cuda.synchronize()
                dims, grid, cuts = (C.c_size_t * 1)(n), (C.c_int32 * 1)(1), (C.c_size_t * 2)(0, n)
                ptrs = (C.c_void_p * 1)(src.data_ptr())

                def k22():
                    _lib.call("dab_index_gather", rt.ctx, es, C.c_void_p(out.data_ptr()), C.c_void_p(idx1.data_ptr()), _lib.I64, n, 1, dims,
                              grid, cuts, ptrs, C.c_void_p(bad.data_ptr()))

                ref = torch.empty_like(src)

                def tsel():
                    torch.index_select(src, 0, idx0, out=ref)

                ta, tb = timed_pair(rt, k22, tsel)
                rt.sync()
                torch.cuda.synchronize()
                same = torch.equal(out.view(torch.uint8), ref.view(torch.uint8)) and int(bad.item()) == -1
                by = n * (8 + 2 * es)
                print(f"n=2^{n.bit_length() - 1} {np.dtype(T).name:8s} {name:28s} {ta:9.3f} {by / ta / 1e6:8.1f} {tb:16.3f} {by / tb / 1e6:8.1f}"
                      f" {ta / tb:10.3f}  {'equal' if same else 'MISMATCH'}", flush=True)
                assert same, name
                del idx0, idx1, ref
            del src, out
            torch.cuda.empty_cache()


def whole_calls():
    rt = dab.init(workers_per_rank=8, use_dist=False)
    n = 1 << 26
    rng = np.random.default_rng(5)
    v = dab.distribute(rng.standard_normal(n))
    p = dab.sortperm(v)
    new = timed_wall(rt, lambda: v[p])
    old = timed_wall(rt, lambda: v[np.asarray(p) - 1].to_darray(), rounds=3)
    a, b = v[p], v[np.asarray(p) - 1].to_darray()
    same = np.array_equal(dab.to_array(a).view(np.uint64), dab.to_array(b).view(np.uint64))
    print(f"v[p], 2^26 Float64 on 8 workers: {new:.2f} ms; host composition v[asarray(p) - 1].to_darray(): {old:.2f} ms; "
          f"factor {old / new:.1f}x; results {'equal' if same else 'MISMATCH'}", flush=True)
    assert same


if __name__ == "__main__":
    rt = dab.init(workers_per_rank=1, use_dist=False)
    torch.cuda.set_device(rt.device)
    kernel_cases(rt)
    dab.d_closeall()
    whole_calls()
    dab.d_closeall()
