#!/usr/bin/env python
"""Single-GPU rates of ``d[key] = v`` (row f14) against the torch call that does the same work on the same memory.

  K24  the scatter d[I] = v as the flow runs it on one chunk (dab_fill zeroes the bitmap, dab_scatter_check, dab_scatter) against
       torch.Tensor.index_copy_, n = 2^26 and 2^28 Int64 indices into a Float32 or Float64 destination of n elements, for an identity,
       a uniform random permutation and a permutation shuffled within 64 KiB windows.  Unique indices make index_copy_ deterministic,
       so the outputs are compared bit for bit.  With duplicates (n / 4 distinct targets) the winner pass runs too: reported only.
  K25  whole calls d[m] = v (plan with its device synchronise, then dab_expand) at 2^28 Float32, densities 0.001 / 0.5 / 0.999,
       against masked_scatter_; d[m] = x against masked_fill_; compared bit for bit.
  views  the block write d[a:b, :] = E from a DArray E, against the rate of copy(d) on the same bytes.

CUDA events (host clock to a device synchronise for whole calls), every shape warmed up, the two implementations alternated, medians.
Prints the card's name, power limit and max SM clock, read in the same run."""
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


def timed_pair(rt, fa, fb, reps=5, rounds=7, wall=False):
    """Median ms of fa (dab events on the ctx stream, or the host clock to a synchronise with ``wall``) and fb (torch events),
    alternated round by round."""
    for _ in range(2):
        fa()
        fb()
    ta, tb = [], []
    for _ in range(rounds):
        rt.sync()
        torch.cuda.synchronize()
        if wall:
            t0 = time.perf_counter()
            for _ in range(reps):
                fa()
            rt.sync()
            ta.append((time.perf_counter() - t0) * 1e3 / reps)
        else:
            e0, e1 = rt.event(), rt.event()
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


def k24_cases(rt):
    print(f"{'K24 case':48s} {'K24 ms':>9s} {'index_copy_ ms':>15s} {'K24/torch':>10s}", flush=True)
    dev = torch.device("cuda", rt.device)
    for n in (1 << 26, 1 << 28):
        g = torch.Generator(device=dev)
        g.manual_seed(n)
        for tt in (torch.float32, torch.float64):
            es = torch.empty(0, dtype=tt).element_size()
            src = torch.rand(n, device=dev, generator=g, dtype=torch.float64).to(tt)
            out = torch.zeros(n, device=dev, dtype=tt)
            ref = torch.zeros(n, device=dev, dtype=tt)
            bits = torch.zeros(-(-n // 32), device=dev, dtype=torch.int32)
            win = torch.zeros(n, device=dev, dtype=torch.int32)
            status = torch.tensor([-1, 0], device=dev, dtype=torch.int64)
            lin = torch.zeros(1, device=dev, dtype=torch.int64)
            zero = np.zeros(1, dtype=np.int32)
            w = 65536 // es
            pats = {"identity": lambda: torch.arange(n, device=dev),
                    "random permutation": lambda: torch.randperm(n, device=dev, generator=g),
                    "shuffled in 64 KiB windows": lambda: torch.argsort(torch.arange(n, device=dev) // w
                                                                        + torch.rand(n, device=dev, generator=g, dtype=torch.float64) * 0.5),
                    "duplicates (n/4 targets)": lambda: torch.randint(0, n // 4, (n,), device=dev, generator=g)}
            dims, grid, cuts = (C.c_size_t * 1)(n), (C.c_int32 * 1)(1), (C.c_size_t * 2)(0, n)
            dptr, bptr, wptr = (C.c_void_p * 1)(out.data_ptr()), (C.c_void_p * 1)(bits.data_ptr()), (C.c_void_p * 1)(win.data_ptr())
            for name, make in pats.items():
                idx0 = make().to(torch.int64)
                idx1 = idx0 + 1
                dup = name.startswith("dup")
                torch.cuda.synchronize()

                def k24():
                    _lib.call("dab_fill", rt.ctx, _lib.I32, C.c_void_p(bits.data_ptr()), bits.numel(), C.c_void_p(zero.ctypes.data))
                    _lib.call("dab_scatter_check", rt.ctx, C.c_void_p(idx1.data_ptr()), _lib.I64, n, 1, dims, grid, cuts, bptr,
                              C.c_void_p(status.data_ptr()))
                    if dup:
                        _lib.call("dab_fill", rt.ctx, _lib.I32, C.c_void_p(win.data_ptr()), n, C.c_void_p(zero.ctypes.data))
                        _lib.call("dab_scatter_winners", rt.ctx, C.c_void_p(idx1.data_ptr()), _lib.I64, n, n, C.c_void_p(lin.data_ptr()), 4, 1,
                                  dims, grid, cuts, wptr)
                    _lib.call("dab_scatter", rt.ctx, es, C.c_void_p(idx1.data_ptr()), _lib.I64, n, C.c_void_p(src.data_ptr()), None, n,
                              C.c_void_p(lin.data_ptr()), 4 if dup else 0, 1, dims, grid, cuts, dptr, wptr if dup else None)

                def tcopy():
                    ref.index_copy_(0, idx0, src)

                ta, tb = timed_pair(rt, k24, tcopy)
                rt.sync()
                torch.cuda.synchronize()
                flag = status.cpu().numpy().view(np.uint64)
                if dup:
                    same = "report only"
                else:
                    same = "equal" if torch.equal(out.view(torch.uint8), ref.view(torch.uint8)) and flag[0] == np.uint64(2**64 - 1) else "MISMATCH"
                print(f"n=2^{n.bit_length() - 1} {str(tt)[6:]:8s} {name:30s} {ta:9.3f} {tb:15.3f} {ta / tb:10.3f}  {same}", flush=True)
                assert same != "MISMATCH", name
                del idx0, idx1
            del src, out, ref, bits, win
            torch.cuda.empty_cache()


def k25_cases(rt):
    n = 1 << 28
    dev = torch.device("cuda", rt.device)
    d = dab.dzeros((n,), procs=[1], dtype=np.float32)
    D = torch.zeros(n, device=dev, dtype=torch.float32)
    chunk = d.chunks[1]
    print(f"{'K25 case (whole calls)':48s} {'d[m]=v ms':>9s} {'torch ms':>15s} {'ratio':>10s}", flush=True)
    for density in (0.001, 0.5, 0.999):
        mh = torch.rand(n, device=dev, dtype=torch.float32) < density
        m = dab.dzeros((n,), procs=[1], dtype=np.bool_)
        torch.cuda.synchronize()
        _lib.call("dab_d2d", rt.ctx, C.c_void_p(m.chunks[1].ptr), C.c_void_p(mh.data_ptr()), n)
        cnt = int(mh.sum().item())
        vh = torch.rand(cnt, device=dev, dtype=torch.float32)
        v = dab.dzeros((cnt,), procs=[1], dtype=np.float32)
        torch.cuda.synchronize()                                  # the copies below run on the library's stream
        _lib.call("dab_d2d", rt.ctx, C.c_void_p(v.chunks[1].ptr), C.c_void_p(vh.data_ptr()), 4 * cnt)
        rt.sync()

        def ours():
            d[m] = v

        def theirs():
            D.masked_scatter_(mh, vh)

        ta, tb = timed_pair(rt, ours, theirs, reps=3, rounds=5, wall=True)
        got = torch.empty_like(D)
        _lib.call("dab_d2d", rt.ctx, C.c_void_p(got.data_ptr()), C.c_void_p(chunk.ptr), 4 * n)
        rt.sync()
        same = "equal" if torch.equal(got.view(torch.uint8), D.view(torch.uint8)) else "MISMATCH"
        print(f"d[m] = v, 2^28 Float32, density {density:<6} vs masked_scatter_  {ta:9.3f} {tb:15.3f} {ta / tb:10.3f}  {same}", flush=True)
        assert same == "equal"
        ta, tb = timed_pair(rt, lambda: d.__setitem__(m, np.float32(0.25)), lambda: D.masked_fill_(mh, 0.25), reps=3, rounds=5, wall=True)
        _lib.call("dab_d2d", rt.ctx, C.c_void_p(got.data_ptr()), C.c_void_p(chunk.ptr), 4 * n)
        rt.sync()
        same = "equal" if torch.equal(got.view(torch.uint8), D.view(torch.uint8)) else "MISMATCH"
        print(f"d[m] = x, 2^28 Float32, density {density:<6} vs masked_fill_      {ta:9.3f} {tb:15.3f} {ta / tb:10.3f}  {same}", flush=True)
        assert same == "equal"
        m.close()
        v.close()
        del mh, vh, got
    d.close()
    del D
    torch.cuda.empty_cache()


def view_case(rt):
    rows, cols = 1 << 14, 1 << 14                                 # 2^28 Float32
    d = dab.dzeros((rows, cols), procs=[1], dtype=np.float32)
    E = dab.drand((rows // 2, cols), procs=[1], dtype=np.float32)
    a, b = rows // 4, rows // 4 + rows // 2

    def block():
        d[a:b, :] = E

    def cp():
        dab.copy(E).close()

    for _ in range(2):
        block()
        cp()
    tw, tc = [], []
    for _ in range(5):
        for f, acc in ((block, tw), (cp, tc)):
            rt.sync()
            t0 = time.perf_counter()
            f()
            rt.sync()
            acc.append((time.perf_counter() - t0) * 1e3)
    tw, tc = float(np.median(tw)), float(np.median(tc))
    by = 2 * 4 * (b - a) * cols
    print(f"d[a:b, :] = E, 2^27 Float32 elements: {tw:.3f} ms ({by / tw / 1e6:.0f} GB/s); copy(E): {tc:.3f} ms ({by / tc / 1e6:.0f} GB/s)",
          flush=True)
    ok = np.array_equal(np.asarray(d[a:a + 3, 0:5]), np.asarray(E[0:3, 0:5]))
    print("block write equals its source:", ok, flush=True)
    assert ok
    d.close()
    E.close()


if __name__ == "__main__":
    rt = dab.init(workers_per_rank=1, use_dist=False)
    torch.cuda.set_device(rt.device)
    k24_cases(rt)
    k25_cases(rt)
    view_case(rt)
    dab.d_closeall()
