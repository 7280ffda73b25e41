#!/usr/bin/env python
"""Single-GPU times of K26 (dab_sortperm_slices, the chunk step of sortperm(A; dims)) against its yardsticks, on 2^28 elements:
  * K13 (dab_sort_slices, the chunk step of sort(A; dims) = mapslices(sort, A, dims)) on the same chunk,
  * torch.sort(dim=..., stable=True) on the same data (values and indices),
  * for fibres longer than DAB_SORTPERM_SLICES_SMEM_LEN also K21 (dab_sort_pairs, the chunk step of sortperm(v) of a DVector) on all
    2^28 keys as one vector.
Fibres of 32, 1024, 4096 (the shared-memory limit) and 65536 elements, along dims=1 (contiguous fibres) and dims=2 (strided fibres), for
Float32 and Float64 uniform keys in [0, 1) (no NaNs, no signed zeros: torch's stable order is then isless, and K26's indices are
checked against torch's, mapped to global linear indices, in the same run).  CUDA events, every shape warmed up, each case alternated
with its yardsticks, medians of the rounds.  Prints the card's name, power limit and max SM clock, read in the same run."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)

LOG2N = int(os.environ.get("PERF_SORT_DIMS_LOG2N", "28"))
N = 1 << LOG2N
ROUNDS, REPS = 5, 3


def ms(rt, fn):
    e0, e1 = rt.event(), rt.event()
    rt.sync()
    rt.record(e0)
    for _ in range(REPS):
        fn()
    rt.record(e1)
    rt.sync()
    t = rt.elapsed_ms(e0, e1) / REPS
    rt.event_destroy(e0)
    rt.event_destroy(e1)
    return t


def ms_torch(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


def main():
    rt = dab.init(workers_per_rank=1, use_dist=False)
    for T, tt in ((np.float32, torch.float32), (np.float64, torch.float64)):
        g = torch.Generator(device="cuda").manual_seed(1)
        tkeys = torch.rand(N, device="cuda", dtype=tt, generator=g)
        keys = dab.B200Array.from_numpy(rt, tkeys.cpu().numpy())
        perm = dab.B200Array.empty(rt, (N,), np.int64)
        srt = dab.B200Array.empty(rt, (N,), T)
        need = C.c_size_t()
        _lib.check(_lib.lib().dab_sort_pairs_scratch_bytes(dab.dab_dtype(T), N, C.byref(need)))
        pscr = dab.B200Array.empty(rt, (need.value,), np.uint8)
        kout = dab.B200Array.empty(rt, (N,), T)
        for ln in (32, 1024, _lib.SORTPERM_SLICES_SMEM_LEN, 1 << 16):
            m = N // ln
            for dim in (1, 2):
                shape = (ln, m) if dim == 1 else (m, ln)
                inner, outer = (1, m) if dim == 1 else (m, 1)
                SZ = C.c_size_t * 2

                def k26():
                    _lib.call("dab_sortperm_slices", rt.ctx, dab.dab_dtype(T), C.c_void_p(keys.ptr), 2, SZ(*shape), SZ(0, 0), SZ(*shape), dim,
                              C.c_void_p(perm.ptr), 0, None, None)

                def k13():
                    _lib.call("dab_sort_slices", rt.ctx, dab.dab_dtype(T), C.c_void_p(keys.ptr), C.c_void_p(srt.ptr), inner, ln, outer)

                tv = tkeys.view(m, ln) if dim == 1 else tkeys.view(ln, m)
                tdim = 1 if dim == 1 else 0

                def tsort():
                    return torch.sort(tv, dim=tdim, stable=True)

                def k21():
                    _lib.call("dab_sort_pairs", rt.ctx, dab.dab_dtype(T), C.c_void_p(keys.ptr), C.c_void_p(kout.ptr), None, 1,
                              C.c_void_p(perm.ptr), C.c_void_p(pscr.ptr), need.value, N)

                # correctness against torch's stable indices, mapped to global linear indices
                k26()
                rt.sync()
                idx = tsort()[1].to(torch.int64)
                if dim == 1:
                    want = idx + 1 + ln * torch.arange(m, device="cuda", dtype=torch.int64).view(m, 1)
                else:
                    want = 1 + torch.arange(m, device="cuda", dtype=torch.int64).view(1, m) + m * idx
                got = torch.from_numpy(perm.to_numpy()).cuda()
                ok = bool(torch.equal(got, want.reshape(-1)))
                del idx, want, got
                fns = {"sortperm K26": lambda: ms(rt, k26), "sort K13": lambda: ms(rt, k13), "torch.sort": lambda: ms_torch(tsort)}
                if ln > _lib.SORTPERM_SLICES_SMEM_LEN:
                    fns["DVector sortperm K21"] = lambda: ms(rt, k21)
                for f in fns.values():                           # warm every shape
                    f()
                times = {k: [] for k in fns}
                for _ in range(ROUNDS):                          # alternate the case with its yardsticks
                    for k, f in fns.items():
                        times[k].append(f())
                med = {k: float(np.median(v)) for k, v in times.items()}
                ratio = med["sortperm K26"] / med["sort K13"]
                extra = ""
                if "DVector sortperm K21" in med:
                    extra = f"  vs K21 {med['sortperm K26'] / med['DVector sortperm K21']:.2f}x"
                print(f"{np.dtype(T).name:8s} len {ln:6d} dims={dim}: " + "  ".join(f"{k} {v:8.3f} ms" for k, v in med.items())
                      + f"  K26/K13 {ratio:.2f}x{extra}  indices == torch: {ok}", flush=True)
        for b in (keys, perm, srt, pscr, kout):
            b.free()
        del tkeys
        torch.cuda.empty_cache()
    dab.d_closeall()


if __name__ == "__main__":
    main()
