#!/usr/bin/env python
"""Single-GPU rates of the pair sort K21 (dab_sort_pairs with vals = NULL, the step under sortperm) against the keys-only K11
(dab_sort), the packed-word route (dab_sort_by_key with an Int64 iota as values) and torch.sort(stable=True) (values and indices),
on 2^28 full-range keys of each dtype; then whole sortperm(d) and sort(d) calls on 8 workers for 2^26 Float64 (host clock around the
call, ending in a device synchronise).  CUDA events, every shape warmed up, medians of repeats.  Algorithmic bytes per element
(k = key bytes, P = digit passes: 4 or 8 for full-range keys):
  pairs        k + (k + k + 4) + (P - 2) (2k + 8) + (k + 4 + k + 8)     68 B (32-bit keys), 200 B (64-bit)
  dab_sort     k (1 + 2P)                                               36 B, 136 B
  sort_by_key  12 pack + 136 K11 + 24 gather = 172 B; 64-bit keys, two rounds: 16 + 136 + 24 + 136 + 32 = 344 B
               (K11 on 8-byte words, 8 passes; the iota itself, 8 B more, is not timed)
  torch.sort   k + k + 8 (keys read, keys and indices written: the least any sort moves)
The pair sort's permutation is checked against torch's stable indices, in the same run.  Prints the card's name, power limit and max
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


def timed(rt, fn, reps=5, rounds=5):
    for _ in range(2):
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


def timed_torch(fn, reps=5, rounds=5):
    for _ in range(2):
        fn()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return float(np.median(out))


def timed_wall(rt, fn, rounds=5):
    fn()
    out = []
    for _ in range(rounds):
        rt.sync()
        t0 = time.perf_counter()
        fn()
        rt.sync()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def report(name, ms, per_elem, n):
    gbs = per_elem * n / ms / 1e6
    print(f"{name:44s} {ms:9.3f} ms {gbs:9.1f} GB/s  ({per_elem} B/elem)", flush=True)
    return ms


rt = dab.init(workers_per_rank=1, use_dist=False)
torch.cuda.set_device(0)
n = 1 << 28
p = C.c_void_p
rows = []
for dt in (torch.float32, torch.int32, torch.float64, torch.int64):
    k = torch.empty((), dtype=dt).element_size()
    P = 4 if k == 4 else 8
    if dt.is_floating_point:
        keys = torch.randn(n, dtype=dt, device="cuda")
    else:
        info = torch.iinfo(dt)
        keys = torch.randint(info.min, info.max, (n,), dtype=dt, device="cuda")
    code = {torch.float32: _lib.F32, torch.float64: _lib.F64, torch.int32: _lib.I32, torch.int64: _lib.I64}[dt]
    keys_out = torch.empty_like(keys)
    tmp = torch.empty_like(keys)
    vals_out = torch.empty(n, dtype=torch.int64, device="cuda")
    iota = torch.arange(n, dtype=torch.int64, device="cuda")
    need = C.c_size_t()
    _lib.check(_lib.lib().dab_sort_pairs_scratch_bytes(code, n, C.byref(need)))
    pscratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().dab_sort_by_key_scratch_bytes(code, n, C.byref(need)))
    bscratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def pairs():
        _lib.call("dab_sort_pairs", rt.ctx, code, p(keys.data_ptr()), p(keys_out.data_ptr()), None, 0, p(vals_out.data_ptr()),
                  p(pscratch.data_ptr()), pscratch.numel(), n)

    def keys_only():
        _lib.call("dab_sort", rt.ctx, code, p(keys.data_ptr()), p(keys_out.data_ptr()), p(tmp.data_ptr()), n)

    def by_key():
        _lib.call("dab_sort_by_key", rt.ctx, code, p(keys.data_ptr()), 8, p(iota.data_ptr()), p(vals_out.data_ptr()),
                  p(bscratch.data_ptr()), bscratch.numel(), n)

    name = str(dt).replace("torch.", "")
    t_pairs = report(f"dab_sort_pairs {name} 2^28 (vals = NULL)", timed(rt, pairs), k + (2 * k + 4) + (P - 2) * (2 * k + 8) + (2 * k + 12), n)
    t_keys = report(f"dab_sort {name} 2^28", timed(rt, keys_only), k * (1 + 2 * P), n)
    t_bykey = report(f"dab_sort_by_key {name} 2^28 (Int64 iota)", timed(rt, by_key), 172 if k == 4 else 344, n)
    t_torch = report(f"torch.sort(stable=True) {name} 2^28", timed_torch(lambda: torch.sort(keys, stable=True)), 2 * k + 8, n)
    print(f"  pairs / packed-word route: {t_pairs / t_bykey:.3f}   pairs / dab_sort: {t_pairs / t_keys:.3f}   "
          f"pairs / torch.sort: {t_pairs / t_torch:.3f}", flush=True)
    pairs()
    rt.sync()
    ref = torch.sort(keys, stable=True)
    torch.cuda.synchronize()
    assert torch.equal(vals_out, ref.indices), name                  # no -0.0 or NaN in these keys: torch's stable order is isless'
    assert torch.equal(keys_out, ref.values), name
    rows.append((name, t_pairs, t_keys, t_bykey, t_torch))
    del keys, keys_out, tmp, vals_out, iota, pscratch, bscratch, ref
    torch.cuda.empty_cache()

dab.d_closeall()

rt8 = dab.init(workers_per_rank=8, use_dist=False)
m = 1 << 26
d = dab.drand((m,), dtype=np.float64, seed=5)


def run_sortperm():
    dab.sortperm(d).close()


def run_sort():
    dab.sort(d).close()


t_sp = timed_wall(rt8, run_sortperm)
t_s = timed_wall(rt8, run_sort)
print(f"{'sortperm(d) Float64 2^26, 8 workers':44s} {t_sp:9.3f} ms", flush=True)
print(f"{'sort(d) Float64 2^26, 8 workers':44s} {t_s:9.3f} ms", flush=True)
print(f"  sortperm / sort: {t_sp / t_s:.3f}", flush=True)
dab.d_closeall()
