#!/usr/bin/env python
"""The bench step (y .= a.*x .+ b, then s = sum(y)) with and without the fused map-store-reduce kernel, in one process.

A fused round runs the step as bench.py does: dab_affine is deferred and sum(y) consumes it (one kernel, 8 B/element).  A flushed
round is identical except for rt.launches() between broadcast_into and sum: dab_launch_count queues the deferred affine without a
sync, which reproduces the unfused launch sequence (broadcast kernel, then reduce kernel: 12 B/element).  Rounds alternate, each is
timed with CUDA events over --steps steps like bench.py, and both modes must produce the same sum bit for bit.

  python tools/perf_fused_step.py [--log2n 30 31] [--rounds 5] [--steps 20] [--profile DIR]

--profile DIR adds a separate torch.profiler run per size (written under DIR): the per-step kernel time of each mode and the host
gap between steps (step time minus kernel time).  Prints a table and one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402

A_COEF, B_COEF, SEED = 1.5, 0.25, 1234


def card(rt):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(rt.device), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as ex:  # the numbers below are still printed; the card line says why it is missing
        return {"error": repr(ex)[:200]}


def profile_kernels(rt, run, steps, trace_path):
    """Mean device time per step of every kernel `run` launches, from torch.profiler (CUPTI sees every kernel in the process)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    rt.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        rt.sync()
    prof.export_chrome_trace(trace_path)
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t > 0:
            per[ev.key] = per.get(ev.key, 0.0) + t / 1e3 / steps
    return per


def short(name):
    if "AffineStore" in name:
        return "reduce_kernel<float, ..., AffineStore<float>> (fused)"
    if "reduce_kernel" in name:
        return "reduce_kernel<float, ...> (plain)"
    if "ew1_kernel" in name:
        return "ew1_kernel<float, AffineF<float>, 2>"
    return name[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, nargs="+", default=[30, 31])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--profile", metavar="DIR")
    args = ap.parse_args()
    rounds = max(5, args.rounds)
    rt = dab.init(workers_per_rank=1, use_dist=False)
    a, b = np.float32(A_COEF), np.float32(B_COEF)
    f = lambda v: a * v + b  # noqa: E731
    info = card(rt)
    print(f"card: {info}", flush=True)
    result = {"card": info, "rounds": rounds, "steps": args.steps, "sizes": {}}
    for log2n in args.log2n:
        n = 1 << log2n
        x = dab.drand((n,), dtype=np.float32, seed=SEED)
        y = dab.similar(x)

        def fused():
            dab.broadcast_into(y, f, x)
            return dab.sum(y)

        def flushed():
            dab.broadcast_into(y, f, x)
            rt.launches()
            return dab.sum(y)

        def timed(fn):
            rt.sync()
            e0, e1 = rt.event(), rt.event()
            rt.record(e0)
            s = None
            for _ in range(args.steps):
                s = fn()
            rt.record(e1)
            ms = rt.elapsed_ms(e0, e1) / args.steps
            rt.event_destroy(e0)
            rt.event_destroy(e1)
            return ms, s

        for _ in range(max(8, (160 >> max(0, log2n - 30)) // 2)):   # ~0.3 s of warm-up in each mode: clocks and pools settle
            fused()
            flushed()
        l0 = rt.launches()
        fused()
        l_fused = rt.launches() - l0
        l0 = rt.launches()
        flushed()
        l_flushed = rt.launches() - l0
        times = {"fused": [], "flushed": []}
        sums = {"fused": set(), "flushed": set()}
        for r in range(rounds):
            order = ("fused", "flushed") if r % 2 == 0 else ("flushed", "fused")
            for mode in order:
                ms, s = timed(fused if mode == "fused" else flushed)
                times[mode].append(ms)
                sums[mode].add(np.float32(s).tobytes())
        st = {m: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "all_ms": v} for m, v in times.items()}
        ratio = st["flushed"]["median_ms"] / st["fused"]["median_ms"]
        disjoint = st["fused"]["max_ms"] < st["flushed"]["min_ms"]
        same = len(sums["fused"] | sums["flushed"]) == 1
        entry = {"n": n, "launches_per_step": {"fused": l_fused, "flushed": l_flushed}, "modes": st, "ratio_median": ratio,
                 "ranges_disjoint": disjoint, "sum_bit_identical": same,
                 "value_GBs": {m: 12.0 * n / (st[m]["median_ms"] * 1e-3) / 1e9 for m in st},
                 "hbm_GBs": {"fused": 8.0 * n / (st["fused"]["median_ms"] * 1e-3) / 1e9,
                             "flushed": 12.0 * n / (st["flushed"]["median_ms"] * 1e-3) / 1e9}}
        print(f"2^{log2n} Float32 ({4 * n / 2**30:.0f} GiB per array), {rounds} alternating rounds x {args.steps} steps, launches/step "
              f"fused {l_fused} flushed {l_flushed}", flush=True)
        for m in ("fused", "flushed"):
            print(f"  {m:8s} median {st[m]['median_ms']:.4f} ms/step  min {st[m]['min_ms']:.4f}  max {st[m]['max_ms']:.4f}   "
                  f"value-equivalent {entry['value_GBs'][m]:7.1f} GB/s (12 B/elem credited), HBM traffic {entry['hbm_GBs'][m]:7.1f} GB/s",
                  flush=True)
        print(f"  ratio flushed/fused (median) {ratio:.3f}; ranges disjoint: {disjoint}; sum bit-identical across modes: {same}", flush=True)
        if args.profile:
            os.makedirs(args.profile, exist_ok=True)
            prof = {}
            for mode, fn in (("fused", fused), ("flushed", flushed)):
                per = profile_kernels(rt, fn, args.steps, os.path.join(args.profile, f"fused_step_{mode}_2p{log2n}.pt.trace.json"))
                kern = {short(k): v for k, v in per.items()}
                k_ms = sum(per.values())
                prof[mode] = {"kernels_ms_per_step": kern, "kernel_ms_per_step": k_ms,
                              "host_gap_ms_per_step": st[mode]["median_ms"] - k_ms}
                print(f"  profile {mode}: " + ", ".join(f"{k} {v:.4f} ms" for k, v in kern.items()) +
                      f"; host gap {st[mode]['median_ms'] - k_ms:.4f} ms/step (event step time minus kernel time)", flush=True)
            fk = [v for k, v in prof["fused"]["kernels_ms_per_step"].items() if "fused" in k]
            if fk:
                prof["fused"]["fused_kernel_GBs_8B_per_elem"] = 8.0 * n / (fk[0] * 1e-3) / 1e9
                print(f"  fused kernel: {fk[0]:.4f} ms, {prof['fused']['fused_kernel_GBs_8B_per_elem']:.1f} GB/s on 8 B/elem", flush=True)
            entry["profile"] = prof
        result["sizes"][f"2^{log2n}"] = entry
        x.close()
        y.close()
    print(json.dumps(result), flush=True)
    dab.d_closeall()
    rt.shutdown()


if __name__ == "__main__":
    main()
