#!/usr/bin/env python
"""Single-GPU times of the stream compaction K23 behind d[mask] and findall(mask), as whole calls on one worker (count, tile scans,
host plan, compaction), against dab.copy(d) (the identity broadcast: one read and one write of d) and torch.masked_select /
torch.nonzero on the same device memory (the tensors alias the DArray's chunks).

Cases: n = 2^28 and 2^30 Float32 and Float64 elements, masks x < t of uniform data at densities 0.001, 0.5 and 0.999.  Algorithmic
bytes: n * (2 + s) + count * s for d[mask] (the mask is read twice, the values once, the selected values written once; s = element
size) and n * 2 + count * 8 for findall.  Every call ends in a device synchronise (the output length is data-dependent, so each of
the four calls synchronises inside too); host clock, every shape warmed up, the calls alternated, medians of repeats.  Results are
compared bit for bit with torch's in the same run.  Prints the card's name, power limit and max SM clock, read in the same run."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import darray_b200 as dab  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)


class _Dev:
    """A torch view of one DArray chunk (``__cuda_array_interface__``): torch's kernels read the same bytes."""

    def __init__(self, ch):
        self.__cuda_array_interface__ = {"shape": (ch.size,), "typestr": ch.dtype.str, "data": (ch.ptr, False), "version": 3}


def timed(rt, fns, rounds=7):
    """Median ms of each function, host clock around the call and a synchronise of both streams, alternated round by round."""
    for f in fns:
        f()
    out = [[] for _ in fns]
    for _ in range(rounds):
        for i, f in enumerate(fns):
            rt.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            rt.sync()
            torch.cuda.synchronize()
            out[i].append((time.perf_counter() - t0) * 1e3)
    return [float(np.median(o)) for o in out]


def main():
    rt = dab.init(workers_per_rank=1, use_dist=False)
    dev = torch.device("cuda", rt.device)
    torch.cuda.set_device(dev)
    print(f"{'case':34s} {'d[m] ms':>9s} {'GB/s':>7s} {'masked_select':>14s} {'ratio':>6s} {'findall ms':>11s} {'GB/s':>7s} {'nonzero':>9s}"
          f" {'ratio':>6s} {'copy ms':>8s} {'GB/s':>7s}", flush=True)
    for n in (1 << 28, 1 << 30):
        for T in (np.float32, np.float64):
            s = np.dtype(T).itemsize
            d = dab.drand((n,), procs=[1], dtype=T, seed=n)
            td = torch.as_tensor(_Dev(d.chunks[1]), device=dev)
            copy_ms = timed(rt, [lambda: dab.copy(d).close()])[0]
            for density in (0.001, 0.5, 0.999):
                m = dab.broadcast(lambda x: x < T(density), d)
                tm = torch.as_tensor(_Dev(m.chunks[1]), device=dev)
                t_ours, t_sel, t_idx, t_nz = timed(rt, [lambda: d[m].close(), lambda: torch.masked_select(td, tm),
                                                        lambda: dab.findall(m).close(), lambda: torch.nonzero(tm)])
                R = d[m]
                cnt = R.dims[0]
                r = torch.masked_select(td, tm)
                same = cnt == r.numel() and (not cnt or torch.equal(torch.as_tensor(_Dev(R.chunks[1]), device=dev).view(torch.uint8),
                                                                    r.view(torch.uint8)))
                R.close()
                del r
                F = dab.findall(m)
                f = torch.nonzero(tm).reshape(-1)
                same_idx = F.dims[0] == cnt and (not cnt or torch.equal(torch.as_tensor(_Dev(F.chunks[1]), device=dev) - 1, f))
                F.close()
                del f
                by = n * (2 + s) + cnt * s
                by_idx = n * 2 + cnt * 8
                print(f"n=2^{n.bit_length() - 1} {np.dtype(T).name:8s} density {density:<6} {t_ours:9.3f} {by / t_ours / 1e6:7.1f}"
                      f" {t_sel:14.3f} {t_ours / t_sel:6.2f} {t_idx:11.3f} {by_idx / t_idx / 1e6:7.1f} {t_nz:9.3f} {t_idx / t_nz:6.2f}"
                      f" {copy_ms:8.3f} {2 * n * s / copy_ms / 1e6:7.1f}  {'equal' if same and same_idx else 'MISMATCH'}", flush=True)
                assert same and same_idx
                m.close()
                del tm
                torch.cuda.empty_cache()
            del td
            d.close()


if __name__ == "__main__":
    main()
