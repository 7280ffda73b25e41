"""K27 against torch.linalg.solve / torch.linalg.det on the same data (CUDA events, medians of 10 after 3 warm-ups).

    python tools/perf_ldiv.py [--gib 1]

For n in {4, 10, 16, 32, 64}, Float32 and Float64, A is a batch of well-conditioned n x n matrices of about --gib GiB and B one vector per
matrix.  Prints one line per case: K27's time, its share of the HBM bound (bytes = A + B read, X written, at 3.35 TB/s), torch's time and
the ratio, and the largest relative difference to torch.  The card name and its power limit are read in the same run.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402

HBM = 3.35e12


def _time(fn, reps=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    rt = dab.init(workers_per_rank=1, use_dist=False)
    ptr = C.c_void_p()
    _lib.call("dab_stream", rt.ctx, C.byref(ptr))
    stream = torch.cuda.ExternalStream(ptr.value)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {smi or torch.cuda.get_device_name(0)}")
    with torch.cuda.stream(stream):                                # K27 runs on the ctx stream: torch and the events share it
        run(rt, args)
    dab.d_closeall()


def run(rt, args):
    for T, tt in ((np.float32, torch.float32), (np.float64, torch.float64)):
        es = np.dtype(T).itemsize
        for n in (4, 10, 16, 32, 64):
            batch = int(args.gib * 2 ** 30 // (n * n * es))
            g = torch.Generator(device="cuda").manual_seed(n)
            A = torch.randn((batch, n, n), device="cuda", dtype=tt, generator=g) / (3 * n ** 0.5) + torch.eye(n, device="cuda", dtype=tt)
            b = torch.randn((batch, n, 1), device="cuda", dtype=tt, generator=g)
            # column-major slices for K27: the (n, n) slice of A.mT is A's row-major storage read column-major
            Acm = A.transpose(1, 2).contiguous()
            X = torch.empty_like(b)
            D = torch.empty((batch,), device="cuda", dtype=tt)
            st = torch.empty((1,), device="cuda", dtype=torch.int64)
            dt = _lib.F32 if T == np.float32 else _lib.F64

            def k27_solve():
                _lib.call("dab_ldiv_batched", rt.ctx, dt, n, 1, C.c_void_p(Acm.data_ptr()), n * n, C.c_void_p(b.data_ptr()), n,
                          C.c_void_p(X.data_ptr()), batch, C.c_void_p(st.data_ptr()))

            def k27_det():
                _lib.call("dab_det_batched", rt.ctx, dt, n, C.c_void_p(Acm.data_ptr()), n * n, C.c_void_p(D.data_ptr()), batch)

            torch.cuda.synchronize()
            t_s = _time(k27_solve)
            t_d = _time(k27_det)
            t_ts = _time(lambda: torch.linalg.solve(A, b))
            t_td = _time(lambda: torch.linalg.det(A))
            torch.cuda.synchronize()
            assert (int(st.item()) & ((1 << 64) - 1)) == (1 << 64) - 1
            xs, dd = torch.linalg.solve(A, b), torch.linalg.det(A)
            err_x = float(((X - xs).abs().amax(dim=(1, 2)) / xs.abs().amax(dim=(1, 2))).max())
            err_d = float(((D - dd).abs() / dd.abs()).max())
            eps = float(np.finfo(T).eps)
            ok = err_x <= 64 * n * eps and err_d <= 64 * n * eps
            bytes_s = batch * (n * n + 2 * n) * es
            bytes_d = batch * (n * n + 1) * es
            print(f"{np.dtype(T).name:7s} n={n:2d} batch={batch:9d}  solve {t_s:8.3f} ms ({bytes_s / (t_s * 1e-3) / HBM:5.1%} of HBM)  "
                  f"torch {t_ts:8.3f} ms  ratio {t_ts / t_s:5.2f}x  |  det {t_d:8.3f} ms ({bytes_d / (t_d * 1e-3) / HBM:5.1%})  "
                  f"torch {t_td:8.3f} ms  ratio {t_td / t_d:5.2f}x  |  max rel diff x {err_x:.1e} det {err_d:.1e} {'ok' if ok else 'MISMATCH'}",
                  flush=True)
            del A, b, Acm, X, D
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
