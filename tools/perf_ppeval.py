#!/usr/bin/env python
"""Rates of the two ppeval kernels on one GPU, with CUDA events after a warm-up, and the card's name and power limit read in the same run.

  dab_matmul_batched       matrix x vector at 2^16 slices of 10x10, 64x64 and 256x256, Float64 and Float32: GB/s on the bytes of A, B
                           and C, and the share of the 3.35 TB/s H100 SXM data sheet; matrix x matrix at 32x32x32 and 256x256x256:
                           GFLOP/s on 2mnk per slice.  Yardsticks in the same run: torch.bmm on the same bytes (the column-major slices
                           read as transposed row-major ones), and a per-slice dab_gemm loop at 64x64x64.
  dab_eigvals_sym_batched  matrices/s for 2^16 random symmetric Float64 matrices of 8x8, 10x10, 32x32 and 64x64, against
                           torch.linalg.eigvalsh on the same batch (in 16 calls of 4096: cusolver refuses 2^16 in one).
Operands are generated on the device by torch and handed to the kernels as raw pointers.
Run: python tools/perf_ppeval.py  (needs a GPU; prints one line per measurement)."""
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
    return subprocess.run(["nvidia-smi", "-i", str(rt.device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


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


def torch_timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(reps):
        fn()
    s1.record()
    torch.cuda.synchronize()
    return s0.elapsed_time(s1) / reps


print("card:", card(), flush=True)
import torch  # noqa: E402

torch.manual_seed(0)
TT = {np.float32: torch.float32, np.float64: torch.float64}


def bmm(T, m, n, k, batch, yard=True):
    es = np.dtype(T).itemsize
    A = torch.randn(batch * m * k, dtype=TT[T], device="cuda")
    B = torch.randn(batch * k * n, dtype=TT[T], device="cuda")
    Cm = torch.empty(batch * m * n, dtype=TT[T], device="cuda")
    code = dab.dab_dtype(np.dtype(T))
    torch.cuda.synchronize()                                       # the operands exist before the library's stream reads them
    fn = lambda: _lib.call("dab_matmul_batched", rt.ctx, code, m, n, k, C.c_void_p(A.data_ptr()), m * k, C.c_void_p(B.data_ptr()), k * n,  # noqa: E731
                           C.c_void_p(Cm.data_ptr()), batch)
    ms = timed(fn)
    # the same product in torch: column-major A_b (m x k) is row-major (k x m), i.e. A_b^T; C_b^T = B_b^T A_b^T
    At, Bt, Ct = A.view(batch, k, m), B.view(batch, n, k), torch.empty(batch, n, m, dtype=TT[T], device="cuda")
    tms = torch_timed(lambda: torch.bmm(Bt, At, out=Ct)) if yard else float("nan")
    rt.sync()
    ref = torch.bmm(Bt.double(), At.double()).reshape(-1) if batch * m * n <= (1 << 27) else None
    if ref is not None:
        err = (Cm.double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-300)
    else:
        err = float("nan")
    del A, B, Cm, At, Bt, Ct
    torch.cuda.empty_cache()
    return ms, tms, es, err


for T in (np.float64, np.float32):
    for s in (10, 64, 256):
        batch = 1 << 16
        ms, tms, es, err = bmm(T, s, 1, s, batch)
        gbs = (s * s + s + s) * es * batch / ms / 1e6
        print(f"matmul_batched {np.dtype(T).name} matvec {s}x{s} x {batch}: {ms:8.3f} ms {gbs:7.0f} GB/s ({gbs * 1e9 / HBM:5.1%} of 3.35 TB/s); "
              f"torch.bmm {tms:8.3f} ms -> torch/ours {tms / ms:5.2f}; max rel err {err:.1e}", flush=True)
    for s, batch in ((32, 1 << 16), (256, 1 << 11)):
        ms, tms, es, err = bmm(T, s, s, s, batch)
        gf = 2.0 * s * s * s * batch / ms / 1e6
        print(f"matmul_batched {np.dtype(T).name} matmat {s}x{s}x{s} x {batch}: {ms:8.3f} ms {gf:9.0f} GFLOP/s; torch.bmm {tms:8.3f} ms "
              f"-> torch/ours {tms / ms:5.2f}; max rel err {err:.1e}", flush=True)
    # per-slice dab_gemm loop at 64x64x64 (the path a batched kernel replaces)
    s, nb = 64, 1024
    A = torch.randn(nb * s * s, dtype=TT[T], device="cuda")
    B = torch.randn(nb * s * s, dtype=TT[T], device="cuda")
    Cm = torch.empty(nb * s * s, dtype=TT[T], device="cuda")
    es = np.dtype(T).itemsize
    code = dab.dab_dtype(np.dtype(T))
    torch.cuda.synchronize()

    def loop():
        for b in range(nb):
            o = b * s * s * es
            _lib.call("dab_gemm", rt.ctx, code, 0, s, s, s, C.c_void_p(A.data_ptr() + o), s, C.c_void_p(B.data_ptr() + o), s,
                      C.c_void_p(Cm.data_ptr() + o), s)

    ms_loop = timed(loop, reps=2)
    ms_b = timed(lambda: _lib.call("dab_matmul_batched", rt.ctx, code, s, s, s, C.c_void_p(A.data_ptr()), s * s, C.c_void_p(B.data_ptr()),
                                   s * s, C.c_void_p(Cm.data_ptr()), nb))
    print(f"matmul_batched {np.dtype(T).name} {nb} x 64x64x64: {ms_b:8.3f} ms; per-slice dab_gemm loop {ms_loop:8.3f} ms -> "
          f"{ms_loop / ms_b:6.1f}x", flush=True)
    del A, B, Cm
    torch.cuda.empty_cache()

B = 1 << 16
for n in (8, 10, 32, 64):
    X = torch.randn(B, n, n, dtype=torch.float64, device="cuda")
    S = (X + X.transpose(1, 2)).contiguous()
    W = torch.empty(B * n, dtype=torch.float64, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ms = timed(lambda: _lib.call("dab_eigvals_sym_batched", rt.ctx, _lib.F64, C.c_void_p(S.data_ptr()), n, B, C.c_void_p(W.data_ptr()),
                                 C.c_void_p(st.data_ptr())), reps=3)
    # torch in calls of 4096 matrices: cusolver's batched syev refuses the whole 2^16 batch (CUSOLVER_STATUS_INVALID_VALUE)
    out = []
    tms = torch_timed(lambda: out.append(torch.cat([torch.linalg.eigvalsh(S[i:i + 4096]) for i in range(0, B, 4096)])), reps=1, warm=1)
    rt.sync()
    ref = out[-1].reshape(-1)
    err = (W - ref).abs().max().item() / ref.abs().max().item()
    print(f"eigvals_sym_batched Float64 {B} x {n}x{n}: {ms:8.3f} ms {B / ms * 1e3:12.0f} matrices/s; torch.linalg.eigvalsh (16 calls) {tms:8.3f} ms "
          f"{B / tms * 1e3:12.0f} matrices/s -> torch/ours {tms / ms:5.2f}; status {int(st.item())}; max rel err {err:.1e}", flush=True)
    del X, S, W, st
    torch.cuda.empty_cache()
dab.d_closeall()
rt.shutdown()
