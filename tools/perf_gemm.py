#!/usr/bin/env python
"""K12 timing: dab_gemm (wgmma 3xTF32) on square and chunk-shaped Float32 problems, the SIMT kernel beside it; error vs fp64 on a slice."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import darray_b200 as dab  # noqa: E402
from darray_b200 import _lib  # noqa: E402


def main():
    rt = dab.init(use_dist=False)
    if os.environ.get("GEMM_KC"):
        rt.set_option("gemm_kc", int(os.environ["GEMM_KC"]))
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("bf16_tflops", 1590.0) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 1590.0
    shapes = [(4096, 4096, 4096), (8192, 8192, 8192), (16384, 8192, 4096), (8192, 128, 8192)]
    if os.environ.get("GEMM_KC"):
        shapes = [(8192, 8192, 8192)]
    for (m, n, k) in shapes:
        A = dab.drand((m, k), dtype=np.float32, seed=1)
        B = dab.drand((k, n), dtype=np.float32, seed=2)
        Cc = dab.B200Array.empty(rt, (m, n), np.float32)
        a, b = dab.localpart(A), dab.localpart(B)
        for simt in (0, 2, 1):
            if simt == 1 and m * n * k > 2 ** 37:
                continue
            rt.set_option("gemm_simt", 1 if simt == 1 else 0)
            rt.set_option("gemm_rawhi", 1 if simt == 2 else 0)
            call = lambda: _lib.call("dab_gemm", rt.ctx, _lib.F32, 0, m, n, k, C.c_void_p(a.ptr), m, C.c_void_p(b.ptr), k, C.c_void_p(Cc.ptr), m)
            for _ in range(2):
                call()
            e0, e1 = rt.event(), rt.event()
            rt.sync()
            reps = 5
            rt.record(e0)
            for _ in range(reps):
                call()
            rt.record(e1)
            ms = rt.elapsed_ms(e0, e1) / reps
            tf = 2.0 * m * n * k / ms / 1e9
            # error on a 64 x 64 corner vs fp64 from the regenerated inputs
            from oracle import core as ocore
            rows = 64
            Ah = np.stack([ocore.rand_u01_f32(1, j * m, rows) for j in range(k)], axis=1).astype(np.float64)       # A[:64, :]
            Bh = np.stack([ocore.rand_u01_f32(2, j * k, k) for j in range(64)], axis=1).astype(np.float64)         # B[:, :64]
            want = Ah @ Bh
            host = np.empty((rows,), dtype=np.float32)
            worst = 0.0
            for j in range(0, 64, 21):
                _lib.call("dab_d2h", rt.ctx, C.c_void_p(host.ctypes.data), C.c_void_p(Cc.ptr + 4 * j * m), 4 * rows)
                rt.sync()
                worst = max(worst, float(np.abs(host - want[:, j]).max() / np.abs(want[:, j]).min()))
            print(json.dumps({"kernel": {0: "wgmma_3xtf32", 1: "simt", 2: "wgmma_3xtf32_rawhi"}[simt], "m": m, "n": n, "k": k, "ms": round(ms, 4), "useful_TFLOPs": round(tf, 1),
                              "tf32_mma_TFLOPs": round(3 * tf, 1) if simt != 1 else None, "frac_of_bf16_peak_div2_div3": round(tf / (peak / 2 / 3), 3) if simt != 1 else None,
                              "max_rel_err_vs_fp64": worst}), flush=True)
        rt.set_option("gemm_simt", 0)
        rt.set_option("gemm_rawhi", 0)
        Cc.free()
        A.close()
        B.close()


if __name__ == "__main__":
    main()
