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
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("bf16_tflops", 1590.0) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 1590.0
    shapes = [(4096, 4096, 4096), (8192, 8192, 8192), (16384, 8192, 4096), (8192, 128, 8192)]
    for (m, n, k) in shapes:
        A = dab.drand((m, k), dtype=np.float32, seed=1)
        B = dab.drand((k, n), dtype=np.float32, seed=2)
        Cc = dab.B200Array.empty(rt, (m, n), np.float32)
        a, b = dab.localpart(A), dab.localpart(B)
        simt = m * n * k <= 2 ** 37
        if simt:   # the SIMT kernel serves a leading dimension TMA cannot address: A copied into m + 1 rows
            Ap = dab.B200Array.empty(rt, (m + 1, k), np.float32)
            z4 = _lib.sz4((0, 0, 0, 0))
            _lib.call("dab_copy_box", rt.ctx, 4, C.c_void_p(Ap.ptr), _lib.sz4((m + 1, k)), z4, C.c_void_p(a.ptr), _lib.sz4((m, k)), z4, _lib.sz4((m, k)))
        for kernel, pa, lda in [("wgmma_3xtf32", a.ptr, m)] + ([("simt", Ap.ptr, m + 1)] if simt else []):
            call = lambda: _lib.call("dab_gemm", rt.ctx, _lib.F32, 0, m, n, k, C.c_void_p(pa), lda, C.c_void_p(b.ptr), k, C.c_void_p(Cc.ptr), m)
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
            tc = kernel != "simt"
            print(json.dumps({"kernel": kernel, "m": m, "n": n, "k": k, "ms": round(ms, 4), "useful_TFLOPs": round(tf, 1),
                              "tf32_mma_TFLOPs": round(3 * tf, 1) if tc else None, "frac_of_bf16_peak_div2_div3": round(tf / (peak / 2 / 3), 3) if tc else None,
                              "max_rel_err_vs_fp64": worst}), flush=True)
        if simt:
            Ap.free()
        Cc.free()
        A.close()
        B.close()


if __name__ == "__main__":
    main()
