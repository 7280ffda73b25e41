#!/usr/bin/env python
"""Single-GPU rates of the sparse tile products (K18 dab_spmv, K19 dab_csc_to_csr) on one Float64 chunk, for three seeded host-built
matrices: a 5-point Laplacian on a 4096^2 grid, 32 entries in every column of a 2^22 x 2^22 matrix, and a matrix with power-law row lengths.
For each: the K19 build time, the A*x and A'*x kernel times (CUDA events, medians after warm-up), GB/s on the algorithmic bytes
nnz*(4 + sizeof T) + 8*(rows + 1) + sizeof T*(m + n) (x counted once: the minimum), torch's cuSPARSE CSR product on the same matrix as a
yardstick, and a bit check of sampled rows against the ordered-fold model.  Prints the card's name, power limit and max SM clock, read in
the same run."""
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import darray_b200 as dab  # noqa: E402
import sparse_oracle as so  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)


def timed(rt, fn, reps=20, rounds=5):
    for _ in range(3):
        fn()
    out = []
    for _ in range(rounds):
        e0, e1 = rt.event(), rt.event()
        rt.sync()
        rt.record(e0)
        for _ in range(reps):
            fn()
        rt.record(e1)
        out.append(rt.elapsed_ms(e0, e1) / reps)
        rt.event_destroy(e0)
        rt.event_destroy(e1)
    return float(np.median(out))


def torch_ms(fn, reps=20, rounds=5):
    import torch
    for _ in range(3):
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


def laplacian(k):
    """5-point Laplacian on a k x k grid, CSC (symmetric), rows ascending in each column."""
    N = k * k
    j = np.arange(N, dtype=np.int64)
    offs = [(-k, j >= k), (-1, j % k != 0), (0, np.ones(N, bool)), (1, j % k != k - 1), (k, j < N - k)]
    rows = np.stack([np.where(m, j + o, -1) for o, m in offs], axis=1)
    vals = np.stack([np.full(N, 4.0 if o == 0 else -1.0) for o, _ in offs], axis=1)
    keep = rows >= 0
    indptr = np.zeros(N + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(keep.sum(axis=1))
    return sp.csc_matrix((vals[keep], rows[keep].astype(np.int32), indptr), shape=(N, N))


def uniform_cols(n, per, rng):
    """n x n, exactly `per` entries in every column, one in each of `per` equal row bands (rows strictly ascending)."""
    band = n // per
    rows = (np.arange(per, dtype=np.int64) * band)[None, :] + rng.integers(0, band, (n, per))
    indptr = np.arange(n + 1, dtype=np.int64) * per
    return sp.csc_matrix((rng.standard_normal(n * per), rows.reshape(-1).astype(np.int32), indptr), shape=(n, n))


def power_law_rows(n, rng):
    """n x n with Pareto row lengths (1 .. 10^5 entries, mean about 10), columns evenly spread in each row; returned as CSC."""
    L = np.minimum(1 + (rng.pareto(1.2, n) * 4).astype(np.int64), min(100000, n))
    indptr = np.zeros(n + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(L)
    r = np.repeat(np.arange(n, dtype=np.int64), L)
    k = np.arange(indptr[-1], dtype=np.int64) - indptr[r]
    step = n // L[r]
    cols = rng.integers(0, step) + k * step
    return sp.csr_matrix((rng.standard_normal(indptr[-1]), cols.astype(np.int32), indptr), shape=(n, n)).tocsc()


def run(name, S, rt, rng):
    import torch
    m, n = S.shape
    t0 = time.perf_counter()
    DS = dab.distribute(S)
    ch = next(iter(DS.chunks.values()))
    print(f"{name}: {m} x {n}, nnz {ch.nnz}, distribute (host) {time.perf_counter() - t0:.1f} s", flush=True)
    isz = 8
    x = dab.B200Array.from_numpy(rt, rng.standard_normal(n))
    xt = dab.B200Array.from_numpy(rt, rng.standard_normal(m))
    y, yt = dab.B200Array.empty(rt, (m,), np.float64), dab.B200Array.empty(rt, (n,), np.float64)
    rt.sync()
    e0, e1 = rt.event(), rt.event()
    rt.record(e0)
    ch.csr()
    rt.record(e1)
    rt.sync()
    print(f"  K19 build (first call)   {rt.elapsed_ms(e0, e1):9.3f} ms", flush=True)
    for trans, out, xin, rows in ((False, y, x, m), (True, yt, xt, n)):
        ms = timed(rt, lambda: ch.matvec(trans, xin.ptr, out.ptr))
        nbytes = ch.nnz * (4 + isz) + 8 * (rows + 1) + isz * (m + n)
        # cuSPARSE through torch on the same CSR arrays (A'*x: the CSC arrays read as the CSR of A')
        ptr, idx, val = (ch.colptr, ch.rowval, ch.nzval) if trans else ch.csr()
        tA = torch.sparse_csr_tensor(torch.from_numpy(ptr.to_numpy()).cuda(), torch.from_numpy(idx.to_numpy().astype(np.int64)).cuda(),
                                     torch.from_numpy(val.to_numpy()).cuda(), size=(rows, n if not trans else m))
        tx = torch.from_numpy(xin.to_numpy()).cuda().reshape(-1, 1)
        tms = torch_ms(lambda: tA @ tx)
        # sampled rows against the ordered-fold model
        got = out.to_numpy()
        hp, hi, hv, hx = ptr.to_numpy(), idx.to_numpy(), val.to_numpy(), xin.to_numpy()
        sample = np.unique(np.concatenate([rng.integers(0, rows, 2000), [int(np.argmax(np.diff(hp)))]]))
        sub_len = np.diff(hp)[sample]
        sptr = np.zeros(sample.size + 1, dtype=np.int64)
        sptr[1:] = np.cumsum(sub_len)
        take = np.concatenate([np.arange(hp[r], hp[r + 1]) for r in sample])
        ok = so.same_bits(got[sample], so.fold_rows(sptr, hi[take], hv[take], hx))
        label = "A'*x" if trans else "A*x "
        print(f"  {label} K18 {ms:9.4f} ms {nbytes / ms / 1e6:8.1f} GB/s | cuSPARSE {tms:9.4f} ms {nbytes / tms / 1e6:8.1f} GB/s | "
              f"K18/cuSPARSE time {ms / tms:5.2f} | sampled rows bit-exact: {ok}", flush=True)
        del tA, tx
        torch.cuda.empty_cache()
    for b in (x, xt, y, yt):
        b.free()
    DS.close()


def main():
    rt = dab.init(workers_per_rank=1, use_dist=False)
    rng = np.random.default_rng(2026)
    run("laplacian 4096^2", laplacian(4096), rt, rng)
    run("uniform 32/col 2^22", uniform_cols(1 << 22, 32, rng), rt, rng)
    run("power-law rows 2^20", power_law_rows(1 << 20, rng), rt, rng)
    dab.d_closeall()


if __name__ == "__main__":
    main()
