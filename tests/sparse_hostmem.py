"""TEST INFRASTRUCTURE -- the sparse entry points (K18 ``dab_spmv``, K19 ``dab_csc_to_csr``) for the host-memory emulation of the C ABI
(tests/hostmem_abi.py), so that the host runtime around sparse DArrays can run on a CPU-only machine.

``install()`` adds the two methods to ``hostmem_abi.HostMemABI``; every emulation instance, the ones the ``hostmem`` fixture and the
``DAB_HOSTMEM=1`` session create included, then serves them.  The test modules that drive sparse DArrays against the emulation call it at
import.  Where the algorithm is the thing under test the emulation follows the kernels:

* ``dab_spmv`` is the ordered fold of tests/sparse_oracle.py (from zero, in storage order, every operation rounded in T);
* ``dab_csc_to_csr`` is the composition of dab_sparse.cu step by step: pack ``row << 32 | k``, sort the words with the emulated K11
  (``dab_sort``), unpack the column by a search of ``colptr`` and the value by position, and ``rowptr[r]`` = the count of words below
  ``r << 32``.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm
import sparse_oracle as so


def dab_spmv(self, ctx, dtype, nrows, nnz, ptr, idx, val, x, out):
    nrows, nnz, dt = int(nrows), int(nnz), hm._NP[int(dtype)]
    if nrows == 0:
        return 0
    p = hm._view(ptr, nrows + 1, np.int64).copy()
    assert int(p[-1] - p[0]) == nnz
    iv = hm._view(hm._addr(idx), int(p[-1]), np.int32).copy()
    nx = int(iv[p[0]:].max()) + 1 if nnz else 0
    hm._view(out, nrows, dt)[:] = so.fold_rows(p, iv, hm._view(hm._addr(val), int(p[-1]), dt).copy(), hm._view(x, nx, dt).copy())
    self.launches += 1
    return 0


def dab_csc_to_csr(self, ctx, dtype, m, n, nnz, colptr, rowval, nzval, rowptr, colidx, val):
    m, n, nnz, dt = int(m), int(n), int(nnz), hm._NP[int(dtype)]
    if m > 0x7FFFFFFF or n > 0x7FFFFFFF or nnz >= 0xFFFFF000:
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    words = np.empty(nnz, dtype=np.int64)
    if nnz:
        words[:] = (hm._view(rowval, nnz, np.int32).astype(np.int64) << 32) | np.arange(nnz, dtype=np.int64)   # csr_pack_kernel
        tmp = np.empty(nnz, dtype=np.int64)
        self.dab_sort(ctx, hm.I64, words.ctypes.data, words.ctypes.data, tmp.ctypes.data, nnz)
        k = words & 0xFFFFFFFF
        cp = hm._view(colptr, n + 1, np.int64)
        hm._view(colidx, nnz, np.int32)[:] = np.searchsorted(cp[:n], k, side="right") - 1                      # csr_unpack_kernel
        hm._view(val, nnz, dt)[:] = hm._view(nzval, nnz, dt)[k]
        self.launches += 2
    hm._view(rowptr, m + 1, np.int64)[:] = np.searchsorted(words, np.arange(m + 1, dtype=np.int64) << 32, side="left")  # csr_rowptr_kernel
    self.launches += 1
    return 0


def install():
    """Add the sparse entry points to the emulation class (idempotent)."""
    hm.HostMemABI.dab_spmv = dab_spmv
    hm.HostMemABI.dab_csc_to_csr = dab_csc_to_csr
