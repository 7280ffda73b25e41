"""TEST INFRASTRUCTURE -- K26 (``dab_sortperm_slices``) for the host-memory emulation of the C ABI (tests/hostmem_abi.py), so that the host
flow of ``sort(A; dims)`` / ``sortperm(A; dims)`` can run on a CPU-only machine.

``install()`` adds the method to ``hostmem_abi.HostMemABI``, together with K21 (tests/sortperm_hostmem.py), which the DVector forms use,
and K22 (tests/take_hostmem.py), which ``A[sortperm(A; dims)]`` uses.
``install_slices(fake)`` adds K13 (tests/mapslices_oracle.py) to one emulation instance, for ``sort(A; dims)`` without ``by``.  The
emulation follows the kernel's definition: per fibre, a STABLE argsort of ``sortby_radix_key`` (the order-preserving radix key with every
NaN collapsed to the top key), mapped to the 1-based global linear index of each element; the values are moved as bytes.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm
import sortperm_hostmem
import take_hostmem

SMEM_LEN = 4096                                                  # DAB_SORTPERM_SLICES_SMEM_LEN


def _arr(p, n, ctype):
    import ctypes as C
    return [int(x) for x in C.cast(p, C.POINTER(ctype * n)).contents]


def dab_sortperm_slices(self, ctx, key_dtype, keys, ndim, chunk_dims, chunk_lo, global_dims, dim, perm, val_bytes, vals, vals_out):
    import ctypes as C
    key_dtype, ndim, dim, val_bytes = int(key_dtype), int(ndim), int(dim), int(val_bytes)
    if not (chunk_dims and chunk_lo and global_dims):
        return 2                                                                                               # DAB_ERR_ARG
    if ndim > 8:
        return 6                                                                                               # DAB_ERR_UNSUPPORTED
    if not (ndim >= 1 and 1 <= dim <= ndim):
        return 2
    cd, lo, gd = (_arr(x, ndim, C.c_size_t) for x in (chunk_dims, chunk_lo, global_dims))
    if cd[dim - 1] != gd[dim - 1] or any(lo[k] + cd[k] > gd[k] for k in range(ndim)):
        return 2
    if key_dtype not in (hm.F32, hm.F64, hm.I32, hm.I64):
        return 6
    if (hm._addr(vals) == 0) != (hm._addr(vals_out) == 0) or (hm._addr(vals) and val_bytes not in (4, 8)):
        return 2
    n = int(np.prod(cd))
    if n == 0:
        return 0
    if not (hm._addr(keys) and hm._addr(perm)):
        return 2
    if cd[dim - 1] > SMEM_LEN and n >= 0xFFFFF000:
        return 6
    shape = tuple(cd)
    e = hm.by_radix_key(hm._view(keys, n, hm._utype(key_dtype)).copy(), key_dtype).reshape(shape, order="F")
    order = np.argsort(e, axis=dim - 1, kind="stable")              # per fibre: the positions s in rank order
    G = np.cumprod([1] + gd[:-1])
    gidx = np.ones(shape, dtype=np.int64)                           # 1-based global linear index of every chunk element
    for k in range(ndim):
        sh = [1] * ndim
        sh[k] = cd[k]
        gidx = gidx + ((lo[k] + np.arange(cd[k], dtype=np.int64)) * int(G[k])).reshape(sh)
    hm._view(perm, n, np.int64)[:] = np.take_along_axis(gidx, order, axis=dim - 1).reshape(-1, order="F")
    if hm._addr(vals):
        u = np.uint32 if val_bytes == 4 else np.uint64
        v = hm._view(vals, n, u).copy().reshape(shape, order="F")
        hm._view(vals_out, n, u)[:] = np.take_along_axis(v, order, axis=dim - 1).reshape(-1, order="F")
    self.launches += 1
    return 0


def install():
    """Add K26 (and K21, and K22 for ``A[sortperm(A; dims)]``) to the emulation class (idempotent)."""
    sortperm_hostmem.install()
    take_hostmem.install()
    hm.HostMemABI.dab_sortperm_slices = dab_sortperm_slices


def install_slices(fake):
    """K13 on one emulation instance: ``sort(A; dims)`` without ``by`` is ``mapslices(sort, A, dims)``."""
    import mapslices_oracle
    return mapslices_oracle.install_hostmem(fake)
