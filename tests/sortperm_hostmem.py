"""TEST INFRASTRUCTURE -- the pair sort K21 (``dab_sort_pairs`` and its scratch query) for the host-memory emulation of the C ABI
(tests/hostmem_abi.py), so that the host flow of ``sortperm`` can run on a CPU-only machine.

``install()`` adds the two methods to ``hostmem_abi.HostMemABI``; every emulation instance, the ones the ``hostmem`` fixture and the
``DAB_HOSTMEM=1`` session create included, then serves them.  The emulation follows the kernel's definition, not a NumPy shortcut on the
floats: a STABLE argsort of ``sortby_radix_key`` (the order-preserving radix key with every NaN collapsed to the top key), the sorted keys
decoded from those radix keys (so every NaN comes out as the one canonical NaN), and ``vals[perm]`` or ``base + perm``.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm


def _stride(nbytes: int) -> int:
    return (nbytes + 255) & ~255


def dab_sort_pairs_scratch_bytes(self, key_dtype, n, out):
    key_dtype = int(key_dtype)
    if key_dtype not in (hm.F32, hm.F64, hm.I32, hm.I64):
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    kb = 8 if key_dtype in (hm.F64, hm.I64) else 4
    out._obj.value = _stride(int(n) * kb) + 2 * _stride(int(n) * 4)
    return 0


def dab_sort_pairs(self, ctx, key_dtype, keys, keys_out, vals, base, vals_out, scratch, scratch_bytes, n):
    import ctypes as C
    n, key_dtype = int(n), int(key_dtype)
    if n == 0:
        return 0
    if n >= 0xFFFFF000:
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    need = C.c_size_t()
    st = self.dab_sort_pairs_scratch_bytes(key_dtype, n, C.byref(need))
    if st:
        return st
    assert int(scratch_bytes) >= need.value and hm._addr(scratch) % 16 == 0 and hm._addr(vals) != hm._addr(vals_out)
    u = hm._utype(key_dtype)
    e = hm.by_radix_key(hm._view(keys, n, u).copy(), key_dtype)
    perm = np.argsort(e, kind="stable")
    v = hm._view(vals, n, np.int64).copy() if hm._addr(vals) else np.int64(int(base)) + np.arange(n, dtype=np.int64)
    hm._view(keys_out, n, u)[:] = hm.radix_dec(e[perm], key_dtype)
    hm._view(vals_out, n, np.int64)[:] = v[perm]
    self.launches += 1
    return 0


def install():
    """Add the pair-sort entry points to the emulation class (idempotent)."""
    hm.HostMemABI.dab_sort_pairs = dab_sort_pairs
    hm.HostMemABI.dab_sort_pairs_scratch_bytes = dab_sort_pairs_scratch_bytes
