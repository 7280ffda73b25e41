"""TEST INFRASTRUCTURE -- the tiled dimension permutation K28 (``dab_permute_box``) for the host-memory emulation of the C ABI
(tests/hostmem_abi.py), so that the host flow of ``permutedims`` / ``permutedims!`` can run on a CPU-only machine.

``install()`` adds the method to ``hostmem_abi.HostMemABI``; every emulation instance, the ones the ``hostmem`` fixture and the
``DAB_HOSTMEM=1`` session create included, then serves it.  The emulation follows the kernel's definition, not a whole-array NumPy
shortcut: it refuses what the kernel refuses (``DAB_ERR_ARG``: a null pointer, ndim outside 2..8, an element size other than 1, 2, 4, 8
or 16, destination stride of dimension 0 other than 1, not exactly one other dimension with source stride 1), launches nothing for a
zero extent, and otherwise computes, for every coordinate t of the box, the element offsets ``sum(t_k * stride[k])`` on both sides from
the given strides and extents and copies the element's bytes.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm

ERR_ARG = 2


def dab_permute_box(self, ctx, elem_bytes, ndim, dst, dst_strides, src, src_strides, extent):
    nd, es = int(ndim), int(elem_bytes)
    if not hm._addr(dst) or not hm._addr(src) or dst_strides is None or src_strides is None or extent is None:
        return ERR_ARG
    if not 2 <= nd <= 8 or es not in hm._UNIT:
        return ERR_ARG
    ds = [int(dst_strides[k]) for k in range(nd)]
    ss = [int(src_strides[k]) for k in range(nd)]
    ext = [int(extent[k]) for k in range(nd)]
    if ds[0] != 1 or sum(1 for s in ss[1:] if s == 1) != 1:
        return ERR_ARG
    if min(ext) == 0:
        return 0

    def offsets(strides):
        tot = np.zeros((), dtype=np.int64)
        for k in range(nd):
            tot = tot[..., None] + np.arange(ext[k], dtype=np.int64) * strides[k]
        return tot.reshape(-1)

    do, so = offsets(ds), offsets(ss)
    dt = hm._UNIT[es]
    lo_d, lo_s = int(do.min()), int(so.min())
    dv = hm._view(hm._addr(dst) + lo_d * es, int(do.max()) - lo_d + 1, dt)
    sv = hm._view(hm._addr(src) + lo_s * es, int(so.max()) - lo_s + 1, dt)
    dv[do - lo_d] = sv[so - lo_s]
    self.launches += 1
    return 0


def install():
    """Add the permutation to the emulation class (idempotent)."""
    hm.HostMemABI.dab_permute_box = dab_permute_box
