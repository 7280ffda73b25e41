"""TEST INFRASTRUCTURE -- the indexed gather K22 (``dab_index_gather``) for the host-memory emulation of the C ABI (tests/hostmem_abi.py),
so that the host flow of ``d[I::DArray]`` can run on a CPU-only machine.

``install()`` adds the method to ``hostmem_abi.HostMemABI``; every emulation instance, the ones the ``hostmem`` fixture and the
``DAB_HOSTMEM=1`` session create included, then serves it.  The emulation follows the kernel's definition, not a whole-array NumPy
shortcut: each index is split into coordinates of the source dims, each coordinate's chunk is the largest grid position whose cut does
not exceed it (``tk_search``), the element is read from that chunk's pointer at the chunk-local column-major offset, and ``*bad_pos``
gets the smallest position of an index outside ``[1, prod(dims)]``, whose output element is left untouched.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm

MAX_DIMS, MAX_CHUNKS = 8, 1024


def dab_index_gather(self, ctx, elem_bytes, out, idx, idx_dtype, n, ndim, dims, grid, cuts, chunk_ptrs, bad_pos):
    es, n, nd, idx_dtype = int(elem_bytes), int(n), int(ndim), int(idx_dtype)
    if es not in (1, 4, 8, 16) or idx_dtype not in (hm.I32, hm.I64):
        return 2                                                                                                # DAB_ERR_ARG
    if not 1 <= nd <= MAX_DIMS:
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    if n == 0:
        return 0
    dims = [int(dims[k]) for k in range(nd)]
    grid = [int(grid[k]) for k in range(nd)]
    if int(np.prod(grid)) > MAX_CHUNKS:
        return 6
    cut, o = [], 0
    for k in range(nd):
        ck = np.array([int(cuts[o + c]) for c in range(grid[k] + 1)], dtype=np.int64)
        if ck[0] != 0 or ck[-1] != dims[k] or np.any(np.diff(ck) < 0):
            return 2
        cut.append(ck)
        o += grid[k] + 1
    ptrs = [hm._addr(chunk_ptrs[c]) if chunk_ptrs[c] else 0 for c in range(int(np.prod(grid)))]
    for c, p in enumerate(ptrs):
        g = np.unravel_index(c, grid, order="F")
        if not p and all(cut[k][g[k] + 1] > cut[k][g[k]] for k in range(nd)):
            return 2                                                                                            # a non-empty chunk needs a pointer
    g = hm._view(idx, n, np.int32 if idx_dtype == hm.I32 else np.int64).astype(np.int64) - 1
    length = int(np.prod(dims))
    okm = (g >= 0) & (g < length)
    if not okm.all():
        b = hm._view(bad_pos, 1, np.uint64)
        b[0] = min(int(b[0]), int(np.argmin(okm)))
    pos = np.nonzero(okm)[0]
    rem = g[pos]
    chunk = np.zeros(pos.size, dtype=np.int64)
    off = np.zeros(pos.size, dtype=np.int64)
    mult = np.ones(pos.size, dtype=np.int64)
    cstride = 1
    for k in range(nd):
        x = rem % dims[k] if k + 1 < nd else rem
        rem = rem // dims[k]
        c = np.searchsorted(cut[k][:grid[k]], x, side="right") - 1                 # largest c < grid with cut <= x
        off += (x - cut[k][c]) * mult
        mult *= cut[k][c + 1] - cut[k][c]
        chunk += c * cstride
        cstride *= grid[k]
    dt = hm._UNIT[es]
    ov = hm._view(out, n, dt)
    for c in np.unique(chunk):
        sel = chunk == c
        assert ptrs[c], "the cut search never selects an empty chunk"
        o_c = off[sel]
        src = hm._view(ptrs[c], int(o_c.max()) + 1, dt)
        ov[pos[sel]] = src[o_c]
    self.launches += 1
    return 0


def install():
    """Add the indexed gather to the emulation class (idempotent)."""
    hm.HostMemABI.dab_index_gather = dab_index_gather
