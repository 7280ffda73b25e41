"""TEST INFRASTRUCTURE -- the scatter K24 (``dab_scatter_check`` / ``dab_scatter_winners`` / ``dab_scatter``) and the masked expansion K25
(``dab_expand``) for the host-memory emulation of the C ABI (tests/hostmem_abi.py), so that the host flow of ``d[key] = v`` can run on a
CPU-only machine.

``install()`` adds the methods to ``hostmem_abi.HostMemABI``, together with K22 (tests/take_hostmem.py) and K23 with the K17 scans
(tests/compact_hostmem.py), which the flow shares.  The emulation follows the kernels' definitions: each index is located in the
destination table as K22 locates it (coordinates, the largest cut not above each, the chunk-local column-major offset); the check pass
records the first bad position and sets one bit per destination in the chunk's bitmap, flagging a bit that was set already; the winner
pass keeps the largest 1-based global position (run table) per destination; the store pass writes every valid index, or only the
winners.  ``dab_expand`` ranks each tile's true elements, reads position ``run_info[2r] + tile_incl[b] - count(b) + rank`` through
the value table (positions at or past its length are not read) and stores into the chunk; its scalar mode stores the scalar.
"""
from __future__ import annotations

import numpy as np

import compact_hostmem
import hostmem_abi as hm
import take_hostmem

MAX_DIMS, MAX_CHUNKS, TILE = 8, 1024, 4096


def _table(ndim, dims, grid, cuts, ptrs):
    """(dims, grid, per-dim cuts, chunk pointers) or a status code, with K22's checks."""
    nd = int(ndim)
    if not 1 <= nd <= MAX_DIMS:
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    dims = [int(dims[k]) for k in range(nd)]
    grid = [int(grid[k]) for k in range(nd)]
    if int(np.prod(grid)) > MAX_CHUNKS:
        return 6
    cut, o = [], 0
    for k in range(nd):
        ck = np.array([int(cuts[o + c]) for c in range(grid[k] + 1)], dtype=np.int64)
        if ck[0] != 0 or ck[-1] != dims[k] or np.any(np.diff(ck) < 0):
            return 2                                                                                            # DAB_ERR_ARG
        cut.append(ck)
        o += grid[k] + 1
    p = [hm._addr(ptrs[c]) if ptrs[c] else 0 for c in range(int(np.prod(grid)))]
    for c, a in enumerate(p):
        g = np.unravel_index(c, grid, order="F")
        if not a and all(cut[k][g[k] + 1] > cut[k][g[k]] for k in range(nd)):
            return 2                                                                                            # a non-empty chunk needs a pointer
    return dims, grid, cut, p


def _locate(tab, g):
    """(chunk, chunk-local offset) of the 0-based linear indices g (all in range)."""
    dims, grid, cut, _ = tab
    nd = len(dims)
    rem = g.copy()
    chunk = np.zeros(g.size, dtype=np.int64)
    off = np.zeros(g.size, dtype=np.int64)
    mult = np.ones(g.size, dtype=np.int64)
    cstride = 1
    for k in range(nd):
        x = rem % dims[k] if k + 1 < nd else rem
        rem = rem // dims[k]
        c = np.searchsorted(cut[k][:grid[k]], x, side="right") - 1
        off += (x - cut[k][c]) * mult
        mult *= cut[k][c + 1] - cut[k][c]
        chunk += c * cstride
        cstride *= grid[k]
    return chunk, off


def _indices(idx, idx_dtype, n):
    return hm._view(idx, n, np.int32 if int(idx_dtype) == hm.I32 else np.int64).astype(np.int64) - 1


def _positions(n, run_len, run_lin):
    k = np.arange(n, dtype=np.int64)
    lin = hm._view(run_lin, -(-n // run_len), np.int64)
    return lin[k // run_len] + k % run_len


def dab_scatter_check(self, ctx, idx, idx_dtype, n, ndim, dims, grid, cuts, bitmap_ptrs, status):
    tab = _table(ndim, dims, grid, cuts, bitmap_ptrs)
    if isinstance(tab, int):
        return tab
    n = int(n)
    if n == 0:
        return 0
    if int(idx_dtype) not in (hm.I32, hm.I64) or not hm._addr(idx) or not hm._addr(status):
        return 2
    g = _indices(idx, idx_dtype, n)
    length = int(np.prod(tab[0]))
    ok = (g >= 0) & (g < length)
    st = hm._view(status, 2, np.uint64)
    if not ok.all():
        st[0] = min(int(st[0]), int(np.argmin(ok)))
    chunk, off = _locate(tab, g[ok])
    for c, o in zip(chunk, off):                                    # one atomicOr each, in any order: the flag does not depend on it
        words = hm._view(tab[3][c], int(o >> 5) + 1, np.uint32)
        bit = np.uint32(1 << int(o & 31))
        if words[o >> 5] & bit:
            st[1] = 1
        words[o >> 5] |= bit
    self.launches += 1
    return 0


def dab_scatter_winners(self, ctx, idx, idx_dtype, n, run_len, run_lin, win_bytes, ndim, dims, grid, cuts, win_ptrs):
    if int(win_bytes) not in (4, 8):
        return 2
    tab = _table(ndim, dims, grid, cuts, win_ptrs)
    if isinstance(tab, int):
        return tab
    n = int(n)
    if n == 0:
        return 0
    if int(idx_dtype) not in (hm.I32, hm.I64) or not hm._addr(idx) or int(run_len) < 1 or not hm._addr(run_lin):
        return 2
    g = _indices(idx, idx_dtype, n)
    ok = (g >= 0) & (g < int(np.prod(tab[0])))
    p = _positions(n, int(run_len), run_lin)[ok] + 1
    chunk, off = _locate(tab, g[ok])
    wt = np.uint32 if int(win_bytes) == 4 else np.uint64
    for c in np.unique(chunk):
        sel = chunk == c
        w = hm._view(tab[3][c], int(off[sel].max()) + 1, wt)
        np.maximum.at(w, off[sel], p[sel].astype(wt))
    self.launches += 1
    return 0


def dab_scatter(self, ctx, elem_bytes, idx, idx_dtype, n, src, scalar, run_len, run_lin, win_bytes, ndim, dims, grid, cuts, chunk_ptrs, win_ptrs):
    es, wb = int(elem_bytes), int(win_bytes)
    if es not in (1, 4, 8, 16) or wb not in (0, 4, 8):
        return 2
    tab = _table(ndim, dims, grid, cuts, chunk_ptrs)
    if isinstance(tab, int):
        return tab
    wtab = _table(ndim, dims, grid, cuts, win_ptrs) if wb else None
    if isinstance(wtab, int):
        return wtab
    n = int(n)
    if n == 0:
        return 0
    if int(idx_dtype) not in (hm.I32, hm.I64) or not hm._addr(idx) or not (hm._addr(src) or hm._addr(scalar)):
        return 2
    if wb and (int(run_len) < 1 or not hm._addr(run_lin)):
        return 2
    dt = hm._UNIT[es]
    g = _indices(idx, idx_dtype, n)
    ok = (g >= 0) & (g < int(np.prod(tab[0])))
    vals = hm._view(src, n, dt) if hm._addr(src) else np.repeat(hm._view(scalar, 1, dt), n)
    chunk, off = _locate(tab, g[ok])
    vals = vals[ok]
    if wb:
        p = _positions(n, int(run_len), run_lin)[ok] + 1
        wt = np.uint32 if wb == 4 else np.uint64
        win = np.array([hm._view(wtab[3][c], int(o) + 1, wt)[o] for c, o in zip(chunk, off)], dtype=np.uint64)
        keep = win == p.astype(np.uint64)
        chunk, off, vals = chunk[keep], off[keep], vals[keep]
    elif chunk.size:
        assert np.unique(np.stack([chunk, off]), axis=1).shape[1] == chunk.size, "the unique-index store pass met a duplicate"
    for c in np.unique(chunk):
        sel = chunk == c
        hm._view(tab[3][c], int(off[sel].max()) + 1, dt)[off[sel]] = vals[sel]
    self.launches += 1
    return 0


def dab_expand(self, ctx, elem_bytes, mask, dst, run_len, runs, tile_incl, run_info, nchunks, cuts, chunk_ptrs, scalar):
    es, run_len, runs, nchunks = int(elem_bytes), int(run_len), int(runs), int(nchunks)
    if es not in (1, 4, 8, 16):
        return 2
    dt = hm._UNIT[es]
    sc = hm._addr(scalar)
    if not sc:
        if not 1 <= nchunks <= MAX_CHUNKS:
            return 6
        cut = np.array([int(cuts[c]) for c in range(nchunks + 1)], dtype=np.int64)
        if cut[0] != 0 or np.any(np.diff(cut) < 0):
            return 2
        ptrs = [hm._addr(chunk_ptrs[c]) if chunk_ptrs[c] else 0 for c in range(nchunks)]
        if any(not p and cut[c + 1] > cut[c] for c, p in enumerate(ptrs)):
            return 2
    if run_len == 0 or runs == 0:
        return 0
    if not hm._addr(mask) or not hm._addr(dst) or not (sc or (hm._addr(tile_incl) and hm._addr(run_info))):
        return 2
    tpr = -(-run_len // TILE)
    m = hm._view(mask, run_len * runs, np.uint8)
    out = hm._view(dst, run_len * runs, dt)
    if sc:
        out[m != 0] = hm._view(scalar, 1, dt)[0]
        self.launches += 1
        return 0
    incl = hm._view(tile_incl, tpr * runs, np.int64)
    info = hm._view(run_info, 2 * runs, np.int64)
    for b in range(tpr * runs):
        r, t = divmod(b, tpr)
        lo = r * run_len + t * TILE
        p = np.nonzero(m[lo:lo + min(TILE, run_len - t * TILE)])[0]
        if p.size == 0:
            continue
        q = info[2 * r] + incl[b] - p.size + np.arange(p.size, dtype=np.int64)
        keep = q < cut[-1]
        q, p = q[keep], p[keep]
        c = np.searchsorted(cut[:nchunks], q, side="right") - 1
        for cc in np.unique(c):
            sel = c == cc
            o = q[sel] - cut[cc]
            out[lo + p[sel]] = hm._view(ptrs[cc], int(o.max()) + 1, dt)[o]
    self.launches += 1
    return 0


def install():
    """Add K24, K25 and the kernels their flow shares (K22, K23, K17 scans) to the emulation class (idempotent)."""
    take_hostmem.install()
    compact_hostmem.install()
    hm.HostMemABI.dab_scatter_check = dab_scatter_check
    hm.HostMemABI.dab_scatter_winners = dab_scatter_winners
    hm.HostMemABI.dab_scatter = dab_scatter
    hm.HostMemABI.dab_expand = dab_expand
