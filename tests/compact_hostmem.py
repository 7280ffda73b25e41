"""TEST INFRASTRUCTURE -- the stream compaction K23 (``dab_compact_count`` / ``dab_compact``) for the host-memory emulation of the C ABI
(tests/hostmem_abi.py), so that the host flow of ``d[mask]``, ``findall`` and ``filter`` can run on a CPU-only machine.

``install()`` adds the methods to ``hostmem_abi.HostMemABI``, together with the scans of K17 (tests/scan_oracle.py) that the flow uses
for its tile tables.  The emulation follows the kernels' definition, not a whole-array NumPy shortcut: the chunk is a table of
``runs`` runs of ``run_len`` elements, each cut into tiles of ``DAB_COMPACT_TILE``; ``dab_compact_count`` counts the nonzero mask
bytes of each tile; ``dab_compact`` ranks the true elements inside each tile, starts the tile's output segment at
``run_info[2r] + tile_incl[b] - count(b)``, and stores each element through the destination table (the largest chunk whose cut does not
exceed the position, at the chunk-local offset).  Positions at or past the output length are not written.
"""
from __future__ import annotations

import numpy as np

import hostmem_abi as hm
import scan_oracle

TILE, INDEX, MAX_CHUNKS = 4096, 0, 1024


def _tiles(run_len, runs):
    tpr = -(-run_len // TILE)
    return tpr, tpr * runs


def dab_compact_count(self, ctx, mask, run_len, runs, counts):
    run_len, runs = int(run_len), int(runs)
    if run_len == 0 or runs == 0:
        return 0
    if not hm._addr(mask) or not hm._addr(counts):
        return 2                                                                                                # DAB_ERR_ARG
    tpr, tiles = _tiles(run_len, runs)
    m = hm._view(mask, run_len * runs, np.uint8)
    cv = hm._view(counts, tiles, np.int32)
    for b in range(tiles):
        r, t = divmod(b, tpr)
        lo = r * run_len + t * TILE
        cv[b] = np.count_nonzero(m[lo:lo + min(TILE, run_len - t * TILE)])
    self.launches += 1
    return 0


def dab_compact(self, ctx, elem_bytes, mask, src, run_len, runs, tile_incl, run_info, nchunks, cuts, chunk_ptrs):
    es, run_len, runs, nchunks = int(elem_bytes), int(run_len), int(runs), int(nchunks)
    if es not in (INDEX, 1, 4, 8, 16):
        return 2
    if not 1 <= nchunks <= MAX_CHUNKS:
        return 6                                                                                                # DAB_ERR_UNSUPPORTED
    cut = np.array([int(cuts[c]) for c in range(nchunks + 1)], dtype=np.int64)
    if cut[0] != 0 or np.any(np.diff(cut) < 0):
        return 2
    ptrs = [hm._addr(chunk_ptrs[c]) if chunk_ptrs[c] else 0 for c in range(nchunks)]
    if any(not p and cut[c + 1] > cut[c] for c, p in enumerate(ptrs)):
        return 2                                                                                                # a non-empty chunk needs a pointer
    if run_len == 0 or runs == 0:
        return 0
    tpr, tiles = _tiles(run_len, runs)
    dt = np.int64 if es == INDEX else hm._UNIT[es]
    m = hm._view(mask, run_len * runs, np.uint8)
    sv = None if es == INDEX else hm._view(src, run_len * runs, dt)
    incl = hm._view(tile_incl, tiles, np.int64)
    info = hm._view(run_info, 2 * runs, np.int64)
    for b in range(tiles):
        r, t = divmod(b, tpr)
        lo = r * run_len + t * TILE
        p = np.nonzero(m[lo:lo + min(TILE, run_len - t * TILE)])[0]                  # the tile's true positions in rank order
        if p.size == 0:
            continue
        q = info[2 * r] + incl[b] - p.size + np.arange(p.size, dtype=np.int64)
        vals = info[2 * r + 1] + t * TILE + p + 1 if es == INDEX else sv[lo + p]
        keep = q < cut[-1]
        q, vals = q[keep], vals[keep]
        c = np.searchsorted(cut[:nchunks], q, side="right") - 1                      # largest c with cut <= q
        for cc in np.unique(c):
            sel = c == cc
            off = q[sel] - cut[cc]
            hm._view(ptrs[cc], int(off.max()) + 1, dt)[off] = vals[sel]
    self.launches += 1
    return 0


def install():
    """Add K23 and the K17 scans to the emulation class (idempotent)."""
    hm.HostMemABI.dab_compact_count = dab_compact_count
    hm.HostMemABI.dab_compact = dab_compact
    for name in ("dab_scan", "dab_scan_totals", "dab_scan_carrier_dtype"):
        if not hasattr(hm.HostMemABI, name):
            setattr(hm.HostMemABI, name, _scan_entry(name))


def _scan_entry(name):
    def call(self, *args):
        scan_oracle.install_hostmem(self)                     # instance attributes from now on
        return getattr(self, name)(*args)
    return call
