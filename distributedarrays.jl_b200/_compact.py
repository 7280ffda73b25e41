"""``d[mask]``, ``findall`` and ``filter`` (row f13): stream compaction by K23 (``dab_compact_count`` / ``dab_compact``).

The reference defines none of these; Base's generic methods iterate the array element by element.  The result's length depends on
the data, so it is planned in three steps, none of which makes a CTA or a GPU wait on another:

1. per local chunk, ``dab_compact_count`` counts the true mask bytes of every tile, and K17 scans the tile table along each run
   (``dab_scan``) and sums each run (``dab_scan_totals``);
2. the run totals of all chunks travel in one ``allgather_small``; every rank lays out the global output offsets of all runs with
   NumPy (host cost O(total runs)), allocates the result and uploads the offsets of its own runs;
3. per local chunk, ``dab_compact`` writes the selected elements (or their 1-based linear indices) into the result's chunks, local
   or CUDA-IPC peer mappings, through K22's destination table.

A RUN is a stretch of a chunk that is contiguous in the global column-major order (DESIGN.md §3.10): with ``k`` the first dimension
whose grid is split (the last one when nothing is split), it holds all of dims ``1..k-1`` and the chunk's range along dim ``k`` at
one set of coordinates along dims ``k+1..``.  Runs are ordered by the outer coordinates, then by the block along dim ``k``.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional

import numpy as np

from . import _lib
from ._darray import B200Array, DArray, SubDArray, procs, similar
from ._take import _source_table
from .layout import shape_of
from .runtime import close_remote_reads, open_remote_reads

MAX_DIMS = 8
MAX_CHUNKS = 1024          # dab_compact's destination table: the result's chunks travel in the kernel's parameter block
_SERVED = {np.dtype(t) for t in (np.bool_, np.int32, np.float32, np.int64, np.float64, np.complex64, np.complex128)}
_JL = {np.dtype(np.float16): "Float16", np.dtype(np.bool_): "Bool", np.dtype(np.int32): "Int32", np.dtype(np.int64): "Int64", np.dtype(np.float32): "Float32",
       np.dtype(np.float64): "Float64", np.dtype(np.complex64): "ComplexF32", np.dtype(np.complex128): "ComplexF64"}


def _non_boolean(name: str) -> TypeError:
    return TypeError(f"TypeError: non-boolean ({name}) used in boolean context")


def run_plan(lay):
    """The runs of every chunk of ``lay``: a list, per chunk in layout order, of ``(run_len, run ids, 0-based global linear index of
    each run's first element)``, and the total number of runs (the global run id space)."""
    dims, grid = lay.dims, lay.grid
    N = len(dims)
    k = next((j for j, g in enumerate(grid) if g > 1), N - 1)
    inner = int(np.prod(dims[:k], dtype=np.int64))
    outer_dims = dims[k + 1:]
    out = []
    for c, Kc in enumerate(lay.indices):
        ext = shape_of(Kc)
        run_len = inner * ext[k]
        if outer_dims:                                         # the global outer coordinates of each run, column-major over the chunk
            loc = np.indices(ext[k + 1:], dtype=np.int64).reshape(len(outer_dims), -1, order="F")
            glob = loc + np.array([r[0] - 1 for r in Kc[k + 1:]], dtype=np.int64).reshape(-1, 1)
            o = np.ravel_multi_index(glob, outer_dims, order="F").astype(np.int64)
        else:
            o = np.zeros(1, dtype=np.int64)
        b = c % grid[k]                                        # grid[:k] are all 1
        out.append((run_len, b + grid[k] * o, inner * (Kc[k][0] - 1) + inner * dims[k] * o))
    return out, grid[k] * int(np.prod(outer_dims, dtype=np.int64))


def _check(d, m):
    """Every refusal of ``d[m]``, before anything is allocated or launched."""
    if d.dtype not in _SERVED:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"logical indexing of a DArray of {d.dtype} (served: {sorted(map(str, _SERVED))})")
    if not 1 <= d.ndim <= MAX_DIMS:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"logical indexing of a DArray of {d.ndim} dimensions (served: 1..{MAX_DIMS})")
    if len(procs(d)) > MAX_CHUNKS:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"a result over {len(procs(d))} workers (served: up to {MAX_CHUNKS})")


def plan(d: DArray, m: DArray, temps: list):
    """Phases 1 and 2 of ``d[m]`` (and of ``d[m] = v``) for a non-empty ``d`` and a Bool DArray ``m`` of its dims: per local non-empty
    chunk the mask block in ``d``'s chunk shape and the scans of its tile counts, then the global output offset of every run.  Returns
    ``(runs, work, plans, offsets)``: ``run_plan(d.layout)``'s runs, the ``(chunk, pid)`` pairs served here, ``plans[chunk] = (mask
    block, inclusive tile scan, run totals)``, and the ``nruns + 1`` offsets whose last entry is ``count(m)``.  Every device block it
    allocates goes to ``temps``, which the caller frees.  Collective."""
    rt = d.rt
    lay = d.layout
    runs, nruns = run_plan(lay)
    mine = [(c, pid) for c, pid in enumerate(lay.pids) if pid in d.chunks]
    work = [(c, pid) for c, pid in mine if d.chunks[pid].size]
    same = m.layout.same_as(lay)
    plans = {}
    fenced = open_remote_reads(rt, [] if same else [m], "device")
    for c, pid in work:
        run_len, ids, _ = runs[c]
        if same:
            blk = m.chunks[pid]
        else:                                              # the mask block in d's chunk shape: a halo read of 1-byte elements
            blk = B200Array.empty(rt, d.chunks[pid].shape, np.bool_, temp=True)
            temps.append(blk)
            SubDArray(m, lay.indices[c], tuple(False for _ in lay.indices[c])).copy_to(blk)
        tiles = -(-run_len // _lib.COMPACT_TILE) * ids.size
        counts = B200Array.empty(rt, (tiles,), np.int32, temp=True)
        incl = B200Array.empty(rt, (tiles,), np.int64, temp=True)
        tot = B200Array.empty(rt, (ids.size,), np.int64, temp=True)
        temps += [counts, incl, tot]
        _lib.call("dab_compact_count", rt.ctx, C.c_void_p(blk.ptr), run_len, ids.size, C.c_void_p(counts.ptr))
        tpr = tiles // ids.size
        _lib.call("dab_scan", rt.ctx, _lib.I32, _lib.SUM, _lib.I64, C.c_void_p(counts.ptr), 1, tpr, ids.size, None, C.c_void_p(incl.ptr))
        _lib.call("dab_scan_totals", rt.ctx, _lib.I32, _lib.SUM, _lib.I64, C.c_void_p(counts.ptr), 1, tpr, ids.size, C.c_void_p(tot.ptr))
        plans[c] = (blk, incl, tot)
    close_remote_reads(rt, fenced, "device")

    # every rank sends the run totals of its chunks in layout order, padded to the longest payload of any rank
    per_rank = [0] * rt.world
    for c, pid in enumerate(lay.pids):
        per_rank[rt.rank_of(pid)] += runs[c][1].size
    payload = np.zeros(max(max(per_rank), 1), dtype=np.int64)
    o = 0
    for c, _ in mine:
        n = runs[c][1].size
        if c in plans:
            payload[o:o + n] = plans[c][2].to_numpy()
        o += n
    totals = np.zeros(nruns, dtype=np.int64)
    cursor = [0] * rt.world
    gathered = rt.allgather_small(payload)
    for c, pid in enumerate(lay.pids):
        r, n = rt.rank_of(pid), runs[c][1].size
        totals[runs[c][1]] = gathered[r][cursor[r]:cursor[r] + n]
        cursor[r] += n
    offsets = np.concatenate([[0], np.cumsum(totals)]).astype(np.int64)
    return runs, work, plans, offsets


def _compact(d: DArray, m: DArray, index: bool) -> DArray:
    """The selected elements of ``d`` (``index``: their 1-based linear indices, Int64) where the Bool DArray ``m`` of ``d``'s dims is
    true, in column-major order, as a DVector with the layout of ``similar(d, T, (count,))``.  Collective."""
    rt = d.rt
    dt = np.dtype(np.int64) if index else d.dtype
    if d.size == 0:
        return similar(d, dt, (0,))
    temps, R = [], None
    try:
        runs, work, plans, offsets = plan(d, m, temps)
        count = int(offsets[-1])

        R = similar(d, dt, (count,))
        if count:
            fenced = open_remote_reads(rt, [R], "device")
            _, grid, cuts, ptrs = _source_table(R)
            es = _lib.COMPACT_INDEX if index else d.dtype.itemsize
            for c, pid in work:
                run_len, ids, lin = runs[c]
                blk, incl, _ = plans[c]
                info = B200Array.empty(rt, (2 * ids.size,), np.int64, temp=True)
                temps.append(info)
                info.copy_from_host(np.stack([offsets[ids], lin]).reshape(-1, order="F"))
                _lib.call("dab_compact", rt.ctx, es, C.c_void_p(blk.ptr), None if index else C.c_void_p(d.chunks[pid].ptr), run_len, ids.size,
                          C.c_void_p(incl.ptr), C.c_void_p(info.ptr), grid[0], cuts, ptrs)
            close_remote_reads(rt, fenced, "device")              # the peer stores into R have landed before its owners read it
    except BaseException:
        if R is not None:
            R.close()                                             # an unexpected failure still leaves nothing allocated
        raise
    finally:
        for t in temps:
            t.free()                                              # stream-ordered
    return R


def getindex_mask(d: DArray, m: DArray) -> DArray:
    """``d[m]`` for a Bool DArray ``m`` of ``d``'s dims (any layout): the elements of ``d`` where ``m`` is true, in column-major
    order, as a DVector of ``d``'s element type with the layout of ``similar(d, (count(m),))``.  Bit-exact copies.  Collective."""
    _check(d, m)
    return _compact(d, m, index=False)


def findall(f, d: Optional[DArray] = None) -> DArray:
    """``findall(mask)`` / ``findall(f, d)``: the 1-based column-major LINEAR indices where ``mask`` (``f.(d)``) is true, as a
    ``DArray{Int64}`` DVector with the layout of ``similar(mask, Int64, (count,))``.  Unlike Julia the result stays on the devices
    (not a host ``Vector``) and an N-d mask gives linear indices, not ``CartesianIndex`` -- the convention of ``findmax(d; dims)``.
    ``f`` is a traced predicate (what ``broadcast`` accepts); a non-Bool result raises Julia's ``TypeError``.  Collective."""
    if d is None:
        m = _operand(f, "findall")
        if m.dtype != np.dtype(np.bool_):
            raise _non_boolean(_JL.get(m.dtype, str(m.dtype)))
        _check(m, m)
        return _compact(m, m, index=True)
    d = _operand(d, "findall")
    _check(d, d)
    if d.rt.nworkers > MAX_CHUNKS:                             # f.(d) gets the default layout over every worker
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"a result over {d.rt.nworkers} workers (served: up to {MAX_CHUNKS})")
    m = _predicate(f, d)
    try:
        _check(m, m)
        return _compact(m, m, index=True)
    finally:
        m.close()


def filter(f: Callable, d: DArray) -> DArray:  # noqa: A001 - mirrors Base.filter
    """``filter(f, d)``: the elements of ``d`` for which the traced predicate ``f`` is true, in column-major order, as a DVector for
    any N (as Julia's ``filter`` on an ``Array``), with the layout of ``similar(d, (count,))``.  Collective."""
    d = _operand(d, "filter")
    _check(d, d)
    m = _predicate(f, d)
    try:
        return _compact(d, m, index=False)
    finally:
        m.close()


def _operand(d, what: str) -> DArray:
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray):
        refuse(what)
    if not isinstance(d, DArray):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} of a {type(d).__name__} is not served (a dense DArray is)")
    return d


def _predicate(f: Callable, d: DArray) -> DArray:
    """``f.(d)``, once the traced result type is known to be Bool (nothing is launched otherwise)."""
    from ._broadcast import _NPT, broadcast, tag_of, trace
    e = trace(f, [tag_of(d.dtype)])
    if e.jt != "bool":
        raise _non_boolean(_JL[_NPT[e.jt]] if e.jt in _NPT else e.jt)
    return broadcast(f, d)
