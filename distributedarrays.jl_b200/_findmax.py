"""``findmax`` / ``findmin`` / ``argmax`` / ``argmin`` of a DArray, with and without ``dims``: index-carrying reductions (K20,
``csrc/dab_findminmax.cu``).

In the reference these come from Base's generic code: ``findmax(f, d)`` is a ``mapfoldl`` over ``pairs(d)`` with one scalar
``getindex`` (a ``remotecall_fetch``) per element, and ``findmax(f, d; dims)`` goes through ``findminmax!``.  Here every chunk is reduced by
one kernel and only the chunk winners travel.

Order (Julia 1.10): ``findmax`` replaces the best ``(v, i)`` by a later ``(x, k)`` when ``isless(v, x)``, ``findmin`` when
``isgreater(v, x)``.  So NaN wins and the first NaN is kept, ``findmax`` prefers +0.0 to -0.0 and ``findmin`` -0.0 to +0.0, and ties keep
the earlier index.  The winner is therefore the maximal element under (order key, then smaller GLOBAL column-major linear index), an order
in which chunks combine in any order: the chunk results are made global and folded by ``dab_combine_findminmax``, and the ``dims`` slabs
carry global indices from the first pass on.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Optional

import numpy as np

from . import _lib
from ._broadcast import broadcast, is_ctag
from ._darray import B200Array, DArray, dab_dtype, is_complex, refuse_float16
from ._mapreduce import _gather_slots, _normalise_region, classify_map, gather_fibres, plan_reducedim
from .layout import reduction_passes, shape_of

_SERVED_MAPS = (_lib.MAP_ID, _lib.MAP_ABS, _lib.MAP_ABS2)
_I64 = C.c_int64


def _not_ordered(dt):
    raise TypeError(f"MethodError: no method matching isless(::{dt}, ::{dt}) -- complex numbers are not ordered")


def _global0(L, pid: int, local: int) -> int:
    """0-based chunk-local linear index of chunk ``pid`` -> 0-based global linear index (column-major)."""
    I = L.localindices(pid)
    coords = np.unravel_index(int(local), shape_of(I), order="F")
    return int(np.ravel_multi_index(tuple(int(c) + lo - 1 for c, (lo, _) in zip(coords, I)), L.dims, order="F"))


def _julia_index(d: DArray, g0: int):
    """Julia's index of the element at 0-based global linear index g0: an Int for a vector, a CartesianIndex (tuple) otherwise."""
    if d.ndim == 1:
        return g0 + 1
    return tuple(int(c) + 1 for c in np.unravel_index(g0, d.dims, order="F"))


def _findminmax(which: int, f: Optional[Callable], d, dims):
    from ._darray import SubDArray
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray):
        refuse("findmax / findmin / argmax / argmin")
    view = isinstance(d, SubDArray)
    refuse_float16("findmax / findmin / argmax / argmin", d)
    if is_complex(d.dtype):                          # every check on the view itself: nothing is copied or launched before an error
        _not_ordered(d.dtype)
    mapc, _, expr = classify_map(f, d.dtype)
    if expr is not None and is_ctag(expr.jt):
        _not_ordered(expr.jt)
    _check_sizes(tuple(d.shape) if view else tuple(d.dims), dims)
    if view:                                         # reduced through DArray(view), as mapreduce does: indices relative to the view
        tmp = d.to_darray()
        try:
            return _findminmax(which, f, tmp, dims)
        finally:
            tmp.close()
    if dims is not None:
        _check_index_geometry(d.layout)
    if mapc not in _SERVED_MAPS:
        tmp = broadcast(f, d)                        # a general f: the elementwise temporary f.(d) (same layout), then the plain reduction
        try:
            return _findminmax(which, None, tmp, dims)
        finally:
            tmp.close()
    if dims is None:
        return _whole(which, mapc, d)
    return _dims(which, mapc, d, dims)


def _check_sizes(shape, dims):
    size = int(np.prod(shape))
    if dims is None:
        if size == 0:
            raise _lib.ArgumentError(_lib.ERR_EMPTY, "reducing over an empty collection is not allowed")
        return
    region = _normalise_region(dims, len(shape))
    if size == 0 and int(np.prod([1 if k + 1 in region else s for k, s in enumerate(shape)])) != 0:
        raise _lib.ArgumentError(_lib.ERR_ARG, "ArgumentError: collection slices must be non-empty")


_MAX_INDEX_DIMS = 8                                  # dab_findminmax_dim: chunk position -> global index over at most 8 dims


def _index_geometry(L, pid: int):
    """(chunk dims, 0-based offsets, global dims) of chunk ``pid`` for the position -> global index map of ``dab_findminmax_dim``, with
    adjacent dims merged wherever the chunk spans the whole global extent of the lower one (then the merged coordinate is still the chunk
    coordinate plus a constant offset).  Only dims that are cut across chunks start a new group, so any layout with fewer than 2^8 chunks
    fits the kernel's 8 dims."""
    I = L.localindices(pid)
    cd, off, gd = [], [], []
    for (lo, hi), g in zip(I, L.dims):
        c, o = hi - lo + 1, lo - 1
        if cd and cd[-1] == gd[-1]:                  # the lower group is whole: merge this dim into it
            off[-1] += gd[-1] * o
            cd[-1] *= c
            gd[-1] *= g
        else:
            cd.append(c)
            off.append(o)
            gd.append(g)
    return cd, off, gd


def _check_index_geometry(L):
    for pid in L.pids:
        if int(np.prod(shape_of(L.localindices(pid)))) and len(_index_geometry(L, pid)[0]) > _MAX_INDEX_DIMS:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"findmax / findmin with dims: chunk {pid} of this layout is cut along more than "
                                        f"{_MAX_INDEX_DIMS} groups of dims; the kernels map chunk positions to global indices over at most "
                                        f"{_MAX_INDEX_DIMS}")


def _whole(which: int, mapc: int, d: DArray):
    rt, code, L = d.rt, dab_dtype(d.dtype), d.layout

    def launch(pid, ch, slot):
        if ch.size:
            _lib.call("dab_findminmax", rt.ctx, code, which, mapc, None, C.c_void_p(ch.ptr), ch.size, C.c_void_p(int(slot)))

    host = _gather_slots(d, launch)
    recs = []
    for pid in L.pids:
        if int(np.prod(shape_of(L.localindices(pid)))) == 0:
            continue
        rec = host[16 * (pid - 1):16 * pid].copy()
        rec[8:16] = np.asarray([_global0(L, pid, int(rec[8:16].view(np.int64)[0]))], dtype=np.int64).view(np.uint8)
        recs.append(rec)
    recs = np.concatenate(recs)
    out = np.zeros(16, dtype=np.uint8)
    _lib.check(_lib.lib().dab_combine_findminmax(code, which, C.c_void_p(recs.ctypes.data), recs.size // 16, C.c_void_p(out.ctypes.data)))
    return out[:d.dtype.itemsize].view(d.dtype)[0], _julia_index(d, int(out[8:16].view(np.int64)[0]))


def _chunk_pass(rt, code, which, mapc, x_ptr, idx_ptr, inner, red, outer, gl, dtype):
    vals = B200Array.empty(rt, (inner * outer,), dtype)          # not pooled: a pass's output may become a chunk of the result
    idx = B200Array.empty(rt, (inner * outer,), np.int64)
    nd, cd, off, gd = gl
    _lib.call("dab_findminmax_dim", rt.ctx, code, which, mapc, C.c_void_p(x_ptr), C.c_void_p(idx_ptr) if idx_ptr else None, inner, red, outer,
              nd, cd, off, gd, C.c_void_p(vals.ptr), C.c_void_p(idx.ptr))
    return vals, idx


def _reduce_chunk(rt, d: DArray, pid: int, ch: B200Array, reg_in, which: int, mapc: int):
    """Phase 1 on one chunk: every maximal run of reduced dims is one (inner, red, outer) pass, last run first; the first pass turns
    positions into 1-based global indices, the later ones carry them (index input).  No reduced dim in the chunk (dims beyond ndims): one
    pass with red = 1, which maps the values and numbers them."""
    code = dab_dtype(d.dtype)
    cd, off, gd = _index_geometry(d.layout, pid)
    nd = len(cd)
    gl = (nd, (_I64 * nd)(*cd), (_I64 * nd)(*off), (_I64 * nd)(*gd))
    if ch.size == 0:                                 # empty along a reduced dim only: a slab of "no element" entries (index -1)
        n = int(np.prod([1 if k + 1 in reg_in else s for k, s in enumerate(ch.shape)]))
        vals, idx = B200Array.empty(rt, (n,), d.dtype), B200Array.empty(rt, (n,), np.int64)
        if n:
            _lib.call("dab_fill", rt.ctx, code, C.c_void_p(vals.ptr), n, C.c_void_p(np.zeros(1, dtype=np.uint64).ctypes.data))
            _lib.call("dab_fill", rt.ctx, _lib.I64, C.c_void_p(idx.ptr), n, C.c_void_p(np.full(1, -1, dtype=np.int64).ctypes.data))
        return vals, idx
    vals = idx = None
    for inner, red, outer in reduction_passes(ch.shape, reg_in):
        if vals is None:
            vals, idx = _chunk_pass(rt, code, which, mapc, ch.ptr, 0, inner, red, outer, gl, d.dtype)
        else:
            nv, ni = _chunk_pass(rt, code, which, _lib.MAP_ID, vals.ptr, idx.ptr, inner, red, outer, gl, d.dtype)
            vals.free()
            idx.free()
            vals, idx = nv, ni
    if vals is None:
        vals, idx = _chunk_pass(rt, code, which, mapc, ch.ptr, 0, ch.size, 1, 1, gl, d.dtype)
    return vals, idx


def _dims(which: int, mapc: int, d: DArray, dims):
    rt, L, N = d.rt, d.layout, d.ndim
    region = _normalise_region(dims, N)
    reg_in = tuple(r for r in region if r <= N)
    Rlayout, fibres = plan_reducedim(L, reg_in)
    Rpids, Rindices = Rlayout.pids, Rlayout.indices
    plens = [int(np.prod(shape_of(ix))) for ix in Rindices]
    code, isz = dab_dtype(d.dtype), d.dtype.itemsize
    Vchunks: Dict[int, B200Array] = {}
    Ichunks: Dict[int, B200Array] = {}
    if d.size == 0:                                  # a zero-length kept dimension: empty results in R's layout
        for rl, owner in enumerate(Rpids):
            if rt.rank_of(owner) == rt.rank:
                Vchunks[owner] = B200Array.empty(rt, shape_of(Rindices[rl]), d.dtype)
                Ichunks[owner] = B200Array.empty(rt, shape_of(Rindices[rl]), np.int64)
        return DArray(Rlayout, d.dtype, Vchunks, rt), DArray(Rlayout, np.dtype(np.int64), Ichunks, rt)
    # ---- phase 1: every chunk reduced along the region, indices made global
    partial = {pid: _reduce_chunk(rt, d, pid, ch, reg_in, which, mapc) for pid, ch in d.chunks.items()}
    # ---- phase 2: the (values, indices) slabs of a fibre gathered on the owner of the R chunk and folded there.  A fibre of one member
    # gathers nothing: its slab is already on the owner.
    stack_temp = 0
    try:
        st, stacks = gather_fibres(rt, L, Rlayout, [m if len(m) > 1 else [] for m in fibres], [(plen * isz, plen * 8) for plen in plens],
                                   {pid: (v.ptr, i.ptr) for pid, (v, i) in partial.items()})
        stack_temp = st.temp
        for rl, (vbase, ibase) in stacks.items():
            owner, members = Rpids[rl], fibres[rl]
            shape = shape_of(Rindices[rl])
            if len(members) == 1:                    # the owner's own slab is the result (no reduced dim cut across chunks)
                v, i = partial.pop(owner)
                v.shape, i.shape = shape, shape
                Vchunks[owner], Ichunks[owner] = v, i
                continue
            Vch, Ich = B200Array.empty(rt, shape, d.dtype), B200Array.empty(rt, shape, np.int64)
            _lib.call("dab_findminmax_dim", rt.ctx, code, which, _lib.MAP_ID, C.c_void_p(vbase), C.c_void_p(ibase), plens[rl],
                      len(members), 1, 0, None, None, None, C.c_void_p(Vch.ptr), C.c_void_p(Ich.ptr))
            Vchunks[owner], Ichunks[owner] = Vch, Ich
    finally:
        rt.free_temp(stack_temp)
        for v, i in partial.values():
            v.free()
            i.free()
    return DArray(Rlayout, d.dtype, Vchunks, rt), DArray(Rlayout, np.dtype(np.int64), Ichunks, rt)


def findmax(f, d=None, dims=None):
    """``findmax(d)`` -> ``(value, index)``; ``findmax(f, d)`` -> ``(f(x), index)``; with ``dims`` -> ``(values::DArray,
    indices::DArray{Int64})`` of 1-based global linear indices.  The index of a whole-array call is Julia's: an Int for a vector, a tuple
    of 1-based ints (CartesianIndex) otherwise."""
    if d is None:
        f, d = None, f
    return _findminmax(_lib.FINDMAX, f, d, dims)


def findmin(f, d=None, dims=None):
    """``findmin`` with the same forms and return values as ``findmax``."""
    if d is None:
        f, d = None, f
    return _findminmax(_lib.FINDMIN, f, d, dims)


def argmax(d, dims=None):
    """``argmax(d)``: the index part of ``findmax(d)``; with ``dims`` the index DArray."""
    v, i = findmax(d, dims=dims)
    if dims is not None:
        v.close()
    return i


def argmin(d, dims=None):
    """``argmin(d)``: the index part of ``findmin(d)``; with ``dims`` the index DArray."""
    v, i = findmin(d, dims=dims)
    if dims is not None:
        v.close()
    return i
