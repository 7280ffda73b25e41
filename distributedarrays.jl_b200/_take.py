"""``d[I]`` with ``I`` a DArray of integers (row f12): the gather of K22 (``dab_index_gather``).

The reference defines no ``getindex(d::DArray, I::DArray)``; Base's generic method allocates ``similar(d, axes(I))`` (reference
src/darray.jl:238) -- a DArray of ``I``'s dims with the default layout over ``procs(d)`` -- and fills it with ``R[k] = d[I[k]]``, where
``I[k]`` is a 1-based column-major LINEAR index into ``d`` (Julia's ``A[I::AbstractArray{<:Integer}]``).  Here every localpart of ``R`` is
one K22 launch: the block of ``I`` it reads (``I``'s own chunk when the layouts agree, a halo read otherwise) holds the indices, and
the kernel finds each element's chunk of ``d`` -- local or a CUDA-IPC peer mapping -- from the cuts of ``d``'s layout.

A DArray key holds Julia indices (1-based), like every index DArray the package returns (``sortperm``, ``findmax(d; dims)``); host
Python sequences keep their 0-based meaning.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._darray import B200Array, DArray, SubDArray, similar
from .layout import rlen, shape_of, unravel
from .runtime import close_remote_reads, open_remote_reads

MAX_DIMS = 8              # dab_index_gather serves sources of 1..8 dimensions
MAX_CHUNKS = 1024         # and at most this many chunks (the source table travels in the kernel's parameter block)
_NONE = np.iinfo(np.int64).max


def _source_table(d: DArray):
    """``dab_index_gather``'s description of ``d``: dims, grid, per-dim cuts (0-based chunk starts from the chunk extents, so empty
    chunks repeat a cut) and one pointer per chunk in column-major grid order (NULL for an empty chunk)."""
    lay = d.layout
    cuts = []
    for k, g in enumerate(lay.grid):
        stride = int(np.prod(lay.grid[:k]))
        c = [0]
        for i in range(g):
            c.append(c[-1] + rlen(lay.indices[i * stride][k]))
        cuts += c
    ptrs = [d.peer_ptr(pid) if all(rlen(r) for r in lay.indices[c]) else None for c, pid in enumerate(lay.pids)]
    return ((C.c_size_t * d.ndim)(*d.dims), (C.c_int32 * d.ndim)(*lay.grid), (C.c_size_t * len(cuts))(*cuts),
            (C.c_void_p * len(ptrs))(*ptrs))


def _check(d, I):
    """Every refusal, before anything is allocated or launched."""
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray) or isinstance(I, SparseDArray):
        refuse("indexing by a DArray")
    from ._darray import refuse_float16
    refuse_float16("d[I] with a DArray index (the index gather has no 2-byte instance)", d)
    T = np.dtype(I.dtype)
    if T == np.bool_:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "logical indexing with a DArray{Bool} is not served (its values are not positions)")
    if T.kind in "fc":
        raise _lib.ArgumentError(_lib.ERR_ARG, f"invalid index: a DArray of {T} (Julia's to_index takes integer indices)")
    if T not in (np.dtype(np.int32), np.dtype(np.int64)):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"index element type {T} is not served (Int32, Int64)")
    if d.ndim > MAX_DIMS:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"indexing a DArray of {d.ndim} dimensions (served: up to {MAX_DIMS})")
    if len(d.layout.pids) > MAX_CHUNKS:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"indexing a DArray of {len(d.layout.pids)} chunks (served: up to {MAX_CHUNKS})")


def _index_value(I: DArray, pos: int) -> int:
    """``I[pos + 1]`` (0-based column-major ``pos``) on every rank: its owner reads it from its chunk, the other ranks contribute 0 to
    one small all-gather."""
    rt = I.rt
    coord = unravel(pos, I.dims)
    val = np.zeros(1, dtype=np.int64)
    for c, (Kc, pid) in enumerate(zip(I.layout.indices, I.layout.pids)):
        if all(k[0] - 1 <= x <= k[1] - 1 for x, k in zip(coord, Kc)):
            if pid in I.chunks:
                loc = [x - k[0] + 1 for x, k in zip(coord, Kc)]
                off = int(np.ravel_multi_index(loc, shape_of(Kc), order="F"))
                v = np.zeros(1, dtype=I.dtype)
                _lib.call("dab_d2h", rt.ctx, C.c_void_p(v.ctypes.data), C.c_void_p(I.chunks[pid].ptr + off * I.dtype.itemsize), I.dtype.itemsize)
                rt.sync()
                val[0] = int(v[0])
            break
    return int(sum(int(a[0]) for a in rt.allgather_small(val)))


def _bounds_error(d: DArray, value: int):
    raise IndexError(f"BoundsError: attempt to access {d.size}-element DArray of size {d.dims} at index [{value}]")


def take(d: DArray, I: DArray) -> DArray:
    """``d[I]``: a DArray of ``I``'s dims and ``d``'s element type, with the layout of ``similar(d, size(I))``, holding
    ``d[I[k]]`` (1-based linear indices).  ``IndexError('BoundsError: ...')`` names the first out-of-range value in column-major
    order of ``I``; nothing is left allocated then.  Collective."""
    _check(d, I)
    rt = d.rt
    R = similar(d, dims=I.dims)
    if R.size == 0:
        return R
    if d.size == 0:
        R.close()
        _bounds_error(d, _index_value(I, 0))
    fenced = open_remote_reads(rt, [d, I], "device")
    dims, grid, cuts, ptrs = _source_table(d)
    code = _lib.I32 if I.dtype == np.int32 else _lib.I64
    work = [(pid, ch) for pid, ch in R.chunks.items() if ch.size]
    bad = B200Array.from_numpy(rt, np.full(max(len(work), 1), -1, dtype=np.int64))   # -1 == ULLONG_MAX: no bad position
    temps = []
    same = I.layout.same_as(R.layout)
    try:
        for i, (pid, ch) in enumerate(work):
            J = R.layout.localindices(pid)
            if same and pid in I.chunks:
                blk = I.chunks[pid]
            else:
                blk = B200Array.empty(rt, shape_of(J), I.dtype, temp=True)
                temps.append(blk)
                SubDArray(I, J, tuple(False for _ in J)).copy_to(blk)
            _lib.call("dab_index_gather", rt.ctx, d.dtype.itemsize, C.c_void_p(ch.ptr), C.c_void_p(blk.ptr), code, ch.size, d.ndim,
                      dims, grid, cuts, ptrs, C.c_void_p(bad.ptr + 8 * i))
    except BaseException:
        bad.free()                                                # an unexpected failure still leaves nothing allocated
        R.close()
        raise
    finally:
        for t in temps:
            t.free()                                              # stream-ordered
    close_remote_reads(rt, fenced, "device")
    slots = bad.to_numpy().view(np.uint64)
    bad.free()
    first = _NONE
    for (pid, ch), s in zip(work, slots):
        if s != np.uint64(0xFFFFFFFFFFFFFFFF):
            J = R.layout.localindices(pid)
            loc = unravel(int(s), ch.shape)
            first = min(first, int(np.ravel_multi_index([x + j[0] - 1 for x, j in zip(loc, J)], I.dims, order="F")))
    first = min(int(a[0]) for a in rt.allgather_small(np.array([first], dtype=np.int64)))
    if first != _NONE:
        R.close()
        _bounds_error(d, _index_value(I, first))
    return R
