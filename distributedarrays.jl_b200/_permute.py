"""``permutedims(A, perm)``, ``permutedims(A)`` and ``permutedims!(dest, src, perm)`` (row f18): K28 ``dab_permute_box``.

The reference defines no method of its own; Base's generic ``permutedims`` reads a DArray with one scalar ``getindex`` -- one
``remotecall_fetch`` -- per element.  Here every chunk of the destination is filled by its owner from the pieces of the source it
needs (local or CUDA-IPC peer loads), one launch per piece:

* ``permute_plan`` is a pure function of the two layouts: per destination chunk the preimage box in the source, split over the source
  chunks by ``layout.slab_plan``; each piece gets its offsets, both stride lists and its extents, collapsed (extent-1 dimensions
  dropped, destination-adjacent dimensions that are contiguous on both sides merged) and a mover;
* a piece whose destination dimension 0 is also contiguous in the source is a batch of contiguous runs: ``dab_gather_box``, and so
  is a piece whose plane of the two contiguous dimensions is too small to fill a tile (``PERMUTE_MIN_PLANE``); any other piece goes to
  ``dab_permute_box``, which tiles that plane through shared memory.

A matrix with ``perm = (2, 1)`` goes through ``copy_transposed`` (K10), exactly as ``copy(transpose(A))``.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

from . import _lib
from ._darray import B200Array, DArray, SubDArray, darray
from .layout import Layout, rlen, shape_of, slab_plan
from .runtime import close_remote_reads, open_remote_reads

MAX_DIMS = 8                                  # dab_gather_box and dab_permute_box serve up to 8 dimensions


@dataclass
class PermutePiece:
    dst_chunk: int                   # 0-based chunk of the destination (owner: dst_layout.pids[dst_chunk])
    src_chunk: int                   # 0-based chunk of the source it reads
    dst_offset: int                  # element offset of the piece's first element in the destination chunk
    src_offset: int                  # and in the source chunk
    extent: Tuple[int, ...]          # collapsed extents, destination dimension order
    dst_strides: Tuple[int, ...]     # elements
    src_strides: Tuple[int, ...]
    mover: str                       # "gather" (dab_gather_box) or "permute" (dab_permute_box)


def _strides(shape: Sequence[int]) -> List[int]:
    return [int(v) for v in np.cumprod((1,) + tuple(shape[:-1]), dtype=np.int64)]


def collapse(extent: Sequence[int], dst_strides: Sequence[int], src_strides: Sequence[int]):
    """Drop extent-1 dimensions, then merge destination-adjacent dimensions k, k+1 when both stride lists are contiguous across them
    (``stride[k+1] == stride[k] * extent[k]`` on both sides).  A box of one element keeps one dimension of extent 1."""
    kept = [(e, d, s) for e, d, s in zip(extent, dst_strides, src_strides) if e != 1] or [(1, 1, 1)]
    out = [list(kept[0])]
    for e, d, s in kept[1:]:
        pe, pd, ps = out[-1]
        if d == pd * pe and s == ps * pe:
            out[-1][0] = pe * e
        else:
            out.append([e, d, s])
    return tuple(o[0] for o in out), tuple(o[1] for o in out), tuple(o[2] for o in out)


# Fewest plane elements (extent of dim 0 x extent of the source-contiguous dim, after collapsing) for which dab_permute_box beats
# dab_gather_box, by element size; below it the tile is mostly idle (one batch entry per tile).  The crossover points measured on an
# H100 with square and rectangular planes of every element size (DESIGN section 6).
PERMUTE_MIN_PLANE = {1: 1536, 2: 512, 4: 1024, 8: 512, 16: 512}
PERMUTE_MIN_SIDE_BYTES = 16               # and each plane side at least this long: 4 x 1024 Float16 planes are faster gathered


def permute_box_applies(extent: Sequence[int], dst_strides: Sequence[int], src_strides: Sequence[int]) -> bool:
    """``dab_permute_box``'s precondition: destination dimension 0 contiguous and exactly one other dimension contiguous in the source."""
    return len(extent) >= 2 and dst_strides[0] == 1 and sum(1 for s in src_strides[1:] if s == 1) == 1


def select_mover(extent: Sequence[int], dst_strides: Sequence[int], src_strides: Sequence[int], elem_bytes: int) -> str:
    """``dab_permute_box`` when it applies and its plane is large enough (``PERMUTE_MIN_PLANE``, ``PERMUTE_MIN_SIDE_BYTES``); otherwise
    ``dab_gather_box`` (the source's unit-stride dimension IS dimension 0: a batch of contiguous runs; a side without a unit stride; or
    a plane so small that most of a tile would be idle)."""
    if not permute_box_applies(extent, dst_strides, src_strides):
        return "gather"
    e0, eq = extent[0], extent[1 + list(src_strides[1:]).index(1)]
    if e0 * eq < PERMUTE_MIN_PLANE[elem_bytes] or min(e0, eq) * elem_bytes < PERMUTE_MIN_SIDE_BYTES:
        return "gather"
    return "permute"


def permute_plan(src_layout: Layout, dst_layout: Layout, perm: Sequence[int], elem_bytes: int) -> List[PermutePiece]:
    """Every launch of ``permutedims!(dest, src, perm)`` (1-based ``perm``; ``size(dest, k) == size(src, perm[k])``) for elements of
    ``elem_bytes`` bytes, in destination chunk order, then source chunk order.  Empty chunks and empty pieces give none."""
    N = len(perm)
    out = []
    for c, I in enumerate(dst_layout.indices):
        if any(rlen(r) == 0 for r in I):
            continue
        J = [None] * N                                     # the preimage box: source dim perm[k] spans I[k]
        for k in range(N):
            J[perm[k] - 1] = I[k]
        dstr = _strides(shape_of(I))
        for piece in slab_plan(src_layout, J):
            sstr = _strides(shape_of(src_layout.indices[piece.chunk]))
            src_off = sum((piece.src[j][0] - 1) * sstr[j] for j in range(N))
            dst_off = sum((piece.dst[perm[k] - 1][0] - 1) * dstr[k] for k in range(N))
            ext = [rlen(piece.src[perm[k] - 1]) for k in range(N)]
            e, ds, ss = collapse(ext, dstr, [sstr[perm[k] - 1] for k in range(N)])
            out.append(PermutePiece(c, piece.chunk, dst_off, src_off, e, ds, ss, select_mover(e, ds, ss, elem_bytes)))
    return out


def _check_perm(perm, N: int) -> Tuple[int, ...]:
    """Base's ``checkdims_perm`` (base/permuteddimsarray.jl) for the length and the permutation."""
    try:
        p = tuple(perm)
    except TypeError:
        raise _lib.ArgumentError(_lib.ERR_ARG, "input is not a permutation") from None
    if len(p) != N:
        raise _lib.ArgumentError(_lib.ERR_ARG, f"expected permutation of size {N}, but length(perm)={len(p)}")
    if not all(isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)) for v in p) or sorted(int(v) for v in p) != list(range(1, N + 1)):
        raise _lib.ArgumentError(_lib.ERR_ARG, "input is not a permutation")
    return tuple(int(v) for v in p)


def _refuse_operand(x, what: str):
    from ._sparse import SparseDArray, refuse
    if isinstance(x, SparseDArray):
        refuse(what)
    if isinstance(x, SubDArray):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} of a view is not served (make it a DArray with .to_darray() first)")
    if not isinstance(x, DArray):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} is served for a dense DArray, not {type(x).__name__}")


def _refuse_dims(N: int, what: str):
    if N > MAX_DIMS:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} of a DArray of {N} dimensions (served: up to {MAX_DIMS})")


def _shares_storage(dest: DArray, src: DArray) -> bool:
    """Whether a chunk of ``dest`` overlaps a chunk of ``src`` in this rank's memory, agreed by every rank."""
    if dest is src:
        return True
    spans = [(ch.ptr, ch.ptr + ch.nbytes) for ch in src.chunks.values() if ch.size]
    mine = any(a < e and s < b for ch in dest.chunks.values() if ch.size for a, b in [(ch.ptr, ch.ptr + ch.nbytes)] for s, e in spans)
    rt = src.rt
    if rt.world == 1:
        return mine
    return any(int(x[0]) for x in rt.allgather_small(np.array([int(mine)], dtype=np.int64)))


def _run(dest: DArray, src: DArray, perm: Tuple[int, ...], src_layout: Layout = None) -> DArray:
    """One launch per piece of ``dest``'s local chunks; ``src_layout`` (default ``src.layout``) describes ``src``'s chunks."""
    rt = src.rt
    es = src.dtype.itemsize
    src_layout = src.layout if src_layout is None else src_layout
    plan = permute_plan(src_layout, dest.layout, perm, es)
    fenced = open_remote_reads(rt, [src], "host")
    try:
        for p in plan:
            pid = dest.layout.pids[p.dst_chunk]
            if pid not in dest.chunks:
                continue
            nd = len(p.extent)
            dptr = C.c_void_p(dest.chunks[pid].ptr + p.dst_offset * es)
            sptr = C.c_void_p(src.peer_ptr(src_layout.pids[p.src_chunk]) + p.src_offset * es)
            LL = C.c_longlong * nd
            ext = (C.c_size_t * nd)(*p.extent)
            if p.mover == "permute":
                _lib.call("dab_permute_box", rt.ctx, es, nd, dptr, LL(*p.dst_strides), sptr, LL(*p.src_strides), ext)
            else:
                _lib.call("dab_gather_box", rt.ctx, es, nd, dptr, LL(*p.dst_strides), None, sptr, LL(*p.src_strides), None, ext)
    finally:
        close_remote_reads(rt, fenced, "host")          # a failed launch on one rank must not leave the others at the fence
    return dest


def permutedims(A: DArray, perm=None) -> DArray:
    """``permutedims(A, perm)``: a new DArray ``B`` of the permuted dims on ``procs(A)`` with the default distribution, ``size(B, k) ==
    size(A, perm[k])`` and ``B[i...] = A[j...]`` with ``j[perm[k]] = i[k]`` (1-based ``perm``, like every ``dims`` here); NumPy's
    ``np.transpose(a, [p - 1 for p in perm])``.  Bit-exact for every element type; complex values are not conjugated.
    ``permutedims(A)`` of a DMatrix is ``perm = (2, 1)``; of a DVector a 1 x n DMatrix (a copy).  Collective."""
    _refuse_operand(A, "permutedims")
    if perm is None:
        if A.ndim == 1:
            return _vector_row(A)
        if A.ndim != 2:
            raise TypeError(f"MethodError: permutedims(A) is defined for a vector or a matrix, not for {A.ndim} dimensions "
                            "(give perm)")
        perm = (2, 1)
    p = _check_perm(perm, A.ndim)
    _refuse_dims(A.ndim, "permutedims")
    if p == (2, 1):
        from ._linalg import copy_transposed, transpose
        return copy_transposed(transpose(A))               # copy(transpose(A)): the same launches, bit for bit
    rt = A.rt
    dims = tuple(A.dims[k - 1] for k in p)
    B = darray(lambda I: B200Array.empty(rt, shape_of(I), A.dtype), dims, procs=list(A.layout.pids), dtype=A.dtype, rt=rt)
    try:
        return _run(B, A, p)
    except BaseException:
        B.close()
        raise


def _vector_row(v: DArray) -> DArray:
    """``permutedims(v::AbstractVector)``: the 1 x n DMatrix holding ``v``, on ``procs(v)`` with the default distribution.  The source is
    read as the n x 1 matrix its chunks already are, so every piece is a contiguous run (``dab_gather_box``)."""
    rt = v.rt
    lay = v.layout
    col = Layout(lay.dims + (1,), lay.grid + (1,), list(lay.pids), [I + ((1, 1),) for I in lay.indices], lay.cuts + [[1, 2]])
    B = darray(lambda I: B200Array.empty(rt, shape_of(I), v.dtype), (1, v.dims[0]), procs=list(lay.pids), dtype=v.dtype, rt=rt)
    try:
        return _run(B, v, (2, 1), src_layout=col)
    except BaseException:
        B.close()
        raise


def permutedims_(dest: DArray, src: DArray, perm) -> DArray:
    """``permutedims!(dest, src, perm)``: fills ``dest`` (any layout, any grid) with ``permutedims(src, perm)``; each rank writes the
    chunks of ``dest`` it owns.  ``dest`` must have ``src``'s element type and must not share storage with ``src``.  Collective."""
    _refuse_operand(src, "permutedims!")
    _refuse_operand(dest, "permutedims! into a destination")
    p = _check_perm(perm, src.ndim)
    if dest.ndim != src.ndim or any(dest.dims[k] != src.dims[p[k] - 1] for k in range(src.ndim)):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "destination tensor of incorrect size")
    _refuse_dims(src.ndim, "permutedims!")
    if dest.dtype != src.dtype:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"permutedims! from {src.dtype} into {dest.dtype} is not served (the element "
                                    "types must be equal; convert first)")
    if _shares_storage(dest, src):
        raise _lib.ArgumentError(_lib.ERR_ARG, "permutedims!: dest and src share storage (the result would be unspecified)")
    return _run(dest, src, p)
