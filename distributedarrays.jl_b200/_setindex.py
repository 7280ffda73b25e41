"""``d[key] = v`` and ``copyto(view, src)`` (row f14): Julia's ``setindex!`` on a DArray, which the reference leaves to Base's generic
method (one remote write per element).

Keys follow ``__getitem__``: host keys (ints, slices with any step, int lists and arrays) are 0-based; a DArray of Int32 / Int64 holds
Julia's 1-based column-major linear indices (K24, ``dab_scatter*``); a Bool DArray of ``d``'s dims is a mask (K25, ``dab_expand``).
Values are a scalar (written to every selected position: Julia's ``d[key] .= x``), a host array (converted with ``astype(d.dtype)``, as
``copyto`` does) or a DArray / SubDArray in any layout (converted by the identity broadcast of ``copyto`` when its element type differs).

The result is Julia's sequential one, bit for bit: a position selected twice keeps the value of its last occurrence in column-major
order of the key; every index is checked before the first store, so a ``BoundsError`` leaves ``d`` unchanged; a value or index that
shares storage with ``d`` is copied first (``Base.unalias``).  Every call is collective.
"""
from __future__ import annotations

import ctypes as C
from typing import List

import numpy as np

from . import _lib
from ._darray import B200Array, DArray, SubDArray, dab_dtype, similar
from .layout import Layout, shape_of, unravel
from .runtime import close_remote_reads, open_remote_reads

_NONE = np.iinfo(np.int64).max


def _squeeze(shape) -> tuple:
    return tuple(int(s) for s in shape if s != 1)


def _mismatch(what, got, want):
    raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"tried to assign {what} of size {tuple(got)} to a selection of size {tuple(want)}")


def _is_scalar(v) -> bool:
    return np.isscalar(v) or (isinstance(v, np.ndarray) and v.ndim == 0)


def _scalar_bytes(d: DArray, v) -> np.ndarray:
    """The scalar as one element of ``d``'s type (``fill!``'s conversion)."""
    return np.asarray(v, dtype=d.dtype).reshape(1)


def _value_darray(v, d: DArray, shape, owned: List[DArray]) -> DArray:
    """The DArray value ``v`` as a DArray of ``d``'s element type and dims ``shape`` (``v``'s dims once singleton dims are dropped): ``v``
    itself when it already is one and shares no storage with ``d``; otherwise a copy, appended to ``owned``."""
    from ._broadcast import copy
    if isinstance(v, SubDArray):
        w = v.to_darray()                                    # a copy: also unaliases a view of d
        owned.append(w)
    elif v is d:
        w = copy(v)
        owned.append(w)
    else:
        w = v
    if w.dims != tuple(shape):                               # the same elements in the same column-major order, other singleton dims
        r = similar(w, dims=tuple(shape))
        owned.append(r)
        rt = w.rt
        big = [k for k, s in enumerate(w.dims) if s != 1]
        fenced = open_remote_reads(rt, [w], "device")
        for pid, ch in r.chunks.items():
            if not ch.size:
                continue
            I = [rg for rg, s in zip(r.layout.localindices(pid), shape) if s != 1]
            J = [(1, 1)] * w.ndim
            for k, rg in zip(big, I):
                J[k] = rg
            SubDArray(w, tuple(J), tuple(False for _ in J)).copy_to(B200Array(rt, ch.ptr, shape_of(J), w.dtype, own=False))
        close_remote_reads(rt, fenced, "device")
        w = r
    if w.dtype != d.dtype:
        from ._darray import copyto, darray_like
        c = darray_like(lambda I: B200Array.empty(w.rt, shape_of(I), d.dtype), w, dtype=d.dtype)
        owned.append(c)
        copyto(c, w)                                         # the identity broadcast of copyto(dest, DArray), with its refusals
        w = c
    return w


def _aux_table(d: DArray, per_chunk, dtype) -> DArray:
    """One zeroed device table per chunk of ``d`` (``per_chunk(chunk length)`` elements of ``dtype``) on the chunk's worker, held as a 1-D
    DArray so that other ranks can map it; the caller closes it."""
    rt = d.rt
    lens = [int(np.prod(shape_of(K))) for K in d.layout.indices]
    sizes = [per_chunk(n) for n in lens]
    ends = np.cumsum(sizes)
    idx = [((int(e) - s + 1, int(e)),) for e, s in zip(ends, sizes)]
    lay = Layout((int(ends[-1]),), (len(sizes),), list(d.layout.pids), idx, [[1] + sorted({int(e) + 1 for e in ends})])
    zero = np.zeros(1, dtype=dtype)
    chunks = {}
    for pid, n in zip(d.layout.pids, sizes):
        if rt.is_local(pid):
            ch = B200Array.empty(rt, (n,), dtype)
            chunks[pid] = ch
            if n:
                _lib.call("dab_fill", rt.ctx, dab_dtype(dtype), C.c_void_p(ch.ptr), n, C.c_void_p(zero.ctypes.data))
    return DArray(lay, dtype, chunks, rt)


def _aux_ptrs(d: DArray, aux: DArray):
    lens = [int(np.prod(shape_of(K))) for K in d.layout.indices]
    return (C.c_void_p * len(lens))(*[aux.peer_ptr(pid) if n else None for n, pid in zip(lens, d.layout.pids)])


# ---- d[I] = v, I a DArray of integers: K24 ---------------------------------------------------------------------------------------------


def setindex_take(d: DArray, I: DArray, v):
    """``d[I] = v`` for a DArray ``I`` of 1-based linear indices (``take``'s keys and refusals).  Duplicates: the last occurrence in
    column-major order of ``I`` wins.  A bad index raises ``IndexError('BoundsError: ...')`` naming the first one, with ``d`` unchanged."""
    from ._broadcast import copy
    from ._compact import run_plan
    from ._take import _bounds_error, _check, _index_value, _source_table
    _check(d, I)
    rt = d.rt
    n = I.size
    scalar = _is_scalar(v)
    if not scalar:
        vs = np.shape(v) if not isinstance(v, (DArray, SubDArray)) else tuple(v.dims)
        if _squeeze(vs) != _squeeze(I.dims):
            _mismatch("an array", vs, I.dims)
    if n == 0:
        return
    if d.size == 0:
        _bounds_error(d, _index_value(I, 0))
    owned: List[DArray] = []
    temps: List[B200Array] = []
    try:
        if I is d:
            I = copy(I)                                       # Base.unalias: the indices are read while d is written
            owned.append(I)
        host = None
        w = None
        if scalar:
            sv = _scalar_bytes(d, v)
        elif isinstance(v, (DArray, SubDArray)):
            w = _value_darray(v, d, I.dims, owned)
        else:
            host = np.asarray(v).astype(d.dtype, copy=False).reshape(I.dims, order="F")
        work = [(c, pid) for c, pid in enumerate(I.layout.pids) if pid in I.chunks and I.chunks[pid].size]
        code = _lib.I32 if I.dtype == np.int32 else _lib.I64
        es = d.dtype.itemsize

        # check pass: bounds and duplicates, before anything is written
        bm = _aux_table(d, lambda m: -(-m // 32), np.int32)
        owned.append(bm)
        status = B200Array.from_numpy(rt, np.tile(np.array([-1, 0], dtype=np.int64), max(len(work), 1)))
        temps.append(status)
        halo = w is not None and not w.layout.same_as(I.layout)
        fenced = open_remote_reads(rt, [d, bm] + ([w] if halo else []), "device")
        dims, grid, cuts, dptrs = _source_table(d)
        bptrs = _aux_ptrs(d, bm)
        blocks = []
        for i, (c, pid) in enumerate(work):
            _lib.call("dab_scatter_check", rt.ctx, C.c_void_p(I.chunks[pid].ptr), code, I.chunks[pid].size, d.ndim, dims, grid, cuts, bptrs,
                      C.c_void_p(status.ptr + 16 * i))
            J = I.layout.localindices(pid)
            if w is None:
                blk = None
                if host is not None:                          # the values of this block of I, uploaded
                    blk = B200Array.empty(rt, shape_of(J), d.dtype, temp=True)
                    temps.append(blk)
                    blk.copy_from_host(host[tuple(slice(lo - 1, hi) for lo, hi in J)])
            elif not halo:
                blk = w.chunks[pid]
            else:                                             # a halo read of the values into the block's shape
                blk = B200Array.empty(rt, shape_of(J), d.dtype, temp=True)
                temps.append(blk)
                SubDArray(w, J, tuple(False for _ in J)).copy_to(blk)
            blocks.append(blk)
        close_remote_reads(rt, fenced, "device")              # every rank's atomics into the bitmaps have landed
        slots = status.to_numpy().view(np.uint64).reshape(-1, 2)
        first, dup = _NONE, 0
        for (c, pid), (s, f) in zip(work, slots):
            dup |= int(f)
            if s != np.uint64(0xFFFFFFFFFFFFFFFF):
                J = I.layout.localindices(pid)
                loc = unravel(int(s), I.chunks[pid].shape)
                first = min(first, int(np.ravel_multi_index([x + j[0] - 1 for x, j in zip(loc, J)], I.dims, order="F")))
        got = rt.allgather_small(np.array([first, dup], dtype=np.int64))
        first = min(int(a[0]) for a in got)
        dup = max(int(a[1]) for a in got)
        if first != _NONE:
            _bounds_error(d, _index_value(I, first))

        # duplicates: the last occurrence of every destination, in a winner table allocated before any store
        wb, win, wptrs, runs = 0, None, None, {}
        if dup:
            wb = 4 if n < (1 << 32) else 8
            win = _aux_table(d, lambda m: m, np.int32 if wb == 4 else np.int64)
            owned.append(win)
            plan, _ = run_plan(I.layout)
            for c, pid in work:
                run_len, _, lin = plan[c]
                t = B200Array.from_numpy(rt, np.ascontiguousarray(lin, dtype=np.int64))
                temps.append(t)
                runs[c] = (run_len, t)
            fenced = open_remote_reads(rt, [win], "device")
            wptrs = _aux_ptrs(d, win)
            for c, pid in work:
                _lib.call("dab_scatter_winners", rt.ctx, C.c_void_p(I.chunks[pid].ptr), code, I.chunks[pid].size, runs[c][0],
                          C.c_void_p(runs[c][1].ptr), wb, d.ndim, dims, grid, cuts, wptrs)
            close_remote_reads(rt, fenced, "device")

        # the stores
        fenced = open_remote_reads(rt, [d] + ([win] if win is not None else []), "device")
        for (c, pid), blk in zip(work, blocks):
            rl, rtab = runs.get(c, (0, None))
            _lib.call("dab_scatter", rt.ctx, es, C.c_void_p(I.chunks[pid].ptr), code, I.chunks[pid].size,
                      None if blk is None else C.c_void_p(blk.ptr), None if blk is not None else C.c_void_p(sv.ctypes.data), rl,
                      None if rtab is None else C.c_void_p(rtab.ptr), wb, d.ndim, dims, grid, cuts, dptrs, wptrs)
        close_remote_reads(rt, fenced, "device")              # the peer stores into d have landed before its owners go on
    finally:
        for t in temps:
            t.free()                                          # stream-ordered
        for a in owned:
            a.close()


# ---- d[m] = v, m a Bool DArray of d's dims: K25 ---------------------------------------------------------------------------------------


def setindex_mask(d: DArray, m: DArray, v):
    """``d[m] = v``: the selected elements of ``d``, in column-major order, take ``v``'s elements in order (``v`` a vector of
    ``count(m)`` elements) or the scalar ``v``."""
    from ._broadcast import copy
    from ._compact import _check, plan
    from ._sparse import SparseDArray, refuse
    from ._take import _source_table
    if isinstance(v, SparseDArray):
        refuse("setindex!")
    _check(d, m)
    rt = d.rt
    scalar = _is_scalar(v)
    if not scalar:
        vs = np.shape(v) if not isinstance(v, (DArray, SubDArray)) else tuple(v.dims)
        if len(_squeeze(vs)) > 1:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"a logical index takes a vector of values, not an array of size {tuple(vs)}")
    if d.size == 0:
        return
    owned: List[DArray] = []
    temps: List[B200Array] = []
    try:
        if m is d:
            m = copy(m)                                       # Base.unalias: the mask is read while d is written
            owned.append(m)
        if scalar:
            sv = _scalar_bytes(d, v)
            same = m.layout.same_as(d.layout)
            fenced = open_remote_reads(rt, [] if same else [m], "device")
            for c, pid in enumerate(d.layout.pids):
                ch = d.chunks.get(pid)
                if ch is None or not ch.size:
                    continue
                if same:
                    blk = m.chunks[pid]
                else:
                    blk = B200Array.empty(rt, ch.shape, np.bool_, temp=True)
                    temps.append(blk)
                    SubDArray(m, d.layout.indices[c], tuple(False for _ in ch.shape)).copy_to(blk)
                _lib.call("dab_expand", rt.ctx, d.dtype.itemsize, C.c_void_p(blk.ptr), C.c_void_p(ch.ptr), ch.size, 1, None, None, 0, None, None,
                          C.c_void_p(sv.ctypes.data))
            close_remote_reads(rt, fenced, "device")
            return
        runs, work, plans, offsets = plan(d, m, temps)
        count = int(offsets[-1])
        vs = np.shape(v) if not isinstance(v, (DArray, SubDArray)) else tuple(v.dims)
        if int(np.prod(vs, dtype=np.int64)) != count:
            _mismatch("an array", vs, (count,))
        if count == 0:
            return
        if isinstance(v, (DArray, SubDArray)):
            w = _value_darray(v, d, (count,), owned)
            fenced = open_remote_reads(rt, [w], "device")
            _, grid, cuts, ptrs = _source_table(w)
        else:                                                 # every rank holds the host vector: one local chunk
            blk = B200Array.empty(rt, (count,), d.dtype, temp=True)
            temps.append(blk)
            blk.copy_from_host(np.asarray(v).astype(d.dtype, copy=False).reshape(count, order="F"))
            fenced = False
            grid, cuts, ptrs = (C.c_int32 * 1)(1), (C.c_size_t * 2)(0, count), (C.c_void_p * 1)(blk.ptr)
        for c, pid in work:
            run_len, ids, lin = runs[c]
            mblk, incl, _ = plans[c]
            info = B200Array.empty(rt, (2 * ids.size,), np.int64, temp=True)
            temps.append(info)
            info.copy_from_host(np.stack([offsets[ids], lin]).reshape(-1, order="F"))
            _lib.call("dab_expand", rt.ctx, d.dtype.itemsize, C.c_void_p(mblk.ptr), C.c_void_p(d.chunks[pid].ptr), run_len, ids.size,
                      C.c_void_p(incl.ptr), C.c_void_p(info.ptr), grid[0], cuts, ptrs, None)
        close_remote_reads(rt, fenced, "device")              # the owners of v keep it until every rank has read it
    finally:
        for t in temps:
            t.free()                                          # stream-ordered
        for a in owned:
            a.close()


# ---- host keys: views -----------------------------------------------------------------------------------------------------------------


def _last_occurrences(v: np.ndarray) -> np.ndarray:
    """0-based positions of the last occurrence of every value of ``v``, in increasing order."""
    _, first_rev = np.unique(v[::-1], return_index=True)
    return np.sort(v.size - 1 - first_rev)


def _axis(off: np.ndarray, rt, tables: List[B200Array]):
    """(base, stride, device table or None) for the element offsets ``off`` along one dim (``dab_gather_box``'s per-dim form)."""
    base = int(off[0])
    off = off - base
    step = int(off[1]) if off.size > 1 else 0
    if off.size <= 1 or np.array_equal(off, step * np.arange(off.size, dtype=np.int64)):
        return base, step, None
    t = B200Array.from_numpy(rt, np.ascontiguousarray(off, dtype=np.int64))
    tables.append(t)
    return base, 0, t.ptr


def setindex_view(S: SubDArray, v):
    """``view[:] = v`` for a view of host keys: per chunk of the parent that the view meets, its owner writes the sub-box with
    ``dab_gather_box`` from the value piece -- a scalar (stride 0), an uploaded slice of a host array, or a halo read of a DArray value.
    A repeated host index keeps the value of its last occurrence."""
    from ._sparse import SparseDArray, refuse
    if isinstance(v, SparseDArray):
        refuse("setindex!")
    d = S.parent
    rt = d.rt
    N = d.ndim
    if N > 8:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "views of arrays with more than 8 dimensions are not served")
    full = S.full_shape
    scalar = _is_scalar(v)
    if not scalar:
        vs = np.shape(v) if not isinstance(v, (DArray, SubDArray)) else tuple(v.dims)
        if _squeeze(vs) != _squeeze(S.shape):
            _mismatch("an array", vs, S.shape)
    if int(np.prod(full, dtype=np.int64)) == 0:
        return
    iv = S.index_vectors()
    keep = [np.arange(x.size, dtype=np.int64) if ix is None else _last_occurrences(x) for x, ix in zip(iv, S.idx)]
    owned: List[DArray] = []
    tables: List[B200Array] = []
    es = d.dtype.itemsize
    try:
        host = w = None
        if scalar:
            one = B200Array.from_numpy(rt, _scalar_bytes(d, v))
            tables.append(one)
        elif isinstance(v, (DArray, SubDArray)):
            w = _value_darray(v, d, full, owned)
        else:
            host = np.asarray(v).astype(d.dtype, copy=False).reshape(full, order="F")
        fenced = open_remote_reads(rt, [w] if w is not None else [], "device")
        for c, Kc in enumerate(d.layout.indices):
            pid = d.layout.pids[c]
            if pid not in d.chunks:
                continue
            sel = [p[(x[p] >= k[0]) & (x[p] <= k[1])] for x, p, k in zip(iv, keep, Kc)]
            if any(s.size == 0 for s in sel):
                continue
            ext = [int(s.size) for s in sel]
            sstr = np.cumprod([1] + list(shape_of(Kc)[:-1])).astype(np.int64)
            dbase, ds, di = 0, [], []
            for k in range(N):
                b, st, tab = _axis((iv[k][sel[k]] - Kc[k][0]) * sstr[k], rt, tables)
                dbase += b
                ds.append(st)
                di.append(tab)
            if scalar:
                src, ss = one.ptr, [0] * N
            else:
                piece = B200Array.empty(rt, ext, d.dtype, temp=True)
                tables.append(piece)
                if host is not None:
                    piece.copy_from_host(host[np.ix_(*sel)])
                else:
                    J = tuple((int(s.min()) + 1, int(s.max()) + 1) for s in sel)
                    SubDArray(w, J, tuple(False for _ in J), tuple(s + 1 for s in sel)).copy_to(piece)
                src, ss = piece.ptr, [int(x) for x in np.cumprod([1] + ext[:-1])]
            LL, VP = C.c_longlong * N, C.c_void_p * N
            _lib.call("dab_gather_box", rt.ctx, es, N, C.c_void_p(d.chunks[pid].ptr + dbase * es), LL(*ds), VP(*di), C.c_void_p(src), LL(*ss),
                      None, (C.c_size_t * N)(*ext))
        close_remote_reads(rt, fenced, "device")
    finally:
        for t in tables:
            t.free()                                          # stream-ordered
        for a in owned:
            a.close()


def copyto_view(dest: SubDArray, src):
    """``copyto!(view, src)``: ``src`` of the view's size, written as ``view[:] = src``."""
    if tuple(np.shape(src) if not isinstance(src, (DArray, SubDArray)) else src.dims) != tuple(dest.shape):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"the view has size {tuple(dest.shape)} but the source has "
                                     f"{tuple(np.shape(src) if not isinstance(src, (DArray, SubDArray)) else src.dims)}")
    setindex_view(dest, src)
    return dest


def setindex(d: DArray, key, v):
    """``DArray.__setitem__``: dispatch on the key as ``__getitem__`` does."""
    from ._darray import refuse_float16
    from ._sparse import SparseDArray
    if isinstance(key, (DArray, SparseDArray)):
        refuse_float16("d[key] = v with a DArray key (the scatter and expansion have no 2-byte instances)", d)
    if isinstance(key, DArray) and key.dtype == np.bool_ and key.dims == d.dims:
        return setindex_mask(d, key, v)
    if isinstance(key, (DArray, SparseDArray)):
        return setindex_take(d, key, v)
    return setindex_view(d._view(key), v)
