"""Scans of DArrays: ``cumsum`` / ``cumprod`` / ``accumulate`` and their ``!`` forms (Julia ``base/accumulate.jl``) on the GPU.

The reference has none: Base's generic ``accumulate!`` writes ``similar(A)`` element by element, which ends in ``setindex!`` on a DArray.
Here every chunk is scanned by ONE ``dab_scan`` launch (include/dab200.h, K17).  When ``dims`` is split across workers, chunk ``g`` along
``dims`` starts from the carry ``init (op) total_0 (op) ... (op) total_(g-1)``: every earlier chunk reduces itself to a slab of carriers
(``dab_scan_totals``), the slabs travel to the later chunks like the partial slabs of ``mapreducedim_between!``
(``_mapreduce.gather_fibres``), and each consumer folds its stack of slabs in grid order with one small ``dab_scan`` along the stack.
The plan of who sends which total to whom is a pure function of the layout (``carry_plan``), so every rank derives the same.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional

import numpy as np

from . import _lib
from ._darray import DArray, SubDArray, B200Array, copyto, dab_dtype, is_complex, makelocal, similar
from ._mapreduce import _op_code, gather_fibres
from .layout import Layout, ravel, shape_of, unravel
from .runtime import close_remote_reads, open_remote_reads

_UNDEF_DIMS = "UndefKeywordError: keyword argument `dims` not assigned"


def result_dtype(dtype, opc: int, widen: bool) -> np.dtype:
    """Element type of the scan's result: ``cumsum`` / ``cumprod`` (``widen``) use ``add_sum`` / ``mul_prod``, which take small integers
    and Bool to Int64 (except ``cumprod`` of Bool: ``&``); ``accumulate(op)`` uses ``promote_op(op, T, T)``: Int32 stays Int32, Bool + Bool
    is Int64.  Complex, UInt8 and Int128 arrays are not served."""
    dt = np.dtype(dtype)
    if is_complex(dt):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"scans of {dt} arrays are not served (no host fallback)")
    if dt in (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int64)):
        return dt
    if dt == np.dtype(np.int32):
        return np.dtype(np.int64) if widen and opc in (_lib.SUM, _lib.PROD) else dt
    if dt == np.dtype(np.bool_):
        return np.dtype(np.int64) if opc == _lib.SUM else dt
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"scans of {dt} arrays are not served (no host fallback)")


def _code(dt: np.dtype) -> int:
    return _lib.I64 if dt == np.dtype(np.int64) else dab_dtype(dt)


def carrier_dtype(in_dt: np.dtype, opc: int, out_dt: np.dtype) -> np.dtype:
    out = C.c_int32()
    _lib.check(_lib.lib().dab_scan_carrier_dtype(_code(in_dt), opc, _code(out_dt), C.byref(out)))
    return {_lib.F64: np.dtype(np.float64), _lib.I64: np.dtype(np.int64)}.get(out.value, in_dt)


def _init_value(init, R: np.dtype):
    """``init`` as a value of the result type R, when R holds it exactly (the first output is ``op(init, x1)`` in R)."""
    v = np.asarray(init)
    x = v.item() if v.ndim == 0 and v.dtype.kind in "biuf" else None
    if isinstance(x, bool):
        x = int(x)
    ok = False
    if x is not None:
        if R.kind == "f":
            ok = (isinstance(x, float) and math.isnan(x)) or (float(R.type(x)) == x if isinstance(x, float) else
                                                              math.isfinite(float(R.type(x))) and int(R.type(x)) == x)
        elif R == np.dtype(np.bool_):
            ok = x in (0, 1)
        else:
            info = np.iinfo(R)
            ok = float(x).is_integer() and info.min <= x <= info.max
    if not ok:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"init={init!r} is not exactly representable in the result type {R}; not served")
    return int(x) if R.kind in "iub" else x


def carry_plan(L: Layout, dims: int) -> List[List[int]]:
    """For every chunk (0-based number in ``L``), the chunks before it along ``dims``, in grid order: the members whose totals make up its
    carry.  Pure function of the layout; ``_mapreduce.exchange_plan(L, L, carry_plan(L, dims), ...)`` is then who sends what to whom."""
    k = dims - 1
    out = []
    for rl in range(len(L.pids)):
        c = list(unravel(rl, L.grid))
        out.append([ravel(c[:k] + [j] + c[k + 1:], L.grid) for j in range(c[k])])
    return out


def _shape3(shape, k: int):
    return int(np.prod(shape[:k], dtype=np.int64)), int(shape[k]), int(np.prod(shape[k + 1:], dtype=np.int64))


def _check_dims(dims, ndim: int, cum: bool):
    if dims is None:
        if ndim != 1:
            if cum:
                raise TypeError(_UNDEF_DIMS)
            raise _lib.ArgumentError(_lib.ERR_ARG, "ArgumentError: Keyword argument dims must be provided for multidimensional arrays")
        return 1
    dims = int(dims)
    if dims <= 0:
        raise _lib.ArgumentError(_lib.ERR_ARG, "ArgumentError: dims must be a positive integer")
    return dims


def _scan_into(op, dest: DArray, src, dims, init, cum: bool) -> DArray:
    """``accumulate!(op, dest, src; dims, init)`` (base/accumulate.jl ``_accumulate!``)."""
    opc = _op_code(op)
    if isinstance(src, SubDArray):
        tmp = src.to_darray()
        try:
            return _scan_into(op, dest, tmp, dims, init, cum)
        finally:
            tmp.close()
    dims = _check_dims(dims, src.ndim, cum)
    if tuple(dest.dims) != tuple(src.dims):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "DimensionMismatch: shape of B must match A")
    R = result_dtype(src.dtype, opc, cum)
    if dims > src.ndim:
        return copyto(dest, src)                      # Julia: copyto!(B, A) -- init is not applied
    if dest.dtype != R:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"a {dest.dtype} destination for the {R} result of this scan is not served")
    ival = None if init is None else _init_value(init, R)
    if src.size == 0:
        return dest
    _run(opc, dest, src, dims, R, ival)
    return dest


def _run(opc: int, dest: DArray, src: DArray, dims: int, R: np.dtype, ival):
    rt, L, k = dest.rt, dest.layout, dims - 1
    cdt = carrier_dtype(src.dtype, opc, R)
    ccode, icode, ocode, isz = _code(cdt), _code(src.dtype), _code(R), cdt.itemsize
    same = src.layout.same_as(L)
    fenced = False if same else open_remote_reads(rt, [src], "device")
    temps: List[B200Array] = []
    stack_temp = 0                                     # the private stack buffer when the exchange arena is not used
    try:
        inputs = {}
        for pid, out in dest.chunks.items():
            if same:
                inputs[pid] = src.chunks[pid]
            elif out.size == 0:
                inputs[pid] = out                      # never read
            else:                                      # another layout: the existing halo fetch into a dense temporary
                inputs[pid] = makelocal(src, L.localindices(pid), pid)
                if inputs[pid] is not src.chunks.get(pid):
                    temps.append(inputs[pid])
        shapes = [shape_of(ix) for ix in L.indices]
        plens = [int(np.prod(s[:k] + s[k + 1:], dtype=np.int64)) for s in shapes]
        fibres = carry_plan(L, dims) if L.grid[k] > 1 else [[] for _ in L.pids]
        if L.grid[k] > 1:
            # chunk totals of every chunk with a successor along dims, then the totals travel to the chunks after it
            G = L.grid[k]
            totals = {}
            for pid, x in inputs.items():
                rl = L.pids.index(pid)
                if unravel(rl, L.grid)[k] < G - 1 and plens[rl]:
                    t = B200Array.empty(rt, (plens[rl],), cdt, temp=True)
                    temps.append(t)
                    _lib.call("dab_scan_totals", rt.ctx, icode, opc, ocode, C.c_void_p(x.ptr), *_shape3(shapes[rl], k), C.c_void_p(t.ptr))
                    totals[pid] = t
            st, stacks = gather_fibres(rt, L, L, fibres, [(plen * isz,) for plen in plens], {pid: (t.ptr,) for pid, t in totals.items()})
            stack_temp = st.temp
        for pid, out in dest.chunks.items():
            rl = L.pids.index(pid)
            if out.size == 0:
                continue
            carry = None
            if ival is not None:
                slab = B200Array.empty(rt, (plens[rl],), cdt, temp=True)
                temps.append(slab)
                v = np.asarray(ival, dtype=cdt)
                _lib.call("dab_fill", rt.ctx, ccode, C.c_void_p(slab.ptr), slab.size, C.c_void_p(v.ctypes.data))
                carry = slab.ptr
            g = len(fibres[rl])
            if g:
                # fold the stack of totals in grid order, seeded with init: one small scan along the stack, its last row is the carry
                base = stacks[rl][0]
                _lib.call("dab_scan", rt.ctx, ccode, opc, ccode, C.c_void_p(base), plens[rl], g, 1, C.c_void_p(carry) if carry else None,
                          C.c_void_p(base))
                carry = base + (g - 1) * plens[rl] * isz
            _lib.call("dab_scan", rt.ctx, icode, opc, ocode, C.c_void_p(inputs[pid].ptr), *_shape3(out.shape, k),
                      C.c_void_p(carry) if carry else None, C.c_void_p(out.ptr))
    finally:
        rt.free_temp(stack_temp)                       # stream-ordered: after the scans that read the stacks
        for t in temps:
            t.free()
        close_remote_reads(rt, fenced, "device")


def _scan_alloc(op, d, dims, init, cum: bool) -> DArray:
    """``accumulate(op, A; dims, init)``: the result is ``similar(A, R)`` -- the default layout over ``procs(A)`` -- filled by
    ``accumulate!``."""
    opc = _op_code(op)
    if isinstance(d, SubDArray):
        tmp = d.to_darray()
        try:
            return _scan_alloc(op, tmp, dims, init, cum)
        finally:
            tmp.close()
    if dims is None and d.ndim != 1:
        if cum:
            raise TypeError(_UNDEF_DIMS)
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "accumulate(op, A) of a multidimensional array without dims (Julia's linear "
                                    "column-major scan) is not served")
    dims = _check_dims(dims, d.ndim, cum)
    R = result_dtype(d.dtype, opc, cum)
    if init is not None and dims <= d.ndim:
        _init_value(init, R)
    out = similar(d, R)
    try:
        return _scan_into(op, out, d, dims, init, cum)
    except BaseException:
        out.close()
        raise


def cumsum(d, dims=None) -> DArray:
    """``cumsum(A; dims)`` (``dims`` may be omitted for a vector): ``accumulate(add_sum, A; dims)``."""
    return _scan_alloc("+", d, dims, None, True)


def cumprod(d, dims=None) -> DArray:
    """``cumprod(A; dims)``: ``accumulate(mul_prod, A; dims)``."""
    return _scan_alloc("*", d, dims, None, True)


def accumulate(op, d, dims=None, init=None) -> DArray:
    """``accumulate(op, A; dims, init)`` for op in ``+ * max min`` (the ``reduce`` vocabulary)."""
    return _scan_alloc(op, d, dims, init, False)


def cumsum_(dest: DArray, src, dims=None) -> DArray:
    """``cumsum!(B, A; dims)``."""
    return _scan_into("+", dest, src, dims, None, True)


def cumprod_(dest: DArray, src, dims=None) -> DArray:
    """``cumprod!(B, A; dims)``."""
    return _scan_into("*", dest, src, dims, None, True)


def accumulate_(op, dest: DArray, src, dims=None, init=None) -> DArray:
    """``accumulate!(op, B, A; dims, init)``."""
    return _scan_into(op, dest, src, dims, init, False)
