"""``ppeval(f, D...; dim)`` (reference src/mapreduce.jl:210-323) on H100.

The reference runs ``_ppeval(f, map(localpart, D)...; dim)`` on every worker of ``procs(D[1])``: the localparts are sliced along
``dim[i]`` (an entry <= 0 passes that argument whole), ``f`` is applied to the i-th slices of all sliced arguments together, and the
results are stacked along a new last dimension, so a worker's chunk is ``(size(f(slices...))..., nlocal)``.  The chunks become
``DArray(reshape(refs, (sd[1:nd-1]..., sd[end])))`` with ``sd = size(procs(D[1]))`` and ``nd`` the chunks' ``ndims``.  Before that, every
dimension of a DArray argument other than its ``dim`` has to be whole on every worker: there is no redistribution.

``f`` is recognised by calling it once, on the host, with a slice tracer for each sliced argument and the broadcast arguments as they
are.  The served forms:

  f(slices...)                                   per chunk
  ---------------------------------------------  ------------------------------------------------------------------------------------
  ``a @ b`` (Julia's ``*``: ``operator.matmul``,  ``dab_matmul_batched``; a matrix slice times a vector or matrix slice, either operand
  a lambda using ``@``, ``dab.matmul``)           possibly a host array that is broadcast (uploaded once, batch stride 0)
  ``ldiv(a, b)`` (Julia's ``a \\ b``)             ``dab_ldiv_batched`` (K27); a square matrix slice and a vector or matrix slice, either
                                                 possibly a broadcast host array; Int32 / Int64 operands are converted to Float64 first
  one sliced argument, any ``mapslices`` slice   the ``mapslices`` chunk code over all dimensions but ``dim`` (``eigvals`` of a square
  function (``eigvals``, ``sort``, ``svdvals``,  slice: ``dab_eigvals_sym_batched``); when ``dim`` is not last, one ``dab_gather_box``
  reductions, elementwise maps, constants)       first moves it last

Python's ``*`` is Julia's ``.*`` in this package, so the reference's ``ppeval(*, A, B)`` is written ``ppeval(operator.matmul, A, B)``.
Anything else raises ``UnsupportedError``; so does a DArray passed with ``dim <= 0`` (the reference would hand ``f`` each worker's
localpart) and a worker that holds no slices.  Every check, the kernels' limits and the result layout included, happens before the first
launch.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import _lib
from ._broadcast import SLICE_TRACING, Expr, tag_of
from ._darray import B200Array, DArray, SubDArray, dab_dtype
from ._broadcast import LocalArg, convert, run_local
from ._slices import SliceLdiv, SliceMatmul, _dense_strides, _gather, _is_slice, check_limits, plan_of, raise_on_status, run_chunk
from .layout import Layout, layout_from_chunk_shapes, ravel, rlen, unravel

_MATMUL_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int32), np.dtype(np.int64))


def _normalise_dim(dim, D) -> Tuple[int, ...]:
    if dim is None:
        return tuple(x.ndim if isinstance(x, DArray) else 0 for x in D)
    if isinstance(dim, (int, np.integer)) and not isinstance(dim, (bool, np.bool_)):
        dim = (dim,)
    if not isinstance(dim, (tuple, list)) or any(isinstance(d, (bool, np.bool_)) or not isinstance(d, (int, np.integer)) for d in dim):
        raise _lib.ArgumentError(_lib.ERR_ARG, f"ppeval: dim must be a tuple of integers, got {dim!r}")
    dim = tuple(int(d) for d in dim)
    if len(dim) != len(D):
        raise _lib.ArgumentError(_lib.ERR_ARG, f"ArgumentError: dim argument has wrong length. length(dim) = {len(dim)} but should be {len(D)}")
    return dim


def result_grid(sd: Sequence[int], nd: int, nprocs: int) -> Tuple[int, ...]:
    """``(sd[1:nd-1]..., sd[end])`` (src/mapreduce.jl:320-322), raising where the reference's reshape would throw."""
    if nd - 1 > len(sd):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"ppeval: results of {nd} dimensions cannot be laid out on a procs grid of "
                                     f"{len(sd)} dimensions")
    grid = tuple(int(g) for g in sd[:nd - 1]) + (int(sd[-1]),)
    if int(np.prod(grid)) != nprocs:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"ppeval: the {nprocs} result chunks do not fill the grid {grid}")
    return grid


def check_tiling(shapes: Sequence[Sequence[int]], grid: Sequence[int]) -> None:
    """``DArray(refs)`` needs the chunks along each grid axis to agree on their extent across the other axes."""
    for lin, s in enumerate(shapes):
        c = unravel(lin, grid)
        for x in range(len(grid)):
            first = [0] * len(grid)
            first[x] = c[x]
            if int(s[x]) != int(shapes[ravel(first, grid)][x]):
                raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"ppeval: result chunks of shapes {[tuple(t) for t in shapes]} do not "
                                             f"tile the grid {tuple(grid)}")


class _MatmulPlan:
    """``a @ b`` of slices: each operand ``("slice", argument index)`` or ``("host", array)``."""

    def __init__(self, ops, m: int, k: int, n: int, vec: bool, dtype: np.dtype):
        self.ops, self.m, self.k, self.n, self.vec, self.dtype = ops, m, k, n, vec, dtype

    def rshape(self) -> Tuple[int, ...]:
        return (self.m,) if self.vec else (self.m, self.n)


def _operands(r, slice_shapes: Dict[int, Tuple[int, ...]], dtypes: Dict[int, np.dtype], what: str):
    """The two operands of ``a @ b`` / ``a \\ b``: ``("slice", argument index)`` or ``("host", array)``, with their shapes and eltypes."""
    ops, shapes, dts = [], [], []
    for x in (r.a, r.b):
        if isinstance(x, Expr):
            if not _is_slice(x) or x.val not in slice_shapes:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a {what} of an expression of a slice is not served "
                                            "(pass the slices themselves)")
            ops.append(("slice", x.val))
            shapes.append(slice_shapes[x.val])
            dts.append(dtypes[x.val])
        elif isinstance(x, (DArray, SubDArray)):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "ppeval: a DArray inside f is not served; pass it as an argument")
        else:
            a = np.asarray(x)
            if a.dtype == object or a.ndim == 0:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a {what} with a {type(x).__name__} is not served")
            ops.append(("host", np.asfortranarray(a)))
            shapes.append(a.shape)
            dts.append(a.dtype)
    return ops, shapes, dts


def _matmul_plan(r: SliceMatmul, slice_shapes: Dict[int, Tuple[int, ...]], dtypes: Dict[int, np.dtype]) -> _MatmulPlan:
    ops, (sa, sb), (ta, tb) = _operands(r, slice_shapes, dtypes, "matrix product")
    if len(sa) != 2:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a * b with a of {len(sa)} dimensions; served: a matrix times a vector "
                                    "or a matrix")
    if len(sb) not in (1, 2):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a * b with b of {len(sb)} dimensions; served: a vector or a matrix")
    if ta != tb or ta not in _MATMUL_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a * b of eltypes {ta} and {tb} (served: equal Float32 Float64 Int32 "
                                    "Int64)")
    m, k = int(sa[0]), int(sa[1])
    if int(sb[0]) != k:
        if len(sb) == 1:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"second dimension of A, {k}, does not match length of x, {sb[0]}")
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"matrix A has dimensions ({m},{k}), matrix B has dimensions ({sb[0]},{sb[1]})")
    return _MatmulPlan(ops, m, k, 1 if len(sb) == 1 else int(sb[1]), len(sb) == 1, ta)


class _LdivPlan:
    """``a \\ b`` of slices: each operand as in ``_MatmulPlan``; ``dtype`` is the working and result eltype (Float64 for integers)."""

    def __init__(self, ops, n: int, nrhs: int, vec: bool, dtype: np.dtype):
        self.ops, self.n, self.nrhs, self.vec, self.dtype = ops, n, nrhs, vec, dtype

    def rshape(self) -> Tuple[int, ...]:
        return (self.n,) if self.vec else (self.n, self.nrhs)


def _ldiv_plan(r: SliceLdiv, slice_shapes: Dict[int, Tuple[int, ...]], dtypes: Dict[int, np.dtype]) -> _LdivPlan:
    ops, (sa, sb), (ta, tb) = _operands(r, slice_shapes, dtypes, "left division")
    if len(sa) != 2:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a \\ b with a of {len(sa)} dimensions; served: a square matrix")
    if len(sb) not in (1, 2):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a \\ b with b of {len(sb)} dimensions; served: a vector or a matrix")
    if ta != tb or ta not in _MATMUL_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a \\ b of eltypes {ta} and {tb} (served: equal Float32 Float64 Int32 "
                                    "Int64)")
    m, n = int(sa[0]), int(sa[1])
    if m != n:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a \\ b with a of {m}x{n}: the least-squares solution of a non-square "
                                    "system (Julia's pivoted QR) is not served")
    if n > _lib.LU_MAX_N:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: a \\ b with a of {n}x{n}; served: n <= {_lib.LU_MAX_N}")
    if int(sb[0]) != n:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"B has leading dimension {sb[0]}, but needs {n}")
    wdt = ta if ta.kind == "f" else np.dtype(np.float64)           # lutype(Int) = Float64
    ops = [(kind, np.asfortranarray(v, dtype=wdt)) if kind == "host" else (kind, v) for kind, v in ops]
    return _LdivPlan(ops, n, 1 if len(sb) == 1 else int(sb[1]), len(sb) == 1, wdt)


def _first_failure(st: np.ndarray, slots, order) -> Tuple[int, ...]:
    """This rank's first failing ``ldiv`` slice from the status words of ``slots``: ``(order(slot, b)..., info)``, or None."""
    best = None
    for slot in slots:
        w = int(st[slot]) & _lib.LU_STATUS_CLEAR
        if w == _lib.LU_STATUS_CLEAR:
            continue
        low = w & 0xFF
        cand = order(slot, w >> 8) + (0 if low == _lib.LU_STATUS_NONFINITE else low,)
        best = cand if best is None or cand < best else best
    return best


def _trace(f, D):
    args = []
    for i, x in enumerate(D):
        args.append(Expr("arg", (), tag_of(x.dtype), i) if isinstance(x, DArray) else x)
    SLICE_TRACING[0] += 1
    try:
        return f(*args)
    except _lib.DabError:
        raise
    except Exception as e:  # noqa: BLE001 - anything f does with the tracers that is not a served form
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: {getattr(f, '__name__', f)!r} is not a served slice function "
                                    f"({type(e).__name__}: {e}); served: a * b (operator.matmul), ldiv, det, eigvals, and for one sliced argument "
                                    "every mapslices slice function") from None
    finally:
        SLICE_TRACING[0] -= 1


def _slices_last(rt, ch: B200Array, d: int, temps: List[B200Array]) -> B200Array:
    """The chunk with its sliced dimension ``d`` moved last (one ``dab_gather_box``), or the chunk itself when it is last already."""
    N = len(ch.shape)
    if d == N:
        return ch
    perm = [j for j in range(N) if j != d - 1] + [d - 1]
    pshape = [ch.shape[j] for j in perm]
    P = B200Array.empty(rt, pshape, ch.dtype, temp=True)
    temps.append(P)
    cstr = _dense_strides(ch.shape)
    _gather(rt, ch.dtype.itemsize, P.ptr, _dense_strides(pshape), ch.ptr, [cstr[j] for j in perm], pshape)
    return P


def ppeval(f, *D, dim=None) -> DArray:
    """``ppeval(f, D...; dim)`` (reference src/mapreduce.jl:300-323).  See the module docstring for the served ``f``."""
    from ._sparse import SparseDArray, refuse
    if any(isinstance(a, SparseDArray) for a in D):
        refuse("ppeval")
    dim = _normalise_dim(dim, D)
    if not D or not isinstance(D[0], DArray):
        raise _lib.ArgumentError(_lib.ERR_ARG, "ppeval: the first argument must be a DArray (its procs are the workers)")
    sliced = []
    for i, x in enumerate(D):
        if isinstance(x, SubDArray):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "ppeval of a view: make it a DArray first (DArray(view))")
        if (x.dtype if isinstance(x, DArray) else np.asarray(x).dtype) == np.dtype(np.float16):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval with a Float16 argument ({i + 1}) is not served (no Float16 slice kernels)")
        if (x.dtype if isinstance(x, DArray) else np.asarray(x).dtype).kind == "c":
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval with a complex argument ({i + 1}) is not served (no complex slice kernels)")
        if isinstance(x, DArray):
            if dim[i] <= 0:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: DArray argument {i + 1} with dim {dim[i]} <= 0 is not served "
                                            "(each worker would receive its own localpart); slice it or pass a host array")
            if dim[i] > x.ndim:
                raise _lib.ArgumentError(_lib.ERR_ARG, f"ppeval: dim {dim[i]} of argument {i + 1} is not a dimension of a {x.ndim}-dimensional "
                                         "DArray")
            if x.ndim > 8:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "ppeval over more than 8 dimensions is not served")
            sliced.append(i)
        elif dim[i] > 0:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: slicing host argument {i + 1} is not served; pass it with dim 0 to "
                                        "broadcast it")
    # ---- every dimension but dim is whole on every worker (src/mapreduce.jl:301-313)
    for i in sliced:
        x = D[i]
        for idxs in x.layout.indices:
            for d in range(1, x.ndim + 1):
                if d != dim[i] and rlen(idxs[d - 1]) != x.dims[d - 1]:
                    raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"dimension {d} is distributed. ppeval requires dimension {d} to be "
                                                 "completely available on all processors.")
    # ---- slices per worker, paired worker by worker as _ppeval pairs the localparts (:215-220)
    D1 = D[0]
    L1: Layout = D1.layout
    pids = list(L1.pids)
    nlocal = {}
    for pid in pids:
        counts = [rlen(D[i].layout.localindices(pid)[dim[i] - 1]) for i in sliced]
        for j, i in enumerate(sliced[1:], 1):
            if counts[j] != counts[0]:
                raise _lib.ArgumentError(_lib.ERR_ARG, f"ArgumentError: lengths of broadcast dimensions must be the same. size(A[1], {dim[0]}) = "
                                         f"{counts[0]} but size(A[{i + 1}], {dim[i]}) = {counts[j]}")
        if counts[0] == 0:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: worker {pid} holds no slices of the first argument (not served)")
        nlocal[pid] = counts[0]
    # ---- what f is
    slice_shapes = {i: tuple(s for d, s in enumerate(D[i].dims, 1) if d != dim[i]) for i in sliced}
    dtypes = {i: D[i].dtype for i in sliced}
    r = _trace(f, D)
    if isinstance(r, SliceMatmul):
        plan = _matmul_plan(r, slice_shapes, dtypes)
        rshape, rdtype = plan.rshape(), plan.dtype
    elif isinstance(r, SliceLdiv):
        plan = _ldiv_plan(r, slice_shapes, dtypes)
        rshape, rdtype = plan.rshape(), plan.dtype
    elif len(sliced) == 1:
        i0 = sliced[0]
        sdims = tuple(range(1, len(slice_shapes[i0]) + 1))
        plan = plan_of(r, sdims, dtypes[i0], what="ppeval")
        pshape0 = slice_shapes[i0] + (1,)
        check_limits(plan, [pshape0], what="ppeval")
        rshape, rdtype = plan.rshape(pshape0), plan.dtype
    else:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"ppeval: f of {len(sliced)} sliced DArrays is served for a * b (operator.matmul) "
                                    "and ldiv only")
    # ---- the result layout: DArray(reshape(refs, (sd[1:nd-1]..., sd[end]))) (:320-322)
    out_shapes = [tuple(rshape) + (nlocal[pid],) for pid in pids]
    grid = result_grid(L1.grid, len(rshape) + 1, len(pids))
    check_tiling(out_shapes, grid)
    layout = layout_from_chunk_shapes(out_shapes, grid, pids)
    # ---- launches
    rt = D1.rt
    temps: List[B200Array] = []
    chunks: Dict[int, B200Array] = {}
    status = cdev = None
    try:
        if isinstance(plan, (_MatmulPlan, _LdivPlan)):
            host = {}
            for kind, v in plan.ops:
                if kind == "host" and id(v) not in host:
                    host[id(v)] = B200Array.from_numpy(rt, v)
                    temps.append(host[id(v)])
        if isinstance(plan, _LdivPlan):
            status = B200Array.empty(rt, (max(1, len(D1.chunks)),), np.int64, temp=True)
        elif isinstance(plan, _MatmulPlan):
            pass
        elif plan.kind in ("svdvals", "eigvals"):
            status = B200Array.empty(rt, (max(1, len(D1.chunks)),), np.int32, temp=True)
        elif plan.kind == "const" and plan.const.size:
            cdev = B200Array.from_numpy(rt, plan.const)
            temps.append(cdev)
        ran = []
        for slot, (pid, ch1) in enumerate(D1.chunks.items()):
            out = B200Array.empty(rt, out_shapes[pids.index(pid)], rdtype)
            chunks[pid] = out
            if out.size == 0 and not (isinstance(plan, _LdivPlan) and plan.n):     # an empty b still factors A (lu checks it)
                continue
            nb = nlocal[pid]
            if isinstance(plan, _MatmulPlan):
                ptrs = []
                for kind, v in plan.ops:
                    if kind == "host":
                        ptrs.append((host[id(v)].ptr, 0))
                    else:
                        P = _slices_last(rt, D[v].chunks[pid], dim[v], temps)
                        ptrs.append((P.ptr, P.size // nb))
                (pa, sa), (pb, sb) = ptrs
                _lib.call("dab_matmul_batched", rt.ctx, dab_dtype(plan.dtype), plan.m, plan.n, plan.k, C.c_void_p(pa), sa, C.c_void_p(pb), sb,
                          C.c_void_p(out.ptr), nb)
            elif isinstance(plan, _LdivPlan):
                ptrs = []
                for kind, v in plan.ops:
                    if kind == "host":
                        ptrs.append((host[id(v)].ptr, 0))
                        continue
                    P = _slices_last(rt, D[v].chunks[pid], dim[v], temps)
                    if P.dtype != plan.dtype:                      # lu of an integer matrix works in Float64
                        W = B200Array.empty(rt, P.shape, plan.dtype, temp=True)
                        temps.append(W)
                        run_local(rt, convert(Expr("arg", (), tag_of(P.dtype), 0), tag_of(plan.dtype)), W, [LocalArg(P, None, tag_of(P.dtype))])
                        P = W
                    ptrs.append((P.ptr, P.size // nb))
                (pa, sa), (pb, sb) = ptrs
                _lib.call("dab_ldiv_batched", rt.ctx, dab_dtype(plan.dtype), plan.n, plan.nrhs, C.c_void_p(pa), sa, C.c_void_p(pb), sb,
                          C.c_void_p(out.ptr), nb, C.c_void_p(status.ptr + 8 * slot))
                ran.append(slot)
            elif plan.kind == "const":
                c = plan.const
                _gather(rt, c.dtype.itemsize, out.ptr, _dense_strides(out.shape), cdev.ptr, _dense_strides(c.shape) + [0], out.shape)
            else:
                i0 = sliced[0]
                P = _slices_last(rt, ch1, dim[i0], temps)
                view = B200Array(rt, out.ptr, plan.out_shape(P.shape), rdtype, own=False)
                run_chunk(rt, plan, P, view, status.ptr + 4 * slot if status is not None else 0, None, temps)
                ran.append(slot)
        if isinstance(plan, _LdivPlan):
            # slices in the order of the result's last dimension (its global index, then the chunk's place on the grid)
            slot_pid = list(D1.chunks)
            raise_on_status(rt, 0, _first_failure(status.to_numpy(), ran, lambda slot, b: (
                layout.localindices(slot_pid[slot])[-1][0] + b, pids.index(slot_pid[slot]))))
        elif status is not None:
            st = status.to_numpy()
            raise_on_status(rt, int(np.bitwise_or.reduce(st[ran], initial=0)) if ran else 0)
    except BaseException:
        for out in chunks.values():
            out.free()
        raise
    finally:
        for t in temps:
            t.free()
        if status is not None:
            status.free()
    return DArray(layout, rdtype, chunks, rt)
