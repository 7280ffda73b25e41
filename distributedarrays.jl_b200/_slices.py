"""``mapslices(f, D; dims)`` (reference src/mapreduce.jl:191-208) on H100.

The reference first makes every slice local -- when a dimension in ``dims`` is split over several workers it redistributes ``D`` onto
``procs(D)`` with ``p = ones``, ``p[nondims] = defaultdist(size(D)[nondims], procs(D))`` (:195-203, a halo read per new chunk) -- then runs
``mapslices(f, localpart(D), dims)`` on every worker and assembles ``DArray(reshape(refs, size(procs(D))))`` from the chunk shapes (:205-207).
Each chunk's result follows Base's shape rule: entry ``j`` of the (ascending) slice dimensions takes ``size(f(slice), j)``, so a scalar
result collapses them to 1 and ``ones(6)`` over ``dims=[1,2]`` gives ``(6, 1, ...)``.

``f`` is recognised by calling it once, on the host, with a tracer for the slice (an ``Expr`` argument, as in broadcast).  The served forms
and the kernels behind them:

  f(slice)                                       per chunk
  ---------------------------------------------  ------------------------------------------------------------------------------------
  ``sort``, one dimension                        ``dab_sort_slices`` on the chunk collapsed to (inner, len, outer)
  ``svdvals``, two dimensions                    one ``dab_gather_box`` packs the slices as (m, n, batch), ``dab_svdvals_batched``,
                                                 one ``dab_gather_box`` scatters (k, 1, batch) back; Int32 / Int64 are converted to
                                                 Float64 first, as Julia's ``svdvals`` does
  ``eigvals``, two dimensions, square slices     the same with ``dab_eigvals_sym_batched`` (real symmetric slices; see ``eigvals``)
  ``det``, two dimensions, square slices         the same with ``dab_det_batched`` (K27), one value per slice
  ``sum/prod/maximum/minimum(g(slice))``, g an   the per-chunk dimensional reduction (``reduce_chunk_dims``); with ``dims=()`` there is
  elementwise traced expression (or identity)    nothing to reduce and it is one elementwise launch of g
  an elementwise expression ``g(slice)``         one elementwise launch (the result has the slice's shape)
  a value that does not depend on the slice      uploaded once, tiled into the chunk by one ``dab_gather_box`` with batch strides 0

Anything else raises ``UnsupportedError``: there is no host fallback.  Every check (``dims``, the form of ``f``, its dimension count, the
kernels' limits) happens before the first launch.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import _lib
from ._broadcast import _NPT, SLICE_TRACING, Expr, LocalArg, convert, run_local, tag_of
from ._darray import B200Array, DArray, SubDArray, darray, dab_dtype
from .layout import Layout, defaultdist, layout_from_chunk_shapes, make_layout, rlen, shape_of
from .runtime import close_remote_reads, open_remote_reads

_SORT_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int32), np.dtype(np.int64))


def tracing() -> bool:
    """True while ``mapslices`` / ``ppeval`` call ``f`` on slice tracers: ``sort``, ``svdvals``, ``eigvals``, ``det``, ``@``, ``ldiv`` and
    the reductions then return a marker."""
    return SLICE_TRACING[0] > 0


class SliceSort:
    """``f(slice) = sort(slice)``."""


class SliceSvdvals:
    """``f(slice) = svdvals(slice)``."""


class SliceEigvals:
    """``f(slice) = eigvals(slice)``."""


class SliceDet:
    """``f(slice) = det(slice)``."""


class SliceMatmul:
    """``f(slices...) = a * b`` (Julia's matrix product, Python's ``@``): each operand a slice tracer or a host array."""

    def __init__(self, a, b):
        self.a, self.b = a, b


class SliceLdiv:
    """``f(slices...) = a \\ b`` (Julia's left division, ``dab.ldiv``): each operand a slice tracer or a host array."""

    def __init__(self, a, b):
        self.a, self.b = a, b


class SliceReduce:
    """``f(slice) = op(g(slice))`` with ``op`` in + * max min and ``g`` an elementwise expression of the slice."""

    def __init__(self, op: int, expr: Expr):
        self.op, self.expr = op, expr


def _is_slice(x) -> bool:
    return isinstance(x, Expr) and x.op == "arg"


def sort_of_slice(x: Expr, by=None, kwargs=None):
    """``sort(slice)`` inside ``mapslices``."""
    if by is not None or kwargs:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices(sort) is served without keyword arguments")
    if not _is_slice(x):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices: sort of an expression of the slice is not served (sort the slice itself)")
    return SliceSort()


def reduce_of_slice(f, op, x: Expr, ds, dims, init) -> SliceReduce:
    """``sum/prod/maximum/minimum([f,] g(slice))`` inside ``mapslices``."""
    from ._mapreduce import _op_code
    if ds or dims is not None or init is not None:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices: reductions of the slice are served without dims, init or extra arguments")
    opc = op if isinstance(op, int) else _op_code(op)
    if opc not in (_lib.SUM, _lib.PROD, _lib.MAX, _lib.MIN):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices: only + * max min reductions of the slice are served")
    return SliceReduce(opc, x if f is None else Expr.wrap(f(x)))


def svdvals(A):
    """``svdvals`` of a slice: ``mapslices(svdvals, D, dims=(d1, d2))``.  There is no distributed SVD; anywhere else this raises."""
    if isinstance(A, Expr) and tracing():
        if not _is_slice(A):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices: svdvals of an expression of the slice is not served")
        return SliceSvdvals()
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "svdvals is served for the slices of a DArray only: mapslices(svdvals, D, dims=(d1, d2))")


def eigvals(A, B=None):
    """``eigvals`` of a real symmetric slice, ascending: ``ppeval(eigvals, D)`` or ``mapslices(eigvals, D, dims=(d1, d2))``.  There is no
    distributed eigensolver; anywhere else this raises.  Julia takes the symmetric path when ``ishermitian(A)`` holds; a slice that is not
    exactly symmetric has complex eigenvalues in general and raises ``UnsupportedError`` once the kernel has flagged it.  The generalised
    problem ``eigvals(A, B)`` is not served."""
    if isinstance(A, Expr) and tracing():
        if B is not None:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "eigvals(A, B): the generalised eigenvalue problem is complex in general and is "
                                        "not served")
        if not _is_slice(A):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "eigvals of an expression of the slice is not served")
        return SliceEigvals()
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "eigvals is served for the slices of a DArray only: ppeval(eigvals, D) or "
                                "mapslices(eigvals, D, dims=(d1, d2))")


def matmul_of_slices(a, b):
    """``a @ b`` while a slice function is traced (``Expr.__matmul__``, ``dab.matmul``); anywhere else it raises."""
    if not tracing():
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "a matrix product of a traced expression is only served inside ppeval")
    return SliceMatmul(a, b)


def det(A):
    """``det`` of a square slice: ``ppeval(det, D)`` or ``mapslices(det, D, dims=(d1, d2))``.  There is no distributed determinant;
    anywhere else this raises.  A triangular slice gives the product of its diagonal, any other the product of its LU factor's diagonal
    with the sign of the row swaps (exactly +0.0 for a zero pivot); det never raises for singular or non-finite input."""
    if isinstance(A, Expr) and tracing():
        if not _is_slice(A):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "det of an expression of the slice is not served")
        return SliceDet()
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "det is served for the slices of a DArray only: ppeval(det, D) or "
                                "mapslices(det, D, dims=(d1, d2))")


def ldiv(a, b):
    """Julia's ``a \\ b`` of slices (Python has no ``\\``): ``ppeval(ldiv, A, B)``, either operand possibly a broadcast host array.  A
    diagonal slice gives ``b ./ d``, a triangular one is solved by substitution, any other through its pivoted LU factorization;
    ``SingularException(i)`` for a zero diagonal entry or pivot, ``ArgumentError`` for a NaN / Inf in a slice that needs the LU path.
    Anywhere else this raises."""
    if tracing() and (isinstance(a, Expr) or isinstance(b, Expr)):
        return SliceLdiv(a, b)
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "ldiv is served for the slices of a DArray only: ppeval(ldiv, A, B)")


# ---- the rules of Base.mapslices ----------------------------------------------------------------------------------------------------


def normalise_dims(dims, ndim: int) -> Tuple[int, ...]:
    """``dims`` as the ascending tuple of distinct slice dimensions; an int, a tuple, a list or a range, possibly empty.  Anything that is
    not a dimension of ``D`` raises ``ArgumentError`` (the reference's ``size(D.indices)[dims]`` has no entry for it)."""
    if isinstance(dims, (bool, np.bool_)):
        raise _lib.ArgumentError(_lib.ERR_ARG, f"mapslices: invalid dims {dims!r}")
    if isinstance(dims, (int, np.integer)):
        dims = (dims,)
    elif isinstance(dims, (tuple, list, range, np.ndarray)):
        dims = tuple(np.asarray(dims).reshape(-1).tolist()) if isinstance(dims, np.ndarray) else tuple(dims)
    else:
        raise _lib.ArgumentError(_lib.ERR_ARG, f"mapslices: dims must be an integer or a collection of integers, got {dims!r}")
    for d in dims:
        if isinstance(d, (bool, np.bool_)) or not isinstance(d, (int, np.integer)) or not 1 <= int(d) <= ndim:
            raise _lib.ArgumentError(_lib.ERR_ARG, f"mapslices: dims {dims!r} are not dimensions of a {ndim}-dimensional DArray")
    return tuple(sorted({int(d) for d in dims}))


def result_shape(shape: Sequence[int], dims: Sequence[int], rshape: Sequence[int]) -> Tuple[int, ...]:
    """Base.mapslices' result size for an array of ``shape`` whose slices over ``dims`` map to arrays of ``rshape`` (``()`` for a
    scalar): dimension ``dims[j]`` takes ``rshape[j]`` (1 past its end), the others are kept."""
    n = len(dims)
    if len(rshape) > n and any(int(s) > 1 for s in rshape[n:]):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"mapslices cannot assign slice f(x) of size {tuple(rshape)} into output of size "
                                     f"{tuple(rshape[:n])}")
    out = [int(s) for s in shape]
    for j, d in enumerate(dims):
        out[d - 1] = int(rshape[j]) if j < len(rshape) else 1
    return tuple(out)


def redistribution_grid(D_dims: Sequence[int], grid: Sequence[int], dims: Sequence[int], nprocs: int):
    """The reference's ``p`` (src/mapreduce.jl:195-199), or None when every slice dimension is already local."""
    if all(grid[d - 1] == 1 for d in dims):
        return None
    N = len(D_dims)
    p = [1] * N
    nondims = [t for t in range(1, N + 1) if t not in dims]
    if nondims:
        for t, g in zip(nondims, defaultdist([D_dims[t - 1] for t in nondims], nprocs)):
            p[t - 1] = g
    return tuple(p)


def _dense_strides(shape: Sequence[int]) -> List[int]:
    s, out = 1, []
    for d in shape:
        out.append(s)
        s *= int(d)
    return out


def _gather(rt, es: int, dst: int, dst_strides, src: int, src_strides, extent):
    N = len(extent)
    if any(int(e) == 0 for e in extent):
        return
    LL, VP = C.c_longlong * N, C.c_void_p * N
    _lib.call("dab_gather_box", rt.ctx, es, N, C.c_void_p(dst), LL(*dst_strides), VP(*([None] * N)), C.c_void_p(src), LL(*src_strides),
              VP(*([None] * N)), (C.c_size_t * N)(*extent))


# ---- the slice function --------------------------------------------------------------------------------------------------------------


class _Plan:
    """What f is (kind), and the result shape / dtype of one chunk."""

    def __init__(self, kind: str, dims: Tuple[int, ...], dtype: np.dtype, **kw):
        self.kind, self.dims, self.dtype = kind, dims, dtype
        self.__dict__.update(kw)

    def rshape(self, shape) -> Tuple[int, ...]:
        sl = [shape[d - 1] for d in self.dims]
        if self.kind == "sort" or self.kind == "map":
            return tuple(sl)
        if self.kind == "svdvals":
            return (min(sl),)
        if self.kind == "eigvals":
            return (sl[0],)
        if self.kind in ("reduce", "det"):
            return ()
        return tuple(self.const.shape)

    def out_shape(self, shape) -> Tuple[int, ...]:
        return result_shape(shape, self.dims, self.rshape(shape))


def _classify(f, D: DArray, dims: Tuple[int, ...]) -> _Plan:
    dt = D.dtype
    tag = tag_of(dt)
    x = Expr("arg", (), tag, 0)
    SLICE_TRACING[0] += 1
    try:
        r = f(x)
    except _lib.DabError:
        raise
    except Exception as e:  # noqa: BLE001 - anything f does with the tracer that is not a served form
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices: {getattr(f, '__name__', f)!r} is not a served slice function "
                                    f"({type(e).__name__}: {e}); served: sort, svdvals, eigvals, det, sum/prod/maximum/minimum of an elementwise "
                                    "expression of the slice, elementwise expressions, constant results") from None
    finally:
        SLICE_TRACING[0] -= 1
    return plan_of(r, dims, dt)


def plan_of(r, dims: Tuple[int, ...], dt: np.dtype, what: str = "mapslices") -> _Plan:
    """The plan of a traced slice function whose result is ``r``, for slices over ``dims`` of an array of eltype ``dt``."""
    from ._mapreduce import _result_dtype, classify_map
    if isinstance(r, SliceMatmul):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}: matrix products of slices are served by ppeval(*, A, B) only")
    if isinstance(r, SliceLdiv):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}: ldiv (a \\ b) of slices is served by ppeval(ldiv, A, B) only")
    if isinstance(r, SliceDet):
        if len(dims) != 2:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(det) is served for matrix slices (two slice dimensions), got dims {dims}")
        if dt not in _SORT_DTYPES:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(det): eltype {dt} (served: Float32 Float64 Int32 Int64)")
        return _Plan("det", dims, dt if dt.kind == "f" else np.dtype(np.float64))
    if isinstance(r, SliceEigvals):
        if len(dims) != 2:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(eigvals) is served for matrix slices (two slice dimensions), got "
                                        f"dims {dims}")
        if dt not in _SORT_DTYPES:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(eigvals): eltype {dt} (served: Float32 Float64 Int32 Int64)")
        return _Plan("eigvals", dims, dt if dt.kind == "f" else np.dtype(np.float64))
    if isinstance(r, SliceSort):
        if len(dims) != 1:
            raise _lib.ArgumentError(_lib.ERR_ARG, f"mapslices(sort): the slice over dims {dims} is not a vector; sort of a multi-dimensional "
                                     "array needs dims")
        if dt not in _SORT_DTYPES:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices(sort): eltype {dt} (served: Float32 Float64 Int32 Int64)")
        return _Plan("sort", dims, dt)
    if isinstance(r, SliceSvdvals):
        if len(dims) != 2:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices(svdvals) is served for two slice dimensions, got dims {dims}")
        if dt not in _SORT_DTYPES:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices(svdvals): eltype {dt} (served: Float32 Float64 Int32 Int64)")
        return _Plan("svdvals", dims, dt if dt.kind == "f" else np.dtype(np.float64))
    if isinstance(r, SliceReduce):
        e = r.expr
        if e.jt not in ("i32", "i64", "f32", "f64"):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices: reductions of {e.jt} values are not served")
        mapc, param, _ = classify_map(lambda _x: e, dt)
        if param is not None:
            mapc = None
        src_dt = dt if mapc is not None else _NPT[e.jt]
        rdt = _result_dtype(src_dt, r.op, mapc if mapc is not None else _lib.MAP_ID)
        return _Plan("reduce", dims, rdt, op=r.op, expr=e, mapc=mapc)
    if isinstance(r, Expr):
        return _Plan("map", dims, _NPT[r.jt], expr=r)
    c = np.asarray(r)
    if c.dtype == object:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices: result of type {type(r).__name__} is not served")
    dab_dtype(c.dtype)
    return _Plan("const", dims, c.dtype, const=np.asfortranarray(c))


# ---- per chunk -----------------------------------------------------------------------------------------------------------------------


def _sort_chunk(rt, plan: _Plan, ch: B200Array, out: B200Array):
    d = plan.dims[0]
    s = ch.shape
    inner, ln, outer = int(np.prod(s[:d - 1])), s[d - 1], int(np.prod(s[d:]))
    _lib.call("dab_sort_slices", rt.ctx, dab_dtype(ch.dtype), C.c_void_p(ch.ptr), C.c_void_p(out.ptr), inner, ln, outer)


def _packed_chunk(rt, plan: _Plan, ch: B200Array, out: B200Array, status_ptr: int, temps: List[B200Array]):
    """svdvals / eigvals / det: the slices packed as (m, n, batch), one batched kernel, the (k, batch) values scattered into the chunk."""
    d1, d2 = plan.dims
    s = ch.shape
    m, n = s[d1 - 1], s[d2 - 1]
    k = 1 if plan.kind == "det" else min(m, n)
    wdt = plan.dtype
    if plan.kind == "det" and n == 0:                              # det of a 0 x 0 matrix is one(T): no kernel
        out.copy_from_host(np.ones(out.shape, dtype=wdt))
        return
    src = ch
    if ch.dtype != wdt:                                            # svdvals / eigvals(::Matrix{Int}) work on Float64
        src = B200Array.empty(rt, s, wdt, temp=True)
        temps.append(src)
        run_local(rt, convert(Expr("arg", (), tag_of(ch.dtype), 0), tag_of(wdt)), src, [LocalArg(ch, None, tag_of(ch.dtype))])
    batch = int(np.prod([s[j] for j in range(len(s)) if j not in (d1 - 1, d2 - 1)]))
    packed = B200Array.empty(rt, (m * n * batch,), wdt, temp=True)
    S = B200Array.empty(rt, (k * batch,), wdt, temp=True)
    temps += [packed, S]
    pstr, sstr, bstr = [], [], 1
    for j in range(len(s)):
        if j == d1 - 1:
            pstr.append(1)
            sstr.append(1)
        elif j == d2 - 1:
            pstr.append(m)
            sstr.append(0)
        else:
            pstr.append(m * n * bstr)
            sstr.append(k * bstr)
            bstr *= s[j]
    es = wdt.itemsize
    _gather(rt, es, packed.ptr, pstr, src.ptr, _dense_strides(s), s)                 # slices -> (m, n, batch)
    if plan.kind == "svdvals":
        _lib.call("dab_svdvals_batched", rt.ctx, dab_dtype(wdt), C.c_void_p(packed.ptr), m, n, batch, C.c_void_p(S.ptr), C.c_void_p(status_ptr))
    elif plan.kind == "det":
        _lib.call("dab_det_batched", rt.ctx, dab_dtype(wdt), n, C.c_void_p(packed.ptr), n * n, C.c_void_p(S.ptr), batch)
    else:
        _lib.call("dab_eigvals_sym_batched", rt.ctx, dab_dtype(wdt), C.c_void_p(packed.ptr), n, batch, C.c_void_p(S.ptr), C.c_void_p(status_ptr))
    _gather(rt, es, out.ptr, _dense_strides(out.shape), S.ptr, sstr, out.shape)      # (k, 1, batch) -> the result chunk


def _reduce_chunk(rt, plan: _Plan, ch: B200Array, out: B200Array, temps: List[B200Array]):
    from ._mapreduce import reduce_chunk_dims
    tag = tag_of(ch.dtype)
    if not plan.dims:                                              # dims=(): op of one value is the value (in the result type)
        run_local(rt, convert(plan.expr, tag_of(out.dtype)), out, [LocalArg(ch, None, tag)])
        return
    src, mapc = ch, plan.mapc
    if mapc is None:                                               # a general map: one elementwise launch into a temporary first
        src = B200Array.empty(rt, ch.shape, _NPT[plan.expr.jt], temp=True)
        temps.append(src)
        run_local(rt, plan.expr, src, [LocalArg(ch, None, tag)])
        mapc = _lib.MAP_ID
    r = reduce_chunk_dims(rt, src, plan.dims, plan.op, mapc, plan.dtype)
    temps.append(r)
    _lib.call("dab_d2d", rt.ctx, C.c_void_p(out.ptr), C.c_void_p(r.ptr), out.nbytes)


def _const_chunk(rt, plan: _Plan, cdev: B200Array, out: B200Array):
    c = plan.const
    cstr = _dense_strides(c.shape)
    src_strides = [0] * out.ndim
    for j, d in enumerate(plan.dims):
        if j < c.ndim:
            src_strides[d - 1] = cstr[j]
    _gather(rt, c.dtype.itemsize, out.ptr, _dense_strides(out.shape), cdev.ptr, src_strides, out.shape)


def check_limits(plan: _Plan, shapes, what: str = "mapslices"):
    """The kernels' limits on the slices of chunks of ``shapes``, checked before anything is launched."""
    if plan.kind not in ("svdvals", "eigvals", "det"):
        return
    d1, d2 = plan.dims
    for s in shapes:
        m, n = s[d1 - 1], s[d2 - 1]
        if plan.kind == "svdvals" and (min(m, n) > _lib.SVDVALS_MAX_K or m * n > _lib.SVDVALS_MAX_ELEMS):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(svdvals): slices of {m}x{n}; served: min(m,n) <= "
                                        f"{_lib.SVDVALS_MAX_K} and m*n <= {_lib.SVDVALS_MAX_ELEMS}")
        if plan.kind in ("eigvals", "det"):
            if m != n:                                             # LinearAlgebra.checksquare
                raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"matrix is not square: dimensions are ({m}, {n})")
            lim = _lib.EIGVALS_SYM_MAX_N if plan.kind == "eigvals" else _lib.LU_MAX_N
            if n > lim:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}({plan.kind}): slices of {m}x{n}; served: n <= {lim}")


def raise_on_status(rt, flags: int, first=None):
    """The status words of dab_svdvals_batched / dab_eigvals_sym_batched, ORed over this rank's chunks, and ``first``, this rank's first
    failing ``ldiv`` slice as ``(order, info)`` (``info`` 0 for a NaN / Inf on the LU path) or None: every rank raises the same
    exception, or none.  ``order`` sorts the slices as the result's last dimension does, so the failure raised is the lowest of all ranks'."""
    if rt.world > 1:                                               # the ranks stay in step: one gather of both
        firsts = []
        for f, fi in rt.allgather_object((flags, first)):
            flags |= int(f)
            if fi is not None:
                firsts.append(tuple(fi))
        first = min(firsts) if firsts else None
    if first is not None:
        if first[-1] == 0:
            raise _lib.ArgumentError(_lib.ERR_ARG, "ArgumentError: matrix contains Infs or NaNs")
        raise _lib.SingularException(first[-1])
    if flags & 1:
        raise _lib.ArgumentError(_lib.ERR_ARG, "ArgumentError: matrix contains Infs or NaNs")
    if flags & 2:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "eigvals: a slice is not symmetric; its eigenvalues are complex in general and "
                                    "complex element types are not served")


def run_chunk(rt, plan: _Plan, ch: B200Array, out: B200Array, status_ptr: int, cdev, temps: List[B200Array]):
    """One chunk of a mapslices plan: ``out`` (already of the result shape) from ``ch``."""
    if plan.kind == "sort":
        _sort_chunk(rt, plan, ch, out)
    elif plan.kind in ("svdvals", "eigvals", "det"):
        _packed_chunk(rt, plan, ch, out, status_ptr, temps)
    elif plan.kind == "reduce":
        _reduce_chunk(rt, plan, ch, out, temps)
    elif plan.kind == "map":
        run_local(rt, plan.expr, out, [LocalArg(ch, None, tag_of(ch.dtype))])
    else:
        _const_chunk(rt, plan, cdev, out)


def _redistribute(D: DArray, p) -> DArray:
    """``DArray(size(D), procs(D), p) do I; D[I...] end`` (src/mapreduce.jl:200-202): every new chunk is one halo read."""
    rt = D.rt
    fenced = open_remote_reads(rt, [D], "device")

    def init(I):
        ch = B200Array.empty(rt, shape_of(I), D.dtype)
        if ch.size:
            SubDArray(D, tuple(I), tuple(False for _ in I)).copy_to(ch)
        return ch

    DD = darray(init, D.dims, list(D.layout.pids), p, dtype=D.dtype, rt=rt)
    close_remote_reads(rt, fenced, "device")
    return DD


def mapslices(f, D: DArray, dims) -> DArray:
    """``mapslices(f, D; dims)`` (reference src/mapreduce.jl:191-208).  See the module docstring for the served ``f``."""
    from ._sparse import SparseDArray, refuse
    if isinstance(D, SparseDArray):
        refuse("mapslices")
    if isinstance(D, SubDArray):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices of a view: make it a DArray first (DArray(view))")
    if D.dtype.kind == "c":
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mapslices of a {D.dtype} DArray is not served (no complex slice kernels)")
    from ._darray import refuse_float16
    refuse_float16("mapslices", D)
    N = D.ndim
    dims = normalise_dims(dims, N)
    if N > 8:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices over more than 8 dimensions is not served")
    plan = _classify(f, D, dims)
    # ---- the working layout and every chunk's result shape: pure host logic, checked before anything is launched
    p = redistribution_grid(D.dims, D.layout.grid, dims, len(D.layout.pids))
    L: Layout = D.layout if p is None else make_layout(D.dims, list(D.layout.pids), p)
    if any(rlen(r) == 0 for I in L.indices for r in I):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "mapslices over a DArray with an empty localpart is not served")
    in_shapes = [shape_of(I) for I in L.indices]
    out_shapes = [plan.out_shape(s) for s in in_shapes]
    check_limits(plan, in_shapes)
    layout = layout_from_chunk_shapes(out_shapes, L.grid, L.pids)
    # ---- launches
    rt = D.rt
    W = D if p is None else _redistribute(D, p)
    temps: List[B200Array] = []
    chunks: Dict[int, B200Array] = {}
    status = cdev = None
    try:
        if plan.kind in ("svdvals", "eigvals"):
            status = B200Array.empty(rt, (max(1, len(W.chunks)),), np.int32, temp=True)
        if plan.kind == "const":
            cdev = B200Array.from_numpy(rt, plan.const) if plan.const.size else None
        for slot, (pid, ch) in enumerate(W.chunks.items()):
            out = B200Array.empty(rt, out_shapes[L.pids.index(pid)], plan.dtype)
            chunks[pid] = out
            if out.size == 0:
                continue
            run_chunk(rt, plan, ch, out, status.ptr + 4 * slot if status is not None else 0, cdev, temps)
        if status is not None:
            raise_on_status(rt, int(np.bitwise_or.reduce(status.to_numpy()[:len(W.chunks)], initial=0)))
    except BaseException:
        for out in chunks.values():
            out.free()
        raise
    finally:
        for t in temps:
            t.free()
        if status is not None:
            status.free()
        if cdev is not None:
            cdev.free()
        if W is not D:
            W.close()
    return DArray(layout, plan.dtype, chunks, rt)
