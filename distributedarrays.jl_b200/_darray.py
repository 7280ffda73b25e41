"""DArray on H100: each localpart lives in one GPU's HBM.

Python mirror of the reference's L2 layer (src/darray.jl) for exactly what the hot path needs: the ``DArray`` struct
(:25-31), constructors ``DArray(init, dims[, procs, dist])`` (:159-174), ``DArray(refs)`` (:183-216),
``distribute`` (:544-570), ``Array(d)`` (:574-582), ``localpart`` / ``localindices`` / ``locate`` / ``makelocal``
(:309-400, 448-456), range ``getindex`` -> ``SubDArray`` view (:661) and ``Array(::SubDArray)`` -- the halo read
(:584-602, 798-820).  Names, argument meaning and error behaviour follow the reference; only the chunk type differs:
``B200Array`` (device pointer + dims) is the ``A`` in ``DArray{T,N,A}`` (the seam at src/darray.jl:25).

SPMD: every rank executes the same DArray program (like ``@everywhere``); constructors and reductions are collective,
element-wise ops are purely local launches.  Layout metadata is 1-based inclusive like the reference's; Python
``d[a:b, c:d]`` slicing is the usual 0-based half-open and is translated.
"""
from __future__ import annotations

import ctypes as C
import itertools
import weakref
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .layout import Layout, Range, default_procs, layout_from_chunk_shapes, make_layout, rlen, shape_of, slab_plan
from .runtime import Runtime, close_remote_reads, open_remote_reads, runtime

_DT = {np.dtype(np.float32): _lib.F32, np.dtype(np.float64): _lib.F64, np.dtype(np.int32): _lib.I32,
       np.dtype(np.int64): _lib.I64, np.dtype(np.bool_): _lib.U8,   # UInt8 is NOT Bool: unserved eltypes raise (no silent reinterpretation)
       np.dtype(np.complex64): _lib.C64, np.dtype(np.complex128): _lib.C128,   # ComplexF32 / ComplexF64, interleaved (re, im)
       np.dtype(np.float16): _lib.F16}
_NP = {_lib.F32: np.dtype(np.float32), _lib.F64: np.dtype(np.float64), _lib.I32: np.dtype(np.int32),
       _lib.I64: np.dtype(np.int64), _lib.U8: np.dtype(np.bool_), _lib.C64: np.dtype(np.complex64), _lib.C128: np.dtype(np.complex128),
       _lib.F16: np.dtype(np.float16)}


def dab_dtype(dt) -> int:
    dt = np.dtype(dt)
    if dt not in _DT:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"element type {dt} is not served by the GPU backend (no host fallback)")
    return _DT[dt]


def np_dtype(code: int) -> np.dtype:
    return _NP[code]


def is_complex(dt) -> bool:
    return np.dtype(dt).kind == "c"


def component_dtype(dt) -> np.dtype:
    """``real(T)``: the element type of each component of a complex type (the type itself for a real one)."""
    dt = np.dtype(dt)
    return {np.dtype(np.complex64): np.dtype(np.float32), np.dtype(np.complex128): np.dtype(np.float64)}.get(dt, dt)


def refuse_float16(what: str, *xs):
    """Float16 DArrays have storage, data movement, elementwise arithmetic and reductions; ``what`` has no Float16 kernel.  Raises
    ``UnsupportedError`` naming the type when an operand (a DArray, view, transpose, array or scalar) holds Float16 values -- called
    before anything is allocated or launched."""
    for x in xs:
        x = getattr(x, "parent", x) if not hasattr(x, "dtype") else x
        dt = getattr(x, "dtype", None)
        if dt is not None and np.dtype(dt) == np.dtype(np.float16):
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} of Float16 data is not served (no Float16 kernel; no host fallback)")


_allowscalar = [True]


def allowscalar(flag: bool = True):
    """reference src/darray.jl:638-640."""
    _allowscalar[0] = bool(flag)


class B200Array:
    """A dense column-major array in one GPU's HBM: the chunk type ``A`` of ``DArray{T,N,A}``."""

    __slots__ = ("rt", "ptr", "shape", "dtype", "_own", "_keep", "_temp")

    def __init__(self, rt: Runtime, ptr: int, shape: Sequence[int], dtype, own: bool = True, keep=None, temp: bool = False):
        self.rt, self.ptr, self.shape, self.dtype = rt, int(ptr), tuple(int(s) for s in shape), np.dtype(dtype)
        self._own, self._keep, self._temp = own, keep, temp

    @classmethod
    def empty(cls, rt: Runtime, shape: Sequence[int], dtype, temp: bool = False) -> "B200Array":
        """``temp=True``: stream-ordered pool allocation for short-lived scratch (partials, gather stacks); such arrays cannot be
        shared over CUDA IPC, so localparts always use the default."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) if len(shape) else 1
        ptr = rt.alloc_temp(n * dtype.itemsize) if temp else rt.alloc(n * dtype.itemsize)
        return cls(rt, ptr, shape, dtype, temp=temp)

    @classmethod
    def from_numpy(cls, rt: Runtime, a: np.ndarray) -> "B200Array":
        a = np.asarray(a)
        dab_dtype(a.dtype)
        out = cls.empty(rt, a.shape, a.dtype)
        out.copy_from_host(a)
        return out

    @property
    def size(self) -> int:
        return int(np.prod(self.shape)) if len(self.shape) else 1

    @property
    def nbytes(self) -> int:
        return self.size * self.dtype.itemsize

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def copy_from_host(self, a: np.ndarray, sync: bool = True):
        a = np.asarray(a, dtype=self.dtype)
        if tuple(a.shape) != self.shape:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"host array {a.shape} vs chunk {self.shape}")
        if self.size == 0:
            return
        if not a.flags.f_contiguous:
            if a.ndim == 2 and a.strides[0] == a.itemsize and a.strides[1] > 0:
                # a column block of a column-major matrix: strided H2D without a host staging copy
                _lib.call("dab_h2d_2d", self.rt.ctx, C.c_void_p(self.ptr), a.shape[0] * a.itemsize, C.c_void_p(a.ctypes.data),
                          a.strides[1], a.shape[0] * a.itemsize, a.shape[1])
                if sync:
                    self.rt.sync()
                return
            a = np.asfortranarray(a)
        _lib.call("dab_h2d", self.rt.ctx, C.c_void_p(self.ptr), C.c_void_p(a.ctypes.data), self.nbytes)
        if sync:
            self.rt.sync()  # the host buffer may be pageable / temporary

    def to_numpy(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self.dtype, order="F")
        if self.size:
            _lib.call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.ptr), self.nbytes)
            self.rt.sync()
        return out

    def free(self):
        if self._own and self.ptr:
            if self._temp:
                self.rt.free_temp(self.ptr)
            else:
                self.rt.free(self.ptr)
        self.ptr = 0

    def __repr__(self):
        return f"B200Array({self.dtype}, {self.shape}, ptr=0x{self.ptr:x}, dev={self.rt.device})"


def pinned_empty(rt: Runtime, shape, dtype) -> np.ndarray:
    """A NumPy array over page-locked host memory (``dab_host_alloc``): the staging buffer for ``distribute`` / ``copyto!`` so
    that H2D runs at PCIe speed asynchronously on the ctx stream.  Freed when the array is garbage collected."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) if len(shape) else 1
    p = C.c_void_p()
    _lib.call("dab_host_alloc", rt.ctx, max(1, n * dtype.itemsize), C.byref(p))
    buf = (C.c_char * max(1, n * dtype.itemsize)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape, order="F")
    import weakref
    ctx, addr = rt.ctx, p.value
    weakref.finalize(buf, lambda: _lib.lib().dab_host_free(ctx, C.c_void_p(addr)) if ctx else None)
    return arr


_did = [0]


def _next_did(rt: Runtime) -> Tuple[int, int]:
    """``next_did()`` (src/core.jl:55-66).  Collective constructors run in the same order on every rank, so a local
    counter yields the same id everywhere."""
    _did[0] += 1
    return (1, _did[0])


# id -> WeakRef(d), exactly like the reference's registry (src/core.jl:1-30, src/darray.jl:46-49): a DArray that becomes garbage
# releases its localparts through its finalizer, so `x = A @ x` loops do not grow HBM; close(d) / d_closeall() release eagerly.
_REGISTRY: Dict[Tuple[int, int], "weakref.ReferenceType[DArray]"] = {}


def _release_chunks(chunks: Dict[int, "B200Array"], did):
    """``release_localpart`` (src/core.jl:77-82).  Frees are ordered on the ctx stream; every op that let OTHER ranks read these
    chunks ended with a collective fence (``runtime.close_remote_reads``, or the fence after an exchange's arena puts), so nobody
    is still reading when a finalizer runs."""
    for ch in list(chunks.values()):
        try:
            ch.free()
        except Exception:  # interpreter shutdown / runtime already gone: the driver reclaims the memory
            pass
    chunks.clear()
    _REGISTRY.pop(did, None)


class DArray:
    """``DArray{T,N,B200Array}`` (reference src/darray.jl:25-31)."""

    def __init__(self, layout: Layout, dtype, chunks: Dict[int, B200Array], rt: Optional[Runtime] = None):
        self.rt = rt or runtime()
        self.id = _next_did(self.rt)
        self.layout = layout
        self.dtype = np.dtype(dtype)
        self.chunks = chunks  # pid -> B200Array for the workers of THIS rank
        # invariant of the reference constructor (src/darray.jl:35-37)
        if layout.indices and layout.dims != tuple(r[1] for r in layout.indices[-1]):
            raise ValueError("ArgumentError: dimension of DArray (dim) and indices do not match")
        for pid, ch in chunks.items():
            want = shape_of(layout.localindices(pid))
            if ch.shape != want:
                raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"chunk of worker {pid} has shape {ch.shape}, layout says {want}")
        self._handles: Optional[Dict[int, bytes]] = None
        _REGISTRY[self.id] = weakref.ref(self)
        self._fin = weakref.finalize(self, _release_chunks, chunks, self.id)   # finalizer(close, d)  (src/darray.jl:47-49)

    # ---- metadata (same names as the reference struct) ---------------------------------------------------------
    @property
    def dims(self):
        return self.layout.dims

    shape = dims

    @property
    def ndim(self):
        return len(self.layout.dims)

    @property
    def size(self):
        return int(np.prod(self.layout.dims))

    @property
    def pids(self) -> np.ndarray:
        return np.asarray(self.layout.pids).reshape(self.layout.grid, order="F")

    @property
    def indices(self):
        return self.layout.indices

    @property
    def cuts(self):
        return self.layout.cuts

    def __len__(self):
        return self.size

    def __repr__(self):
        return f"DArray({self.dtype}, dims={self.dims}, grid={self.layout.grid}, pids={self.layout.pids})"

    # ---- lifetime (src/core.jl:68-105) ----------------------------------------------------------------------------
    def close(self):
        self._fin()                      # runs _release_chunks once (the chunks dict is emptied in place)

    # ---- peer handles for one-sided halo reads ------------------------------------------------------------------------
    def peer_ptr(self, pid: int) -> int:
        """Device address of worker ``pid``'s chunk as seen from this rank (local pointer or CUDA-IPC mapping)."""
        if pid in self.chunks:
            return self.chunks[pid].ptr
        if self._handles is None:
            raise _lib.DabError(_lib.ERR_ARG, "remote chunk access needs d.share() (collective) first")
        return self.rt.ipc_open(self._handles[pid])

    def share(self):
        """Collective: exchange CUDA IPC handles of all chunks so that any rank can read any chunk over NVLink
        (the GPU counterpart of every worker being able to ``remotecall_fetch`` any chunk, src/darray.jl:458)."""
        if self.rt.world == 1:
            self._handles = {}
            return self
        mine = {pid: self.rt.ipc_handle(ch.ptr) for pid, ch in self.chunks.items() if ch.size}
        allh = self.rt.allgather_object(mine)
        self._handles = {}
        for h in allh:
            self._handles.update(h)
        return self

    # ---- indexing (src/darray.jl:642-661) ---------------------------------------------------------------------------------
    def __getitem__(self, key):
        from ._sparse import SparseDArray
        if isinstance(key, DArray) and key.dtype == np.bool_ and key.dims == self.dims:
            from ._compact import getindex_mask                  # d[mask]: stream compaction on the devices (_compact.py)
            return getindex_mask(self, key)
        if isinstance(key, (DArray, SparseDArray)):
            from ._take import take                              # d[I]: 1-based linear indices held on the devices (_take.py)
            return take(self, key)
        S = self._view(key)
        return S.to_numpy()[()] if S.scalar else S

    def __setitem__(self, key, v):
        """``d[key] = v``: ``setindex!`` for every key ``__getitem__`` takes (_setindex.py).  Collective."""
        from ._setindex import setindex
        setindex(self, key, v)

    def _view(self, key) -> "SubDArray":
        """The view ``d[key]`` selects, for host keys (ints, slices, int lists and arrays; 0-based).  All ints: the one element, a view
        whose ``scalar`` is true."""
        if not isinstance(key, tuple):
            key = (key,)
        if len(key) == 1 and self.ndim > 1 and isinstance(key[0], (int, np.integer)):
            raise IndexError("linear scalar indexing of a multi-dimensional DArray is not supported")
        if len(key) != self.ndim:
            raise IndexError(f"expected {self.ndim} indices")
        if all(isinstance(k, (int, np.integer)) for k in key):
            if not _allowscalar[0]:
                raise RuntimeError("ErrorException: scalar indexing disabled")  # src/darray.jl:640
            J = tuple((int(k) % s + 1, int(k) % s + 1) if -s <= int(k) < s else _oob(k, s) for k, s in zip(key, self.dims))
            return SubDArray(self, J, tuple(True for _ in key))
        J, drop, idx = [], [], []
        for k, s in zip(key, self.dims):
            if isinstance(k, (int, np.integer)):
                kk = int(k)
                if not -s <= kk < s:
                    _oob(kk, s)
                kk %= s
                J.append((kk + 1, kk + 1))
                drop.append(True)
                idx.append(None)
            elif isinstance(k, slice):
                lo, hi, st = k.indices(s)
                if st == 1:
                    J.append((lo + 1, max(lo, hi)))
                    idx.append(None)
                else:                                      # StepRange (src/darray.jl:661): 1-based global indices lo+1 : st : ...
                    v = np.arange(lo, hi, st, dtype=np.int64) + 1
                    J.append((int(v.min()), int(v.max())) if v.size else (1, 0))
                    idx.append(v)
                drop.append(False)
            elif isinstance(k, (list, np.ndarray)) and np.asarray(k).ndim == 1 and (np.asarray(k).size == 0 or np.asarray(k).dtype.kind in "iu"):
                v = np.asarray(k, dtype=np.int64)          # Vector{Int} (0-based here, like every Python index)
                if v.size and (v.min() < -s or v.max() >= s):
                    _oob(int(v.max() if v.max() >= s else v.min()), s)
                v = np.where(v < 0, v + s, v) + 1
                J.append((int(v.min()), int(v.max())) if v.size else (1, 0))
                idx.append(v)
                drop.append(False)
            else:
                raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"index type {type(k).__name__} is not served by the GPU backend")
        return SubDArray(self, tuple(J), tuple(drop), tuple(idx) if builtins_any(i is not None for i in idx) else None)

    def __array__(self, dtype=None, copy=None):
        a = to_array(self)
        return a.astype(dtype) if dtype is not None else a

    # NumPy must defer to the reflected operators below (Array - DArray is a DArray, reference src/mapreduce.jl:186), instead of
    # gathering the DArray through __array__ and computing on the host
    __array_ufunc__ = None

    # ---- binary operators between (D)Arrays of one element type: map_localparts (reference src/mapreduce.jl:134-189) ---------
    def _mlp(self, other, f, swap=False):
        from ._broadcast import map_localparts
        if swap:
            return map_localparts(f, other, self)
        return map_localparts(f, self, other)

    def __neg__(self):
        from ._broadcast import map_
        return map_(lambda x: -x, self)                       # Base.:(-)(D::DArray) = map(-, D)  (:134)

    def __add__(self, o): return self._mlp(o, lambda a, b: a + b)
    def __radd__(self, o): return self._mlp(o, lambda a, b: a + b, True)
    def __sub__(self, o): return self._mlp(o, lambda a, b: a - b)
    def __rsub__(self, o): return self._mlp(o, lambda a, b: a - b, True)
    def __and__(self, o): return self._mlp(o, lambda a, b: a & b)
    def __or__(self, o): return self._mlp(o, lambda a, b: a | b)
    def __xor__(self, o): return self._mlp(o, lambda a, b: a ^ b)
    def __floordiv__(self, o): return self._mlp(o, lambda a, b: a // b)       # div (truncated)
    def __mod__(self, o): return self._mlp(o, lambda a, b: a % b)             # rem (Julia's %)

    def __matmul__(self, x):                                                   # A*x  (reference src/linalg.jl:280-284)
        from ._linalg import matmul
        return matmul(self, x)

    @property
    def T(self):                                                               # transpose(A), lazy (LinearAlgebra.Transpose)
        from ._linalg import Transpose
        return Transpose(self)


builtins_any = any


def _oob(k, s):
    raise IndexError(f"BoundsError: index {k} out of range for dimension of size {s}")


class SubDArray:
    """``view(d, I...)`` (reference src/darray.jl:65, 661).  Every index is an Int (dropped dim), a unit range, a StepRange or a
    Vector{Int}.  ``J`` are the 1-based inclusive bounding ranges; ``idx[k]`` is ``None`` for a unit range (then ``J[k]`` IS the
    index) or the int64 vector of 1-based global indices of a strided / vector-indexed dim."""

    def __init__(self, parent: DArray, J: Tuple[Range, ...], drop: Tuple[bool, ...], idx: Optional[Tuple] = None):
        self.parent, self.J, self.drop = parent, J, drop
        self.idx = idx if idx is not None else tuple(None for _ in J)

    @property
    def scalar(self) -> bool:
        """Every index is an Int: the view holds one element (``d[i, j]``)."""
        return all(self.drop)

    @property
    def unit(self) -> bool:
        return all(i is None for i in self.idx)

    @property
    def full_shape(self):
        return tuple(rlen(j) if ix is None else int(ix.size) for j, ix in zip(self.J, self.idx))

    @property
    def shape(self):
        return tuple(n for n, d in zip(self.full_shape, self.drop) if not d)

    dims = shape

    @property
    def dtype(self):
        return self.parent.dtype

    def index_vectors(self):
        """1-based global indices per dim (unit ranges expanded)."""
        return [np.arange(j[0], j[1] + 1, dtype=np.int64) if ix is None else ix for j, ix in zip(self.J, self.idx)]

    def restrict(self, R: Sequence[Range]) -> "SubDArray":
        """``view(s, R...)`` in the coordinates of the (undropped) view: ``Base.reindex(SD.indices, I)`` of the reference
        (src/darray.jl:606).  ``R`` holds one 1-based inclusive range per KEPT dim."""
        J, idx, it = [], [], iter(R)
        for j, ix, dr in zip(self.J, self.idx, self.drop):
            if dr:
                J.append(j)
                idx.append(None)
                continue
            lo, hi = next(it)
            if ix is None:
                J.append((j[0] + lo - 1, j[0] + hi - 1))
                idx.append(None)
            else:
                v = ix[lo - 1:hi]
                J.append((int(v.min()), int(v.max())) if v.size else (1, 0))
                idx.append(v)
        return SubDArray(self.parent, tuple(J), self.drop, tuple(idx))

    def to_device(self, rt: Optional[Runtime] = None) -> B200Array:
        """Dense device copy of the view on the calling rank's GPU: the halo read (src/darray.jl:584-602, 798-820)."""
        d = self.parent
        rt = rt or d.rt
        out = B200Array.empty(rt, self.full_shape, d.dtype)
        return self.copy_to(out)

    def copy_to(self, out: B200Array) -> B200Array:
        """``copyto!(a, s::SubDArray)`` into an existing dense device array (reference src/darray.jl:598-602, 798-820): one
        peer-load copy kernel per intersecting chunk, asynchronous on the ctx stream."""
        d = self.parent
        rt = out.rt
        full_shape = self.full_shape
        if out.size != int(np.prod(full_shape)) or out.dtype != d.dtype:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"destination {out.shape}/{out.dtype} vs view {full_shape}/{d.dtype}")
        if out.size == 0:
            return out
        if not self.unit or d.ndim > 4:
            return self._gather_to(out)
        for piece in slab_plan(d.layout, self.J):
            pid = d.layout.pids[piece.chunk]
            src_ptr = d.peer_ptr(pid)
            src_shape = shape_of(d.layout.indices[piece.chunk])
            _lib.call("dab_copy_box", rt.ctx, d.dtype.itemsize, C.c_void_p(out.ptr), _lib.sz4(full_shape),
                      _lib.sz4([r[0] - 1 for r in piece.dst] + [0] * (4 - len(piece.dst))), C.c_void_p(src_ptr), _lib.sz4(src_shape),
                      _lib.sz4([r[0] - 1 for r in piece.src] + [0] * (4 - len(piece.src))), _lib.sz4([rlen(r) for r in piece.src]))
        return out

    def _gather_to(self, out: B200Array) -> B200Array:
        """StepRange / Vector{Int} indices (and views of arrays with more than 4 dims): per chunk, the positions of the view that fall
        into the chunk (``indexin_mask``, src/darray.jl:706-710) and their local source indices; affine runs are passed as strides,
        anything else as small device index tables (``dab_gather_box``)."""
        d = self.parent
        rt = out.rt
        N = d.ndim
        if N > 8:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "views of arrays with more than 8 dimensions are not served")
        iv = self.index_vectors()
        dstr = np.cumprod([1] + [len(v) for v in iv[:-1]]).astype(np.int64)
        isz = d.dtype.itemsize
        tables: List[B200Array] = []
        for c, Kc in enumerate(d.layout.indices):
            sel = [np.nonzero((v >= k[0]) & (v <= k[1]))[0] for v, k in zip(iv, Kc)]
            if builtins_any(s.size == 0 for s in sel):
                continue
            sshape = shape_of(Kc)
            sstr = np.cumprod([1] + list(sshape[:-1])).astype(np.int64)
            dbase = sbase = 0
            ds, ss, di, si, ext = [], [], [], [], []
            for k in range(N):
                doff = sel[k].astype(np.int64) * dstr[k]
                soff = (iv[k][sel[k]] - Kc[k][0]) * sstr[k]
                dbase += int(doff[0])
                sbase += int(soff[0])
                doff, soff = doff - doff[0], soff - soff[0]
                ext.append(len(doff))
                for off, strides, tabs in ((doff, ds, di), (soff, ss, si)):
                    step = int(off[1]) if len(off) > 1 else 0
                    if len(off) <= 1 or np.array_equal(off, step * np.arange(len(off), dtype=np.int64)):
                        strides.append(step)
                        tabs.append(None)
                    else:
                        t = B200Array.from_numpy(rt, np.ascontiguousarray(off, dtype=np.int64))
                        tables.append(t)
                        strides.append(0)
                        tabs.append(t.ptr)
            pid = d.layout.pids[c]
            LL, VP = C.c_longlong * N, C.c_void_p * N
            _lib.call("dab_gather_box", rt.ctx, isz, N, C.c_void_p(out.ptr + dbase * isz), LL(*ds), VP(*di), C.c_void_p(d.peer_ptr(pid) + sbase * isz),
                      LL(*ss), VP(*si), (C.c_size_t * N)(*ext))
        for t in tables:
            t.free()                                           # stream-ordered
        return out

    def to_darray(self) -> DArray:
        """``DArray(SD::SubDArray)`` (reference src/darray.jl:603-609): a new DArray of ``size(SD)`` on ``procs(D)`` with the default
        distribution; every chunk is ``Array(D[reindex(SD.indices, I)...])`` -- here a halo read straight into the new localpart."""
        d = self.parent
        rt = d.rt
        shape = self.shape
        fenced = open_remote_reads(rt, [d], "device")

        def init(I):
            ch = B200Array.empty(rt, shape_of(I), d.dtype)
            if ch.size:
                sub = self.restrict(I)
                sub.copy_to(B200Array(rt, ch.ptr, sub.full_shape, d.dtype, own=False))
            return ch

        if len(shape) == 0:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "DArray of a zero-dimensional view")
        out = darray(init, shape, procs=list(d.layout.pids), dtype=d.dtype, rt=rt)
        close_remote_reads(rt, fenced, "device")
        return out

    def to_numpy(self) -> np.ndarray:
        dev = self.to_device()
        a = dev.to_numpy()
        dev.free()
        keep = tuple(0 if dr else slice(None) for dr in self.drop)
        return a[keep]

    def __array__(self, dtype=None, copy=None):
        a = self.to_numpy()
        return a.astype(dtype) if dtype is not None else a

    def __getitem__(self, key):
        """``view(s, I...)`` of a view composes into a view of the parent (Base.reindex)."""
        return self.parent[self._parent_key(key)]

    def __setitem__(self, key, v):
        """``s[key] = v`` writes through to the parent, as a Julia view does (Base.reindex).  Collective."""
        self.parent[self._parent_key(key)] = v

    def _parent_key(self, key) -> tuple:
        """The parent key (0-based) that ``key`` selects in this view."""
        if not isinstance(key, tuple):
            key = (key,)
        kept = [k for k, dr in enumerate(self.drop) if not dr]
        if len(key) != len(kept):
            raise IndexError(f"expected {len(kept)} indices")
        iv = self.index_vectors()
        full = list(self.parent.dims)
        pkey = [None] * len(full)
        for k, dr in enumerate(self.drop):
            if dr:
                pkey[k] = self.J[k][0] - 1
        for k, sub in zip(kept, key):
            v = iv[k] - 1                                     # 0-based global indices of this dim of the view
            if isinstance(sub, (int, np.integer)):
                pkey[k] = int(v[sub])
            else:
                w = v[sub]
                if isinstance(sub, slice) and w.size and np.array_equal(w, np.arange(w[0], w[0] + w.size)):
                    pkey[k] = slice(int(w[0]), int(w[0]) + int(w.size))
                else:
                    pkey[k] = np.asarray(w, dtype=np.int64)
        return tuple(pkey)


# ---- constructors --------------------------------------------------------------------------------------------------------


def _mk(rt: Runtime, layout: Layout, init: Callable, dtype=None) -> DArray:
    chunks: Dict[int, B200Array] = {}
    dts = set()
    for pid in layout.pids:
        if not rt.is_local(pid):
            continue
        I = layout.localindices(pid)
        part = init(I)
        if isinstance(part, np.ndarray) or np.isscalar(part):
            part = B200Array.from_numpy(rt, np.asarray(part) if dtype is None else np.asarray(part, dtype=dtype))
        if part.shape != shape_of(I):
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"init returned shape {part.shape} for indices {I}")
        chunks[pid] = part
        dts.add(part.dtype)
    if dtype is None:
        # "Constructed localparts have different eltype" (src/darray.jl:89-95): checked across all ranks
        alld = set()
        for s in rt.allgather_object(sorted(str(x) for x in dts)):
            alld.update(s)
        if len(alld) > 1:
            for ch in chunks.values():
                ch.free()
            raise RuntimeError(f"ErrorException: Constructed localparts have different `eltype`: {sorted(alld)}")
        dtype = np.dtype(alld.pop()) if alld else np.dtype(np.float64)
    return DArray(layout, dtype, chunks, rt)


def darray(init: Callable, dims: Sequence[int], procs: Optional[Sequence[int]] = None, dist: Optional[Sequence[int]] = None,
           dtype=None, rt: Optional[Runtime] = None) -> DArray:
    """``DArray(init, dims[, procs[, dist]])`` (reference src/darray.jl:159-174).  ``init(I)`` receives the tuple of
    1-based inclusive index ranges of a chunk and returns its data (NumPy array or ``B200Array``)."""
    rt = rt or runtime()
    dims = tuple(int(d) for d in dims)
    if procs is None:
        procs = default_procs(dims, rt.workers())
    return _mk(rt, make_layout(dims, procs, dist), init, dtype)


def darray_like(init: Callable, d: DArray, dtype=None) -> DArray:
    """``DArray(init, d::DArray)`` (src/darray.jl:236): same layout as ``d``."""
    return _mk(d.rt, d.layout, init, dtype)


def darray_from_chunks(parts: Sequence, grid: Sequence[int], pids: Optional[Sequence[int]] = None, rt: Optional[Runtime] = None) -> DArray:
    """``DArray(refs)`` (src/darray.jl:183-216): irregular layout from per-worker chunks, column-major grid order.
    ``parts[k]`` is a NumPy array (uploaded on the owning rank); every rank passes the same list of shapes."""
    rt = rt or runtime()
    n = int(np.prod(grid))
    pids = list(pids) if pids is not None else rt.workers()[:n]
    layout = layout_from_chunk_shapes([np.shape(p) for p in parts], grid, pids)
    by_pid = dict(zip(pids, parts))
    return _mk_from_parts(rt, layout, by_pid)


def _mk_from_parts(rt, layout, by_pid):
    chunks = {pid: B200Array.from_numpy(rt, np.asarray(by_pid[pid])) for pid in layout.pids if rt.is_local(pid)}
    dts = {np.asarray(p).dtype for p in by_pid.values()}
    if len(dts) > 1:
        for ch in chunks.values():
            ch.free()
        raise RuntimeError(f"ErrorException: Constructed localparts have different `eltype`: {sorted(map(str, dts))}")
    return DArray(layout, dts.pop(), chunks, rt)


def distribute(A: np.ndarray, procs: Optional[Sequence[int]] = None, dist: Optional[Sequence[int]] = None,
               like: Optional[DArray] = None, rt: Optional[Runtime] = None) -> DArray:
    """``distribute(A; procs, dist)`` / ``distribute(A, DA)`` (reference src/darray.jl:544-570): every rank uploads the
    slices ``A[idxs...]`` of its own workers (H2D), nothing else moves.  A host sparse matrix (``.tocsc()``) gives a sparse DArray
    (``_sparse.distribute_sparse``)."""
    if hasattr(A, "tocsc"):
        from ._sparse import distribute_sparse
        return distribute_sparse(A, procs, dist, like, rt)
    A = np.asarray(A)
    rt = rt or (like.rt if like is not None else runtime())
    dab_dtype(A.dtype)
    if like is not None:
        if tuple(A.shape) != like.dims:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"Distributed array has size {like.dims} but array has {A.shape}")
        layout = like.layout
    else:
        if procs is None:
            procs = default_procs(A.shape, rt.workers())
        layout = make_layout(A.shape, procs, dist)
    chunks = {}
    for pid in layout.pids:
        if rt.is_local(pid):
            I = layout.localindices(pid)
            ch = B200Array.empty(rt, shape_of(I), A.dtype)
            ch.copy_from_host(A[tuple(slice(lo - 1, hi) for lo, hi in I)], sync=False)
            chunks[pid] = ch
    rt.sync()
    return DArray(layout, A.dtype, chunks, rt)


def _filled(value, dtype):
    def ctor(dims, procs=None, dist=None, rt=None):
        rt = rt or runtime()
        dt = np.dtype(dtype)

        def init(I):
            ch = B200Array.empty(rt, shape_of(I), dt)
            v = np.asarray(value, dtype=dt)
            _lib.call("dab_fill", rt.ctx, dab_dtype(dt), C.c_void_p(ch.ptr), ch.size, C.c_void_p(v.ctypes.data))
            return ch

        return darray(init, dims, procs, dist, dtype=dt, rt=rt)

    return ctor


def dzeros(dims, procs=None, dist=None, dtype=np.float64, rt=None) -> DArray:
    """src/darray.jl:468-472."""
    return _filled(0, dtype)(dims, procs, dist, rt)


def dones(dims, procs=None, dist=None, dtype=np.float64, rt=None) -> DArray:
    """src/darray.jl:481-485."""
    return _filled(1, dtype)(dims, procs, dist, rt)


def dfill(v, dims, procs=None, dist=None, dtype=None, rt=None) -> DArray:
    """src/darray.jl:493-494."""
    return _filled(v, dtype if dtype is not None else np.asarray(v).dtype)(dims, procs, dist, rt)


def drand(dims, procs=None, dist=None, dtype=np.float64, seed: int = 1234, rt=None) -> DArray:
    """``drand`` (src/darray.jl:502-518) with the counter-based generator: element with global column-major linear index
    g is ``(hash32(seed, g) >> 8) * 2^-24`` -- layout-independent and reproducible on the CPU oracle.  A complex element g is
    ``complex(u(2g), u(2g+1))`` of that stream in the component type (Julia's ``rand(Complex{T}) = complex(rand(T), rand(T))``)."""
    rt = rt or runtime()
    dims = tuple(int(d) for d in dims)
    dt = np.dtype(dtype)

    def init(I):
        ch = B200Array.empty(rt, shape_of(I), dt)
        _rand_block(rt, ch, dims, I, seed)
        return ch

    return darray(init, dims, procs, dist, dtype=dt, rt=rt)


def _rand_block(rt, ch: B200Array, dims, I, seed):
    """Fill chunk ``I`` of a global array so that values depend on the GLOBAL linear index only: one launch per
    contiguous run of the chunk (runs = trailing-index combinations of the dims after the first split one)."""
    code = dab_dtype(component_dtype(ch.dtype))
    ncomp = 2 if is_complex(ch.dtype) else 1          # a complex array is filled through its real view of 2n components
    shp = shape_of(I)
    # length of the prefix of dims the chunk spans completely -> contiguous run in global memory
    run, k = 1, 0
    while k < len(dims) and shp[k] == dims[k]:
        run *= dims[k]
        k += 1
    if k < len(dims):
        run *= shp[k]
        k += 1
    strides = np.cumprod((1,) + tuple(dims[:-1])).astype(object)
    rest = [range(r[0] - 1, r[1]) for r in I[k:]]
    base0 = sum(int(strides[j]) * (I[j][0] - 1) for j in range(k))
    off = 0
    for tail in itertools.product(*reversed(rest)):
        tail = tuple(reversed(tail))
        g = base0 + sum(int(strides[k + j]) * tail[j] for j in range(len(tail)))
        _lib.call("dab_rand_u01", rt.ctx, code, C.c_void_p(ch.ptr + off * ch.dtype.itemsize), ncomp * run, int(seed), ncomp * int(g))
        off += run


# ---- access -------------------------------------------------------------------------------------------------------------


def procs(d: DArray) -> List[int]:
    return list(d.layout.pids)


def localpart(d: DArray, pid: Optional[int] = None) -> B200Array:
    """``localpart(d)`` (src/darray.jl:330-337): the chunk of worker ``pid`` (default: this rank's first worker); an
    empty array if that worker holds no part."""
    pid = d.rt.myid() if pid is None else pid
    if pid in d.chunks:
        return d.chunks[pid]
    if not d.rt.is_local(pid):
        raise _lib.DabError(_lib.ERR_ARG, f"worker {pid} does not live on rank {d.rt.rank}")
    return B200Array.empty(d.rt, (0,) * d.ndim, d.dtype)


def localindices(d: DArray, pid: Optional[int] = None):
    """src/darray.jl:394-400."""
    return d.layout.localindices(d.rt.myid() if pid is None else pid)


def locate(d: DArray, *I: int):
    """src/darray.jl:448-456."""
    return d.layout.locate(*I)


def makelocal(d: DArray, J: Sequence[Range], pid: Optional[int] = None) -> B200Array:
    """``makelocal(A, I...)`` (src/darray.jl:351-368) for 1-based unit ranges ``J``: when the ranges lie inside worker
    ``pid``'s chunk and cover it exactly the chunk itself is returned (zero-copy, :357-360); otherwise a dense device
    array is allocated and filled by the halo fetch (:361-366)."""
    pid = d.rt.myid() if pid is None else pid
    lid = d.layout.localindices(pid)
    J = tuple(J)
    if pid in d.chunks and J == lid:
        return d.chunks[pid]
    for j, s in zip(J, d.dims):
        if rlen(j) and (j[0] < 1 or j[1] > s):
            raise IndexError(f"BoundsError: attempt to access {d.dims} DArray at index {J}")
    return SubDArray(d, J, tuple(False for _ in J)).to_device()


def to_array(d: DArray) -> np.ndarray:
    """``Array(d)`` (src/darray.jl:574-582): gather every chunk into a host array (collective; on every rank).  A sparse DArray is
    densified (``Array(d)`` of sparse localparts)."""
    if not isinstance(d, DArray):
        from ._sparse import SparseDArray, to_array as sparse_to_array
        if isinstance(d, SparseDArray):
            return sparse_to_array(d)
    a = np.empty(d.dims, dtype=d.dtype, order="F")
    mine = {pid: ch.to_numpy() for pid, ch in d.chunks.items()}
    for part in d.rt.allgather_object(mine):
        for pid, h in part.items():
            I = d.layout.localindices(pid)
            if all(rlen(r) > 0 for r in I):
                a[tuple(slice(lo - 1, hi) for lo, hi in I)] = h
    return a


def copyto(dest: DArray, src: np.ndarray) -> DArray:
    """``copyto!(dest::SubOrDArray, src::AbstractArray)`` (src/darray.jl:679-687): per worker ``copyto!(localpart(dest), view(src,
    localindices(dest)...))``; a view ``dest`` takes the writes of ``view[:] = src`` (_setindex.py).  A host array is uploaded slice by
    slice; a DArray / SubDArray source (test/darray.jl:225-234) stays on the devices -- one identity broadcast per localpart, the view of
    a differently laid out source being the usual halo fetch."""
    if isinstance(dest, SubDArray):                            # copyto!(view, src): the same writes as view[:] = src
        from ._setindex import copyto_view
        return copyto_view(dest, src)
    if isinstance(src, (DArray, SubDArray)):
        from ._broadcast import broadcast_into
        if tuple(src.dims) != dest.dims:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"DArray has size {dest.dims} but the source has {tuple(src.dims)}")
        return broadcast_into(dest, lambda x: x, src)
    if not isinstance(dest, DArray):
        from ._sparse import refuse
        refuse("copyto!")
    if hasattr(src, "tocsc"):                                  # a host sparse matrix: copyto!(D, Matrix(S)) (ext/SparseArraysExt.jl:16)
        from ._sparse import host_dense
        src = host_dense(src)
    src = np.asarray(src)
    if tuple(src.shape) != dest.dims:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"DArray has size {dest.dims} but array has {src.shape}")
    for pid, ch in dest.chunks.items():
        I = dest.layout.localindices(pid)
        ch.copy_from_host(src[tuple(slice(lo - 1, hi) for lo, hi in I)].astype(dest.dtype, copy=False), sync=False)
    dest.rt.sync()
    return dest


def similar(d: DArray, dtype=None, dims=None) -> DArray:
    """``similar(d[, T[, dims]])`` (src/darray.jl:240-243): ``DArray(I -> Array{T}(undef, ...), dims, procs(d))`` -- uninitialised,
    on ``procs(d)`` with the DEFAULT distribution for those workers (a custom ``dist`` of ``d`` is not inherited, exactly as in the
    reference)."""
    if not isinstance(d, DArray):
        from ._sparse import SparseDArray, refuse
        if isinstance(d, SparseDArray):
            refuse("similar")
    dt = np.dtype(dtype) if dtype is not None else d.dtype
    return darray(lambda I: B200Array.empty(d.rt, shape_of(I), dt), d.dims if dims is None else dims, procs(d), dtype=dt, rt=d.rt)


def reshape(A: DArray, dims) -> DArray:
    """``reshape(A::DVector, d::Dims)`` (reference src/darray.jl:612-636): a NEW DArray of size ``d`` with the default layout whose chunk
    ``I`` holds, column by column, the runs ``A[a:a+nr-1]`` of the vector (``a`` = the linear index of the column's first element).  Here
    the whole chunk is ONE vector-indexed view of ``A`` -- the linear indices of the chunk's elements in column-major order -- read by the
    gather kernel straight into the new localpart (the owners of the runs may be several workers).  Like the reference: only for a
    one-dimensional DArray, ``DimensionMismatch`` unless ``prod(d) == length(A)``."""
    dims = tuple(int(v) for v in (dims if isinstance(dims, (tuple, list)) else (dims,)))
    if A.ndim != 1:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "reshape is defined for a one-dimensional DArray (reference src/darray.jl:612)")
    if int(np.prod(dims, dtype=np.int64)) != A.size:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "dimensions must be consistent with array size")
    rt = A.rt
    fenced = open_remote_reads(rt, [A], "device")
    strides = np.cumprod((1,) + dims[:-1]).astype(np.int64)

    def init(I):
        ch = B200Array.empty(rt, shape_of(I), A.dtype)
        if ch.size:
            lin = np.zeros((), dtype=np.int64)
            for k in range(len(dims) - 1, -1, -1):               # column-major order of the chunk: the first dimension varies fastest
                lo, hi = I[k]
                lin = lin[..., None] + np.arange(lo - 1, hi, dtype=np.int64) * strides[k]
            view = A[lin.reshape(-1)]
            view.copy_to(B200Array(rt, ch.ptr, view.full_shape, A.dtype, own=False))
        return ch

    out = darray(init, dims, dtype=A.dtype, rt=rt)
    close_remote_reads(rt, fenced, "device")
    return out


def fill_(d: DArray, x) -> DArray:
    """``fill!(A::DArray, x)`` (src/darray.jl:822-827)."""
    v = np.asarray(x, dtype=d.dtype)
    for ch in d.chunks.values():
        _lib.call("dab_fill", d.rt.ctx, dab_dtype(d.dtype), C.c_void_p(ch.ptr), ch.size, C.c_void_p(v.ctypes.data))
    return d


def d_closeall():
    """``d_closeall()`` (src/core.jl:97-105)."""
    for ref in list(_REGISTRY.values()):
        d = ref()
        if d is not None:
            d.close()
    _REGISTRY.clear()


def registry_size() -> int:
    """Leak check used by the tests (reference test/runtests.jl:28-37, test/darray.jl:1079-1086)."""
    return sum(1 for ref in list(_REGISTRY.values()) if ref() is not None)
