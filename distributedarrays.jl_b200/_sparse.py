"""Sparse DArrays: ``DArray{T,2,SparseMatrixCSC{T,Int}}`` with every localpart a CSC block in one GPU's HBM (row f9 of the scope table).

The reference's ``DArray{T,N,A}`` is generic in its chunk type, and ``SparseMatrixCSC`` is the one non-``Array`` chunk type it supports:
``distribute(sprandn(...))`` gives sparse localparts (src/darray.jl:544-561, chunk ``I`` is ``A[I...]``), ``ext/SparseArraysExt.jl`` adds
``nnz`` and ``copyto!`` from a sparse matrix, and ``mul!(y, A::DMatrix, x)`` (src/linalg.jl:78-167) works on them unchanged because
``localpart(A)*xj`` dispatches to SparseArrays.  Here:

* ``distribute(S)`` of anything with ``.tocsc()`` (scipy.sparse matrices and arrays; duck-typed, scipy is never imported) uses the layout
  dense ``distribute`` makes; each rank uploads only its own chunks.  The host canonicalises a copy first: rows sorted within each column,
  duplicates summed in storage order, explicitly stored zeros kept.
* each chunk holds ``colptr`` (Int64, 0-based, ncols + 1), ``rowval`` (Int32 local rows, sorted within each column) and ``nzval`` (T);
  the row-major copy that ``A*x`` runs on (K19 ``dab_csc_to_csr``) is built by the first ``A*x`` and kept with the chunk.  No operation
  changes a sparse DArray's values, so the copy cannot go stale; an in-place operation added later must drop it.
* the tile products are K18 ``dab_spmv`` inside the unchanged ``mul!`` of ``_linalg`` (exchange, fences, ``dab_accumulate_stack``).
* every other operation raises ``UnsupportedError`` before it allocates or launches anything.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, Optional, Sequence

import numpy as np

from . import _lib
from ._darray import _REGISTRY, B200Array, DArray, _next_did, _release_chunks, dab_dtype
from .layout import Layout, default_procs, make_layout, rlen, shape_of
from .runtime import Runtime, runtime

SPARSE_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int32), np.dtype(np.int64))
MAX_ROWS = (1 << 31) - 1            # rowval / colidx are Int32
MAX_NNZ = 1 << 32                   # per chunk, exclusive: the K19 words carry the storage position in 32 bits
SERVED = ("a sparse DArray serves distribute, nnz, to_array, localpart, close, and the matrix-vector products A*x, A'*x, "
          "transpose(A)*x and mul!(y, A, x, a, b) with a vector x and a dense DVector y")


def refuse(what: str):
    raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} of a sparse DArray is not served: {SERVED}")


class SparseChunk:
    """One ``SparseMatrixCSC`` localpart in HBM: ``colptr`` / ``rowval`` / ``nzval``, and the row-major copy once ``A*x`` needed it."""

    __slots__ = ("rt", "shape", "dtype", "nnz", "colptr", "rowval", "nzval", "_csr")

    def __init__(self, rt: Runtime, shape, colptr: np.ndarray, rowval: np.ndarray, nzval: np.ndarray):
        self.rt, self.shape, self.dtype = rt, tuple(int(s) for s in shape), np.dtype(nzval.dtype)
        self.nnz = int(nzval.size)
        self.colptr = B200Array.from_numpy(rt, np.ascontiguousarray(colptr, dtype=np.int64))
        self.rowval = B200Array.from_numpy(rt, np.ascontiguousarray(rowval, dtype=np.int32))
        self.nzval = B200Array.from_numpy(rt, np.ascontiguousarray(nzval))
        self._csr = None

    @property
    def csr_built(self) -> bool:
        return self._csr is not None

    def csr(self):
        """``(rowptr, colidx, val)``: the row-major copy (K19), rows ascending and columns ascending within a row; built once."""
        if self._csr is None:
            m, n = self.shape
            rowptr = B200Array.empty(self.rt, (m + 1,), np.int64)
            colidx = B200Array.empty(self.rt, (self.nnz,), np.int32)
            val = B200Array.empty(self.rt, (self.nnz,), self.dtype)
            _lib.call("dab_csc_to_csr", self.rt.ctx, dab_dtype(self.dtype), m, n, self.nnz, C.c_void_p(self.colptr.ptr), C.c_void_p(self.rowval.ptr),
                      C.c_void_p(self.nzval.ptr), C.c_void_p(rowptr.ptr), C.c_void_p(colidx.ptr), C.c_void_p(val.ptr))
            self._csr = (rowptr, colidx, val)
        return self._csr

    def matvec(self, trans: bool, x_ptr: int, r_ptr: int):
        """``r = localpart(A)'*x`` (trans; the CSC arrays read as the rows of A') or ``r = localpart(A)*x`` (the row-major copy): K18."""
        m, n = self.shape
        if trans:
            rows, ptr, idx, val = n, self.colptr, self.rowval, self.nzval
        else:
            rows, (ptr, idx, val) = m, self.csr()
        _lib.call("dab_spmv", self.rt.ctx, dab_dtype(self.dtype), rows, self.nnz, C.c_void_p(ptr.ptr), C.c_void_p(idx.ptr), C.c_void_p(val.ptr),
                  C.c_void_p(x_ptr), C.c_void_p(r_ptr))

    def to_host(self):
        """``(shape, colptr, rowval, nzval)`` as host arrays."""
        return self.shape, self.colptr.to_numpy(), self.rowval.to_numpy(), self.nzval.to_numpy()

    def free(self):
        for a in (self.colptr, self.rowval, self.nzval) + (self._csr or ()):
            a.free()
        self._csr = None

    def __repr__(self):
        return f"SparseChunk({self.dtype}, {self.shape}, nnz={self.nnz})"

    # a dense kernel path that reaches a sparse chunk refuses here, before its first launch
    @property
    def ptr(self):
        refuse("a dense kernel")

    @property
    def size(self):
        refuse("a dense kernel")


class SparseDArray:
    """``DArray{T,2,SparseMatrixCSC{T,Int}}``: the same ``Layout``, registry entry, ``WeakRef`` and finalizer as ``DArray``."""

    __array_ufunc__ = None           # NumPy must not gather it through __array__ either

    def __init__(self, layout: Layout, dtype, chunks: Dict[int, SparseChunk], chunk_nnz: Sequence[int], rt: Optional[Runtime] = None):
        self.rt = rt or runtime()
        self.id = _next_did(self.rt)
        self.layout = layout
        self.dtype = np.dtype(dtype)
        self.chunks = chunks             # pid -> SparseChunk for the workers of THIS rank
        self.chunk_nnz = tuple(int(v) for v in chunk_nnz)   # stored entries of every chunk, in layout order (host metadata on every rank)
        _REGISTRY[self.id] = weakref.ref(self)
        self._fin = weakref.finalize(self, _release_chunks, chunks, self.id)

    @property
    def dims(self):
        return self.layout.dims

    shape = dims

    @property
    def ndim(self):
        return 2

    @property
    def pids(self) -> np.ndarray:
        return np.asarray(self.layout.pids).reshape(self.layout.grid, order="F")

    @property
    def indices(self):
        return self.layout.indices

    @property
    def cuts(self):
        return self.layout.cuts

    def nnz(self) -> int:
        return sum(self.chunk_nnz)

    # the element count and the peer pointers of the dense paths (reductions, scans, slices, halo reads) refuse before any launch
    @property
    def size(self):
        refuse("a dense operation")

    def peer_ptr(self, pid):
        refuse("a halo read")

    def share(self):
        refuse("a halo read")

    def close(self):
        self._fin()

    def __repr__(self):
        return f"SparseDArray({self.dtype}, dims={self.dims}, nnz={self.nnz()}, grid={self.layout.grid}, pids={self.layout.pids})"

    def __matmul__(self, x):
        from ._linalg import matmul
        return matmul(self, x)

    @property
    def T(self):
        from ._linalg import Transpose
        return Transpose(self)

    def __array__(self, dtype=None, copy=None):
        refuse("conversion to a NumPy array (use to_array)")

    def __getitem__(self, key):
        refuse("indexing and views")

    def __setitem__(self, key, value):
        refuse("setindex!")

    def __eq__(self, other):
        refuse("==")

    __ne__ = __eq__
    __hash__ = object.__hash__

    def __iter__(self):
        refuse("iteration")

    def __len__(self):
        refuse("length")

    def __bool__(self):
        refuse("truth value")


def _refused_operator(name):
    def op(self, *args):
        refuse(f"operator {name}")
    return op


for _name in ("add", "radd", "sub", "rsub", "mul", "rmul", "truediv", "rtruediv", "floordiv", "rfloordiv", "mod", "rmod", "pow", "rpow", "and",
              "rand", "or", "ror", "xor", "rxor", "neg", "pos", "abs", "lt", "le", "gt", "ge", "rmatmul"):
    setattr(SparseDArray, f"__{_name}__", _refused_operator(_name))


# ---- construction ----------------------------------------------------------------------------------------------------------------------


def check_host_sparse(S):
    """Shape and element type of a host sparse matrix, refused before anything is converted or allocated."""
    shape = tuple(int(v) for v in S.shape)
    if len(shape) != 2:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"sparse arrays of {len(shape)} dimensions are not served (only sparse matrices)")
    dt = np.dtype(S.dtype)
    if dt not in SPARSE_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"sparse DArrays of element type {dt} are not served (Float32, Float64, Int32, Int64)")
    return shape, dt


def canonical_csc(S):
    """``(shape, indptr, rows, vals)`` of a canonical copy of ``S.tocsc()``: rows ascending within each column, duplicate entries summed in
    storage order (``np.add.at`` applies repeated indices one after another), explicit zeros kept.  The input object is not modified."""
    shape, dt = check_host_sparse(S)
    m, n = shape
    Ac = S.tocsc()
    indptr = np.array(Ac.indptr, dtype=np.int64)
    nnz = int(indptr[-1]) if indptr.size else 0
    rows = np.array(Ac.indices[:nnz], dtype=np.int64)
    vals = np.array(Ac.data[:nnz], dtype=dt)
    if nnz > 1:
        cols = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr))
        if np.any((cols[1:] == cols[:-1]) & (rows[1:] <= rows[:-1])):
            order = np.lexsort((rows, cols))                        # stable: equal (col, row) keep their storage order
            rows, cols, vals = rows[order], cols[order], vals[order]
            first = np.ones(nnz, dtype=bool)
            first[1:] = (cols[1:] != cols[:-1]) | (rows[1:] != rows[:-1])
            if not first.all():
                gid = np.cumsum(first) - 1
                out = vals[first].copy()
                with np.errstate(all="ignore"):                     # Int32 / Int64 sums wrap, as Julia's
                    np.add.at(out, gid[~first], vals[~first])
                rows, cols, vals = rows[first], cols[first], out
            indptr = np.zeros(n + 1, dtype=np.int64)
            indptr[1:] = np.cumsum(np.bincount(cols, minlength=n))
    return shape, indptr, rows, vals


def cut_chunk(indptr: np.ndarray, rows: np.ndarray, vals: np.ndarray, I):
    """Chunk ``A[I...]`` of a canonical CSC matrix, cut from the raw arrays (so stored zeros survive): ``(colptr, rowval, nzval)`` with
    local 0-based rows."""
    (r0, r1), (c0, c1) = I
    ncols = max(0, c1 - c0 + 1)
    seg = indptr[c0 - 1:c0 - 1 + ncols + 1] if ncols else indptr[c0 - 1:c0]
    lo, hi = int(seg[0]), int(seg[-1])
    rr, vv = rows[lo:hi], vals[lo:hi]
    keep = (rr >= r0 - 1) & (rr <= r1 - 1)
    colptr = np.zeros(ncols + 1, dtype=np.int64)
    if ncols:
        cc = np.repeat(np.arange(ncols, dtype=np.int64), np.diff(seg))
        colptr[1:] = np.cumsum(np.bincount(cc[keep], minlength=ncols))
    return colptr, (rr[keep] - (r0 - 1)).astype(np.int32), vv[keep]


def distribute_sparse(S, procs: Optional[Sequence[int]] = None, dist: Optional[Sequence[int]] = None, like=None,
                      rt: Optional[Runtime] = None) -> SparseDArray:
    """``distribute(S; procs, dist)`` / ``distribute(S, DA)`` of a host sparse matrix (reference src/darray.jl:544-570)."""
    shape, dt = check_host_sparse(S)
    rt = rt or (like.rt if like is not None else runtime())
    if like is not None:
        if tuple(shape) != tuple(like.dims):
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"Distributed array has size {tuple(like.dims)} but array has {shape}")
        layout = like.layout
    else:
        if procs is None:
            procs = default_procs(shape, rt.workers())
        layout = make_layout(shape, procs, dist)
    for I in layout.indices:
        if rlen(I[0]) > MAX_ROWS or rlen(I[1]) > MAX_ROWS:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"sparse chunks of more than 2^31-1 rows or columns are not served (chunk {shape_of(I)})")
    shape, indptr, rows, vals = canonical_csc(S)
    parts = [cut_chunk(indptr, rows, vals, I) for I in layout.indices]
    for (colptr, rv, nz), I in zip(parts, layout.indices):
        if nz.size >= MAX_NNZ:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"sparse chunks of 2^32 or more stored entries are not served (chunk {shape_of(I)} "
                                        f"holds {nz.size})")
    chunks = {}
    for c, pid in enumerate(layout.pids):
        if rt.is_local(pid):
            chunks[pid] = SparseChunk(rt, shape_of(layout.indices[c]), *parts[c])
    rt.sync()
    return SparseDArray(layout, dt, chunks, [p[2].size for p in parts], rt)


def host_dense(S) -> np.ndarray:
    """``Matrix(S)`` of a host sparse matrix: every stored value in its place (a stored -0.0 stays -0.0), duplicates summed."""
    shape, indptr, rows, vals = canonical_csc(S)
    a = np.zeros(shape, dtype=vals.dtype)
    a[rows, np.repeat(np.arange(shape[1], dtype=np.int64), np.diff(indptr))] = vals
    return a


# ---- access ----------------------------------------------------------------------------------------------------------------------------


def to_array(S: SparseDArray) -> np.ndarray:
    """``Array(S)``: the dense host matrix (collective).  The three arrays of every chunk are copied back and densified on the host."""
    a = np.zeros(S.dims, dtype=S.dtype, order="F")
    mine = {pid: ch.to_host() for pid, ch in S.chunks.items()}
    for part in S.rt.allgather_object(mine):
        for pid, (shape, colptr, rowval, nzval) in part.items():
            (r0, _), (c0, _) = S.layout.localindices(pid)
            cols = np.repeat(np.arange(shape[1], dtype=np.int64), np.diff(colptr))
            a[rowval.astype(np.int64) + (r0 - 1), cols + (c0 - 1)] = nzval
    return a
