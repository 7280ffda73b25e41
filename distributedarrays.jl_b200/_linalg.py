"""Level-2 linear algebra and transposes on DArrays (widening row f4/f3 of the scope table; all HBM-bound).

Mirrors the reference's ``src/linalg.jl``:

* ``transpose(D)`` / ``adjoint(D)`` lazy wrappers and ``copy`` of them (:1-17)           -> K10 ``dab_transpose_box``
* ``mul!(y::DVector, A::DMatrix, x, a, b)`` and the Adjoint/Transpose forms (:78-167),
  ``A*x``, ``A'*x``, ``transpose(A)*x`` (:280-284, 293-301)                               -> K9 ``dab_gemv`` + the same partial
  exchange as mapreducedim_between (NCCL send/recv to the owner of each y chunk)
* the same ``mul!`` / ``A*x`` / ``A'*x`` with SparseMatrixCSC chunks (``_sparse.SparseDArray``)                   -> K18 ``dab_spmv``
  (A*x on the row-major copy K19 ``dab_csc_to_csr`` builds once per chunk), same exchange and fold
* ``lmul!(D::Diagonal, DA)`` / ``rmul!(DA, D::Diagonal)`` (:169-187)                      -> fused broadcast with extrusion

* ``mul!(C::DMatrix, A::DMatrix, B::AbstractMatrix, a, b)`` and the Adjoint/Transpose forms, ``A*B``, ``A'*B`` (:189-311)
                                                                                          -> K12 ``dab_gemm`` (wgmma 3xTF32 tile
  products for Float32, SIMT tiles for Float64 / Int32 / Int64) + the same exchange of the tile results to the owners of C
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from ._darray import refuse_float16, B200Array, DArray, SubDArray, dab_dtype, darray
from ._sparse import SparseDArray, refuse
from .layout import make_layout, rlen, shape_of
from .runtime import Runtime, close_remote_reads, deliver, exchange_stacks, grouped_exchange, open_remote_reads

_GEMV_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int32), np.dtype(np.int64))


class Transpose:
    """``transpose(D)``: lazy wrapper, as LinearAlgebra.Transpose{T,<:DArray{T,2}}."""

    conj = False

    def __init__(self, parent: DArray):
        if parent.ndim != 2:
            raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "transpose/adjoint wrap a DMatrix")
        self.parent = parent

    @property
    def dims(self):
        return (self.parent.dims[1], self.parent.dims[0])

    def copy(self) -> DArray:
        return copy_transposed(self)

    def __matmul__(self, x):
        return matmul(self, x)


class Adjoint(Transpose):
    """``D'`` / ``adjoint(D)`` (reference src/linalg.jl:1-8): the conjugate transpose.  For a real element type it equals the transpose;
    ``copy`` of the adjoint of a ComplexF32 / ComplexF64 DMatrix conjugates every element on the way (``dab_adjoint_box``)."""

    conj = True


def transpose(D: DArray) -> Transpose:
    return Transpose(D)


def adjoint(D: DArray) -> Adjoint:
    return Adjoint(D)


def _refuse_complex(what: str, *xs):
    """Complex matrix products (GEMV / GEMM) have no kernel yet: refuse on the host, before any allocation or launch."""
    for x in xs:
        dt = x.parent.dtype if isinstance(x, Transpose) else (x.dtype if isinstance(x, (DArray, SubDArray, SparseDArray)) else np.asarray(x).dtype)
        if np.dtype(dt).kind == "c":
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} with element type {np.dtype(dt)} is not served (no complex GEMV / GEMM kernel)")


def copy_transposed(W: Transpose) -> DArray:
    """``copy(::Transpose{T,<:DArray{T,2}})`` / ``copy(::Adjoint…)`` (reference src/linalg.jl:1-17):
    ``DArray(reverse(size(D)), procs(D)) do I;  transpose!(lp, convert(Array, D[reverse(I)...]))``.

    Per result chunk: every intersecting source piece is pulled (peer loads when it lives on another GPU) and written transposed
    by one kernel -- the fetched block is never materialised untransposed."""
    D = W.parent
    if isinstance(D, SparseDArray):
        refuse("copy(transpose(A))")
    rt = D.rt
    R = darray(lambda I: B200Array.empty(rt, shape_of(I), D.dtype), W.dims, procs=list(D.layout.pids), dtype=D.dtype, rt=rt)
    fenced = open_remote_reads(rt, [D], "host")
    es = D.dtype.itemsize
    conj = W.conj and D.dtype.kind == "c"                 # the adjoint of a real matrix is its transpose
    from .layout import slab_plan
    for pid, out in R.chunks.items():
        I = R.layout.localindices(pid)                    # ranges of the transposed array held here
        if out.size == 0:
            continue
        J = (I[1], I[0])                                   # D[reverse(I)...]
        dst_ld = rlen(I[0])
        for piece in slab_plan(D.layout, J):
            spid = D.layout.pids[piece.chunk]
            sshape = shape_of(D.layout.indices[piece.chunk])
            (sr, sc), (dr, dc) = piece.src, piece.dst       # source ranges inside the chunk, ranges inside the J-box (1-based)
            rows, cols = rlen(sr), rlen(sc)
            src = D.peer_ptr(spid) + ((sr[0] - 1) + (sc[0] - 1) * sshape[0]) * es
            # J-box element (r, c) -> out[c, r]
            dst = out.ptr + ((dc[0] - 1) + (dr[0] - 1) * dst_ld) * es
            if conj:
                _lib.call("dab_adjoint_box", rt.ctx, dab_dtype(D.dtype), C.c_void_p(dst), dst_ld, C.c_void_p(src), sshape[0], rows, cols)
            else:
                _lib.call("dab_transpose_box", rt.ctx, es, C.c_void_p(dst), dst_ld, C.c_void_p(src), sshape[0], rows, cols)
    close_remote_reads(rt, fenced, "host")
    return R


# ---- matrix-vector ------------------------------------------------------------------------------------------------------------------


def matvec_exchange_plan(L, ylayout, trans: bool, rank_of, my_rank: int):
    """Who ships which tile result where in ``mul!(y, A, x)``: tile (i, j) is computed by the rank holding ``procs(A)[i,j]``
    (``procs(A)[j,i]`` for the transposed product) and consumed by the rank holding ``y.pids[i]`` (reference src/linalg.jl:90-98,
    113-117).  Pure function of the layouts, so every rank derives the same matched send/recv lists (same (i, j) order on both
    sides of each pair -- NCCL matches grouped point-to-point calls between two ranks in issue order)."""
    g0, g1 = L.grid
    gi, gj = (g1, g0) if trans else (g0, g1)
    plan = {"owned": [], "local": [], "sends": [], "recvs": []}
    for i in range(gi):
        orank = rank_of(ylayout.pids[i])
        plen = rlen(ylayout.indices[i][0])
        if orank == my_rank:
            plan["owned"].append(i)
        for j in range(gj):
            trank = rank_of(L.pids[(j + i * g0) if trans else (i + j * g0)])
            if orank == my_rank and trank == my_rank:
                plan["local"].append((i, j, plen))
            elif orank == my_rank:
                plan["recvs"].append((i, j, plen, trank))
            elif trank == my_rank:
                plan["sends"].append((i, j, plen, orank))
    return plan


def _unwrap(A) -> Tuple[DArray, bool]:
    if isinstance(A, Transpose):
        return A.parent, True
    return A, False


def _refuse_sparse_matmat(M):
    if isinstance(M, SparseDArray):
        refuse("the product with a matrix (sparse x dense-matrix, SpMM)")


def _gemv_tile(rt: Runtime, code: int, trans: bool, ch: B200Array, x_ptr: int, r_ptr: int):
    """``R[i,j] = localpart(A)*xj`` / ``localpart(A)'*xj`` of a dense chunk: K9."""
    _lib.call("dab_gemv", rt.ctx, code, 1 if trans else 0, C.c_void_p(ch.ptr), ch.shape[0], ch.shape[1], C.c_void_p(x_ptr), C.c_void_p(r_ptr))


def _spmv_tile(rt: Runtime, code: int, trans: bool, ch, x_ptr: int, r_ptr: int):
    """The same tile product of a SparseMatrixCSC chunk: K18 (SparseArrays' loops, bit for bit)."""
    ch.matvec(trans, x_ptr, r_ptr)


def _x_block(rt: Runtime, x, lo: int, hi: int, dtype: np.dtype) -> B200Array:
    """``convert(localtype(x), x[lo:hi])`` on this rank's GPU: host vectors are sliced and uploaded, DVectors halo-fetched."""
    n = hi - lo + 1
    if isinstance(x, DArray):
        if x.dtype != dtype:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mul!: vector eltype {x.dtype} vs matrix eltype {dtype}")
        out = B200Array.empty(rt, (n,), dtype, temp=True)
        SubDArray(x, ((lo, hi),), (False,)).copy_to(out)
        return out
    h = np.ascontiguousarray(np.asarray(x)[lo - 1:hi], dtype=dtype)
    out = B200Array.empty(rt, (n,), dtype, temp=True)
    if n:
        out.copy_from_host(h, sync=True)
    return out


def mul_(y: DArray, A: Union[DArray, Transpose], x, alpha=1, beta=0) -> DArray:
    """``mul!(y::DVector, A::DMatrix, x::AbstractVector, α=1, β=0)`` (reference src/linalg.jl:78-118) and, for a
    ``Transpose``/``Adjoint`` wrapper, :120-167.  Error contract as the reference: DimensionMismatch when the contracted sizes
    differ, ArgumentError when y's cuts do not match the matrix cuts along the kept dim."""
    _refuse_complex("mul!", y, A, x)
    refuse_float16("mul!", y, A, x)
    M, trans = _unwrap(A)
    if isinstance(y, SparseDArray):
        refuse("mul! into it")
    if isinstance(x, (DArray, np.ndarray)) and len(np.shape(x) if not isinstance(x, DArray) else x.dims) == 2:
        _refuse_sparse_matmat(M)
        return mul_mat_(y, A, x, alpha, beta)
    if M.ndim != 2 or y.ndim != 1:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "mul!: y must be a DVector and A a DMatrix")
    rd, cd = (1, 0) if trans else (0, 1)
    xlen = x.dims[0] if isinstance(x, DArray) else int(np.shape(x)[0])
    if M.dims[cd] != xlen:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"DimensionMismatch: A has {M.dims[cd]} columns, x has length {xlen}")
    if list(y.layout.cuts[0]) != list(M.layout.cuts[rd]):
        raise _lib.ArgumentError(_lib.ERR_ARG, "cuts of output vector must match cuts of %s dimension of matrix" % ("second" if trans else "first"))
    dt = y.dtype
    if dt not in _GEMV_DTYPES or M.dtype != dt:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mul!: eltypes y={dt} A={M.dtype} (served: equal Float32/Float64/Int32/Int64)")
    rt = y.rt
    L = M.layout
    g0, g1 = L.grid
    gi, gj = (g1, g0) if trans else (g0, g1)             # y chunks, tiles per y chunk
    cuts_c = L.cuts[cd]
    isz, code = dt.itemsize, dab_dtype(dt)
    ypids = y.layout.pids
    remote_x = open_remote_reads(rt, [x] if isinstance(x, DArray) else [], "device")
    tile_product = _spmv_tile if isinstance(M, SparseDArray) else _gemv_tile     # chosen by the chunk type, as localpart(A)*xj dispatches

    def tile_pid(i, j):                                    # procs(A)[i,j]  /  procs(A)[j,i]
        return L.pids[(j + i * g0) if trans else (i + j * g0)]

    # ---- where the tile results are combined: on the owner of y's chunk i, a stack of gj slots of plen each
    st = exchange_stacks(rt, [rt.rank_of(p) for p in ypids], [rlen(ix[0]) * gj * isz for ix in y.layout.indices])
    my_tab = st.tables[rt.rank]

    # ---- R[i,j] = localpart(A) * xj on the tile owners (src/linalg.jl:90-98); a tile whose consumer is this rank is written straight
    # into its slot of the stack
    temps: List[B200Array] = []
    xblocks: Dict[int, B200Array] = {}
    remote: Dict[Tuple[int, int], int] = {}                # (i, j) -> the tile result shipped to another rank
    for j in range(gj):
        for i in range(gi):
            pid = tile_pid(i, j)
            if pid not in M.chunks:
                continue
            ch = M.chunks[pid]
            if j not in xblocks:
                xblocks[j] = _x_block(rt, x, cuts_c[j], cuts_c[j + 1] - 1, dt)
            plen = ch.shape[rd]
            orank = rt.rank_of(ypids[i])
            if orank == rt.rank:
                rptr = st.base + my_tab[i] + j * plen * isz
            else:
                r = B200Array.empty(rt, (plen,), dt, temp=True)
                temps.append(r)
                rptr = remote[i, j] = r.ptr
            tile_product(rt, code, trans, ch, xblocks[j].ptr, rptr)
    # ---- ship the tile results to the owner of y's chunk i (the fetch(rij) of :113-115); with the arena, the device fence this ends with
    # also means every reader of x is done with it
    if rt.world > 1:
        plan = matvec_exchange_plan(L, y.layout, trans, rt.rank_of, rt.rank)   # same (i, j) order on both sides of every pair
        deliver(rt, st, [(remote[i, j], plen * isz, peer, i, j * plen * isz) for i, j, plen, peer in plan["sends"]],
                [(peer, i, j * plen * isz, plen * isz) for i, j, plen, peer in plan["recvs"]])
    # ---- scale y (:101-111), then add!(localpart(y), R[i,j], α) for each j (:114-117; j order) -- one fused launch per y chunk
    a_s, b_s = np.asarray(alpha, dtype=dt), np.asarray(beta, dtype=dt)
    for i, off in my_tab.items():
        ych = y.chunks[ypids[i]]
        if ych.size:
            _lib.call("dab_accumulate_stack", rt.ctx, code, C.c_void_p(ych.ptr), ych.size, C.c_void_p(b_s.ctypes.data), C.c_void_p(a_s.ctypes.data),
                      C.c_void_p(st.base + off), ych.size, gj)
    for t in temps + list(xblocks.values()):
        t.free()
    if not st.use_arena:                                   # with the arena, the fence after the puts closed the reads of x
        rt.free_temp(st.temp)
        close_remote_reads(rt, remote_x, "device")
    return y


def matmul(A: Union[DArray, Transpose], x) -> DArray:
    """``A*x`` (reference src/linalg.jl:280-284): y lives on ``procs(A)[:,1]`` with one chunk per grid row; ``A'*x`` /
    ``transpose(A)*x`` (:293-301, 303-311): on ``procs(A)[1,:]``, one chunk per grid column.  Inside ``ppeval`` (a traced slice
    function) the product of slices is recorded for ``dab_matmul_batched`` instead."""
    from ._broadcast import Expr
    if isinstance(A, Expr) or isinstance(x, Expr):
        from ._slices import matmul_of_slices
        return matmul_of_slices(A, x)
    _refuse_complex("A*x", A, x)
    refuse_float16("A*x", A, x)
    M, trans = _unwrap(A)
    xnd = len(x.dims) if isinstance(x, DArray) else np.ndim(x)
    if xnd == 2:
        _refuse_sparse_matmat(M)
        return matmat(A, x)
    if xnd != 1:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "A*x: x must be a vector or a matrix")
    if M.ndim != 2:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "A must be a DMatrix")
    xdt = x.dtype if isinstance(x, DArray) else np.asarray(x).dtype
    T = np.result_type(M.dtype, xdt)                       # promote_op(t*s + t*s)
    if T != M.dtype:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"A*x: eltype {M.dtype} with a {xdt} vector needs a converted copy of A")
    g0, g1 = M.layout.grid
    rd = 1 if trans else 0
    pids = [M.layout.pids[j * g0] for j in range(g1)] if trans else [M.layout.pids[i] for i in range(g0)]
    rt = M.rt
    y = darray(lambda I: B200Array.empty(rt, shape_of(I), T), (M.dims[rd],), procs=pids, dist=[M.layout.grid[rd]], dtype=T, rt=rt)
    return mul_(y, A, x)


# ---- matrix-matrix ------------------------------------------------------------------------------------------------------------------


def matmat_exchange_plan(L, Clayout, trans: bool, rank_of, my_rank: int):
    """Who ships which tile result where in ``_matmatmul!``: R[i,j,k] is computed by the rank holding ``procs(A)[i,j]``
    (``procs(A)[j,i]`` for the transposed forms) and consumed by the rank holding ``C.pids[i,k]`` (reference src/linalg.jl:208-252).
    Pure function of the layouts; both sides of every pair list their transfers in the same (k, i, j) order.  Entries carry the tile
    shape (rows of C chunk i, columns of C chunk k)."""
    g0, g1 = L.grid
    gi, gj = (g1, g0) if trans else (g0, g1)
    c0, gk = Clayout.grid
    plan = {"owned": [], "local": [], "sends": [], "recvs": []}
    for k in range(gk):
        for i in range(gi):
            lin_c = i + k * c0
            orank = rank_of(Clayout.pids[lin_c])
            rows, cols = rlen(Clayout.indices[lin_c][0]), rlen(Clayout.indices[lin_c][1])
            if orank == my_rank:
                plan["owned"].append((i, k))
            for j in range(gj):
                trank = rank_of(L.pids[(j + i * g0) if trans else (i + j * g0)])
                if orank == my_rank and trank == my_rank:
                    plan["local"].append((i, j, k, rows, cols))
                elif orank == my_rank:
                    plan["recvs"].append((i, j, k, rows, cols, trank))
                elif trank == my_rank:
                    plan["sends"].append((i, j, k, rows, cols, orank))
    return plan


def _b_block(rt: Runtime, B, rlo: int, rhi: int, clo: int, chi: int, dtype: np.dtype) -> B200Array:
    """``convert(localtype(B), B[rlo:rhi, clo:chi])`` on this rank's GPU (src/linalg.jl:214, 221-225): host matrices are sliced and
    uploaded, DMatrices halo-fetched (peer loads when the block lives on other GPUs)."""
    shape = (rhi - rlo + 1, chi - clo + 1)
    if isinstance(B, DArray):
        if B.dtype != dtype:
            raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mul!: eltype of B {B.dtype} vs matrix eltype {dtype}")
        out = B200Array.empty(rt, shape, dtype, temp=True)
        if out.size:
            SubDArray(B, ((rlo, rhi), (clo, chi)), (False, False)).copy_to(out)
        return out
    h = np.asfortranarray(np.asarray(B)[rlo - 1:rhi, clo - 1:chi], dtype=dtype)
    out = B200Array.empty(rt, shape, dtype, temp=True)
    if out.size:
        out.copy_from_host(h, sync=True)
    return out


def mul_mat_(Cd: DArray, A: Union[DArray, Transpose], B, alpha=1, beta=0) -> DArray:
    """``mul!(C::DMatrix, A::DMatrix, B::AbstractMatrix, α=1, β=0)`` and the Adjoint / Transpose forms = ``_matmatmul!`` (reference
    src/linalg.jl:189-261).  Same errors as the reference: DimensionMismatch for the contracted / result sizes, ArgumentError when the
    cuts of C's first dimension differ from A's."""
    _refuse_complex("mul!", Cd, A, B)
    refuse_float16("mul!", Cd, A, B)
    M, trans = _unwrap(A)
    _refuse_sparse_matmat(M)
    if isinstance(Cd, SparseDArray) or isinstance(B, SparseDArray):
        refuse("mul! of matrices")
    if M.ndim != 2 or Cd.ndim != 2:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "mul!: C and A must be DMatrices")
    rd, cd = (1, 0) if trans else (0, 1)
    mA, nA = M.dims[rd], M.dims[cd]
    mB, nB = B.dims if isinstance(B, DArray) else tuple(np.shape(B))
    if mB != nA:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"matrix A has dimensions ({mA}, {nA}), matrix B has dimensions ({mB}, {nB})")
    if Cd.dims != (mA, nB):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"result C has dimensions {Cd.dims}, needs ({mA}, {nB})")
    if list(Cd.layout.cuts[0]) != list(M.layout.cuts[rd]):
        raise _lib.ArgumentError(_lib.ERR_ARG, "cuts of the first dimension of the output matrix must match cuts of dimension %d of the first input matrix" % (rd + 1))
    dt = Cd.dtype
    if dt not in _GEMV_DTYPES or M.dtype != dt:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"mul!: eltypes C={dt} A={M.dtype} (served: equal Float32/Float64/Int32/Int64)")
    rt = Cd.rt
    L, CL = M.layout, Cd.layout
    g0, g1 = L.grid
    gi, gj = (g1, g0) if trans else (g0, g1)
    c0, gk = CL.grid
    cuts_c, cuts_k = L.cuts[cd], CL.cuts[1]
    code, isz = dab_dtype(dt), dt.itemsize
    remote_b = open_remote_reads(rt, [B] if isinstance(B, DArray) else [], "host")

    def tile_pid(i, j):
        return L.pids[(j + i * g0) if trans else (i + j * g0)]

    # ---- R[i,j,k] = op(localpart(A)) * Bjk on the tile owners (src/linalg.jl:208-229)
    R: Dict[Tuple[int, int, int], B200Array] = {}
    temps: List[B200Array] = []
    for j in range(gj):
        for k in range(gk):
            bjk = None
            for i in range(gi):
                pid = tile_pid(i, j)
                if pid not in M.chunks:
                    continue
                ch = M.chunks[pid]
                if bjk is None:
                    bjk = _b_block(rt, B, cuts_c[j], cuts_c[j + 1] - 1, cuts_k[k], cuts_k[k + 1] - 1, dt)
                    temps.append(bjk)
                m_t, k_t, n_t = ch.shape[rd], ch.shape[cd], bjk.shape[1]
                r = B200Array.empty(rt, (m_t, n_t), dt, temp=True)
                if r.size:
                    _lib.call("dab_gemm", rt.ctx, code, 1 if trans else 0, m_t, n_t, k_t, C.c_void_p(ch.ptr), max(1, ch.shape[0]), C.c_void_p(bjk.ptr),
                              max(1, k_t), C.c_void_p(r.ptr), max(1, m_t))
                R[(i, j, k)] = r
    # ---- ship the tile results to the owner of C's chunk (i, k): one grouped exchange (the fetch(rijk) of :248-249)
    plan = matmat_exchange_plan(L, CL, trans, rt.rank_of, rt.rank)
    stacks: Dict[Tuple[int, int], B200Array] = {}
    for (i, k) in plan["owned"]:
        lin_c = i + k * c0
        stacks[(i, k)] = B200Array.empty(rt, (int(np.prod(shape_of(CL.indices[lin_c]))) * gj,), dt, temp=True)
    for i, j, k, rows, cols in plan["local"]:
        if rows * cols:
            _lib.call("dab_d2d", rt.ctx, C.c_void_p(stacks[(i, k)].ptr + j * rows * cols * isz), C.c_void_p(R[(i, j, k)].ptr), rows * cols * isz)
    sends = [(R[(i, j, k)].ptr, rows * cols * isz, peer) for i, j, k, rows, cols, peer in plan["sends"] if rows * cols]
    recvs = [(stacks[(i, k)].ptr + j * rows * cols * isz, rows * cols * isz, peer) for i, j, k, rows, cols, peer in plan["recvs"] if rows * cols]
    grouped_exchange(rt, sends, recvs)
    # ---- scale C (:232-240), then add!(localpart(C), R[i,j,k], α) for each j (:243-252; j order)
    a_s, b_s = np.asarray(alpha, dtype=dt), np.asarray(beta, dtype=dt)
    for (i, k), stack in stacks.items():
        cch = Cd.chunks[CL.pids[i + k * c0]]
        nel = cch.size
        if nel == 0:
            continue
        if beta != 1:
            if beta == 0:
                z = np.zeros((), dtype=dt)
                _lib.call("dab_fill", rt.ctx, code, C.c_void_p(cch.ptr), nel, C.c_void_p(z.ctypes.data))
            else:
                _lib.call("dab_binary_scalar", rt.ctx, code, _lib.MUL, C.c_void_p(cch.ptr), C.c_void_p(cch.ptr), C.c_void_p(b_s.ctypes.data), 0, nel)
        for j in range(gj):
            rp = stack.ptr + j * nel * isz
            if alpha != 1:
                _lib.call("dab_binary_scalar", rt.ctx, code, _lib.MUL, C.c_void_p(rp), C.c_void_p(rp), C.c_void_p(a_s.ctypes.data), 1, nel)
            _lib.call("dab_binary", rt.ctx, code, _lib.ADD, C.c_void_p(cch.ptr), C.c_void_p(cch.ptr), C.c_void_p(rp), nel)
    for t in list(R.values()) + temps + list(stacks.values()):
        t.free()
    close_remote_reads(rt, remote_b, "host")
    return Cd


def matmat(A: Union[DArray, Transpose], B) -> DArray:
    """``A*B`` (reference src/linalg.jl:285-292): C on ``procs(A)[:, 1:min(size(procs(A),2), size(procs(B),2))]`` with that grid;
    ``A'*B`` / ``transpose(A)*B`` (:302-311): on ``procs(A)[1:min(size(procs(A),1), size(procs(B),2)), :]`` with grid
    ``(size(procs(A),2), that min)``.  The reference asks ``procs(B)`` for its grid, so B is a DMatrix there; a host matrix is accepted
    here as a one-column grid (what ``distribute`` of a matrix no wider than tall gives on these workers)."""
    _refuse_complex("A*B", A, B)
    refuse_float16("A*B", A, B)
    M, trans = _unwrap(A)
    _refuse_sparse_matmat(M)
    if M.ndim != 2:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "A must be a DMatrix")
    bdt = B.dtype if isinstance(B, DArray) else np.asarray(B).dtype
    T = np.result_type(M.dtype, bdt)                       # promote_op(t*s + t*s)
    if T != M.dtype:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"A*B: eltype {M.dtype} with a {bdt} matrix needs a converted copy of A")
    bcols = B.dims[1] if isinstance(B, DArray) else np.shape(B)[1]
    bg1 = B.layout.grid[1] if isinstance(B, DArray) else 1
    g0, g1 = M.layout.grid
    pg = np.asarray(M.layout.pids).reshape((g0, g1), order="F")
    rt = M.rt
    if not trans:
        nc = min(g1, bg1)
        pids, dims, dist = [int(p) for p in pg[:, :nc].reshape(-1, order="F")], (M.dims[0], bcols), [g0, nc]
    else:
        nr = min(g0, bg1)
        pids, dims, dist = [int(p) for p in pg[:nr, :].reshape(-1, order="F")], (M.dims[1], bcols), [g1, nr]
    Cd = darray(lambda I: B200Array.empty(rt, shape_of(I), T), dims, procs=pids, dist=dist, dtype=T, rt=rt)
    return mul_mat_(Cd, A, B)


# ---- Diagonal scaling ---------------------------------------------------------------------------------------------------------------


def lmul_diag(d, DA: DArray) -> DArray:
    """``lmul!(D::Diagonal, DA::DMatrix)`` with ``d = D.diag`` (reference src/linalg.jl:169-177): DA[i,j] = d[i]*DA[i,j]."""
    from ._broadcast import broadcast_into
    _refuse_complex("lmul!(Diagonal, A)", d, DA)
    refuse_float16("lmul!(Diagonal, A)", d, DA)
    dv = np.asarray(d)
    if DA.ndim != 2 or dv.shape != (DA.dims[0],):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"lmul!: diagonal of length {dv.shape} vs matrix {DA.dims}")
    return broadcast_into(DA, lambda s, a: s * a, dv.astype(DA.dtype).reshape(-1, 1), DA)


def rmul_diag(DA: DArray, d) -> DArray:
    """``rmul!(DA::DMatrix, D::Diagonal)`` (reference src/linalg.jl:179-187): DA[i,j] = DA[i,j]*d[j]."""
    from ._broadcast import broadcast_into
    _refuse_complex("rmul!(A, Diagonal)", DA, d)
    refuse_float16("rmul!(A, Diagonal)", DA, d)
    dv = np.asarray(d)
    if DA.ndim != 2 or dv.shape != (DA.dims[1],):
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"rmul!: diagonal of length {dv.shape} vs matrix {DA.dims}")
    return broadcast_into(DA, lambda a, s: a * s, DA, dv.astype(DA.dtype).reshape(1, -1))
