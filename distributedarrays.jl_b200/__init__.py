"""distributedarrays.jl_b200 -- H100-native backend for the DArray map!/broadcast + mapreduce hot path.

Import it as ``darray_b200`` (the directory name is not a Python identifier; ``darray_b200.py`` at the repo root is a
loader shim).  The public names mirror DistributedArrays.jl's for this path: ``DArray``, ``distribute``, ``localpart``,
``localindices``, ``locate``, ``makelocal``, ``procs``, ``dzeros/dones/dfill/drand``, ``map`` (``map_``), ``map!``
(``map_inplace``), broadcast (``broadcast`` / ``broadcast_into``), ``reduce``, ``mapreduce``, ``sum``, ``prod``,
``maximum``, ``minimum``, ``all``, ``any``, ``count``, ``extrema``, ``findmax`` / ``findmin`` / ``argmax`` / ``argmin`` (with and without
``dims``), ``sort`` and ``sortperm`` of a DVector (``sortperm(d; sample, by)``: stable, 1-based, the layout of ``sort``) and along a
dimension (``sortperm(A; dims, by)``: 1-based global linear indices per fibre, stable; ``sort(A; dims, by)``; segmented sorts on the GPU),
``mapslices`` (with ``sort``, ``svdvals``, ``eigvals``, reductions,
elementwise and constant slice functions), ``ppeval`` (batched slice products ``ppeval(operator.matmul, A, B)``, ``eigvals`` of symmetric
slices, solves ``ppeval(ldiv, A, B)`` (Julia's ``A \\ B``) and determinants ``ppeval(det, A)`` / ``mapslices(det, D, dims)``, and every
``mapslices`` slice function), ``cumsum`` / ``cumprod`` / ``accumulate`` and their ``!`` forms
(``cumsum_`` ...), ``Array(d)`` (``to_array``), range ``getindex``, ``permutedims(A, perm)`` /
``permutedims(A)`` / ``permutedims_(dest, src, perm)`` (Julia's ``permutedims!``; 1-based ``perm``, N-d, a tiled permutation on the GPU),
``d[I]`` with ``I`` a DArray of Int32 / Int64 (a gather on the GPU:
``v[sortperm(v)]``, ``A[findmax(A; dims)[2]]``; a DArray key holds Julia's 1-based linear indices, host Python indices stay 0-based),
logical indexing ``d[mask]`` with a Bool DArray of ``d``'s dims, ``findall(mask)`` / ``findall(f, d)`` (1-based linear indices as a
``DArray{Int64}``) and ``filter(f, d)`` (stream compaction on the GPU; results are DVectors in column-major order); ``d[key] = v`` for
every key ``d[key]`` takes, and ``copyto(view, src)`` (a scatter on the GPU for a DArray key, the last occurrence of a repeated index
winning as in Julia's sequential ``setindex!``; ``d[mask] = v`` as the inverse of compaction; a scalar, host array or DArray value); sparse DArrays (``distribute`` of a scipy.sparse matrix: CSC
localparts, ``nnz``, ``A*x`` / ``A'*x`` / ``mul!``).

Element types: Float32, Float64, Int32, Int64, Bool, ComplexF32, ComplexF64 and Float16 (``np.float16``: storage, data movement,
elementwise arithmetic with Julia's "widen to Float32, operate, round to Float16" semantics, ``Float16(x)`` inside kernels, and
reductions with and without ``dims``; GEMM / GEMV, sort, scans, findmax, ``d[I::DArray]`` / ``d[mask]`` / ``filter`` and the
``d[key] = v`` forms built on them, ``mapslices``, ``ppeval`` and sparse matrices refuse it with ``UnsupportedError``).

Everything computes on the GPU through ``csrc/libdab200.so`` (C ABI: ``include/dab200.h``).  There is no CPU fallback:
importing works anywhere, but the first op without the built extension or without an H100 raises.
"""
from . import _lib
from ._lib import ArgumentError, DabError, DimensionMismatch, InexactError, SingularException, UnsupportedError
from ._broadcast import (Expr, Int128, abs2, broadcast, broadcast_into, ceil, copy, cos, deepcopy, drandn, exp, floor, ifelse, inv, isnan, jl_max, jl_min,
                        log, map_, map_bang, map_inplace, map_localparts, mod, rem, sign, sin, sqrt, tan, tanh, widen)
from ._broadcast import angle, cis, conj, imag, iszero, real  # noqa: F401 -- complex values (complex(x[, y]) below)
from ._broadcast import Float16  # noqa: F401 -- Float16(x) inside a kernel
from ._broadcast import complex_ as complex  # noqa: A004
from ._broadcast import (acos, acosh, acot, acoth, acsc, acsch, asec, asech, asin, asinh, atan, atanh, cbrt, cosh, cospi, cot, coth, csc,  # noqa: F401
                        csch, deg2rad, erf, erfc, erfcinv, erfcx, erfinv, exp10, exp2, expm1, gamma, isfinite, isinf, log10, log1p, log2,
                        loggamma, rad2deg, round_, sec, sech, sinh, sinpi, trunc)
from ._darray import (B200Array, DArray, SubDArray, allowscalar, dab_dtype, np_dtype, copyto, d_closeall, darray, darray_from_chunks, darray_like,
                     dfill, distribute, dones, drand, dzeros, fill_, localindices, localpart, locate, makelocal, pinned_empty, procs,
                     registry_size, reshape, similar, to_array)
from .layout import Layout, chunk_idxs, cuts_for, defaultdist, make_layout, slab_plan
from ._mapreduce import (all, any, axpy_, count, dot, extrema, isequal, mapreduce, mapreducedim, maximum, mean, minimum, nnz, norm,  # noqa: A004
                         prod, reduce, rmul_, sum)
from ._linalg import Adjoint, Transpose, adjoint, copy_transposed, lmul_diag, matmat, matmul, mul_, mul_mat_, rmul_diag, transpose
from ._findmax import argmax, argmin, findmax, findmin
from ._compact import filter, findall  # noqa: A004
from ._sort import sort, sort_with_boundaries, sortperm
from ._scan import accumulate, accumulate_, cumprod, cumprod_, cumsum, cumsum_
from ._slices import det, eigvals, ldiv, mapslices, svdvals
from ._ppeval import ppeval
from ._permute import permutedims, permutedims_
from ._sparse import SparseChunk, SparseDArray
from .runtime import Runtime, init, myid, nworkers, runtime, workers

__all__ = [n for n in dir() if not n.startswith("_")]
