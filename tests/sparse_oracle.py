"""TEST INFRASTRUCTURE -- a model of SparseArrays' matrix-vector loops and of the distributed ``mul!`` around them, for sparse DArrays.

The loops below are stated from memory of the SparseArrays sources; there is no Julia installation here to confirm them against, so they
are this project's reading of those loops, not a transcript:

* ``A*x`` (``_spmatmul!``): ``C`` is zero-filled; for each ``col`` in ascending order, ``αxj = x[col]*true``, then for each stored ``j`` of the
  column, ``C[rv[j]] += nzv[j]*αxj``.  Each output row therefore folds its entries in ascending column order, from zero.
* ``A'*x`` (``_At_or_Ac_mul_B!``): for each ``col``, ``tmp = zero(T)``, ``tmp += nzv[j]*x[rv[j]]`` over the column in storage order, then
  ``C[col] += tmp*true``.

For a real ``T`` both are "fold from +0.0 in T, in column order, every product and add rounded on its own" (``x*true`` is ``x``, and
``0 + tmp`` is ``tmp`` because ``tmp`` is never -0.0).  The reference's ``mul!`` (src/linalg.jl:78-167) then fills ``y`` with zero or scales
it by β and adds ``α*R[i,j]`` in ``j`` order.  NumPy float32 / float64 adds and multiplies round once per operation; Int32 / Int64 wrap
(computed on the unsigned views).  The folds are vectorised across rows: step ``t`` adds the ``t``-th entry of every row that has one.
"""
from __future__ import annotations

import numpy as np

_U = {np.dtype(np.int32): np.uint32, np.dtype(np.int64): np.uint64}


def _carrier(a: np.ndarray) -> np.ndarray:
    return a.view(_U[a.dtype]) if a.dtype in _U else a


def fold_groups(starts: np.ndarray, lens: np.ndarray, terms: np.ndarray) -> np.ndarray:
    """``out[g] = ((0 + terms[s]) + terms[s+1]) + ...`` over ``terms[starts[g] : starts[g] + lens[g]]``, sequentially, for every group ``g``.
    ``terms`` are already in the carrier (unsigned for integers)."""
    G = len(lens)
    out = np.zeros(G, dtype=terms.dtype)
    if G == 0 or terms.size == 0:
        return out
    order = np.argsort(-lens, kind="stable")                      # longest first: the rows alive at step t are a prefix
    ls, ss = lens[order], starts[order]
    acc = np.zeros(G, dtype=terms.dtype)
    alive = G
    with np.errstate(all="ignore"):
        for t in range(int(ls[0])):
            while alive and ls[alive - 1] <= t:
                alive -= 1
            acc[:alive] = acc[:alive] + terms[ss[:alive] + t]
    out[order] = acc
    return out


def fold_rows(ptr: np.ndarray, idx: np.ndarray, val: np.ndarray, x: np.ndarray) -> np.ndarray:
    """K18's contract: ``out[r] = fold(+, val[p]*x[idx[p]])`` over ``p in ptr[r] : ptr[r+1]-1`` from zero, in ``T``."""
    ptr = np.asarray(ptr, dtype=np.int64)
    v, xv = _carrier(np.ascontiguousarray(val)), _carrier(np.ascontiguousarray(x))
    with np.errstate(all="ignore"):
        terms = v[ptr[0]:ptr[-1]] * xv[np.asarray(idx[ptr[0]:ptr[-1]], dtype=np.int64)] if ptr[-1] > ptr[0] else v[:0]
    out = fold_groups(ptr[:-1] - ptr[0], np.diff(ptr), terms)
    return out.view(val.dtype) if val.dtype in _U else out


def canonical_triplets(S):
    """(rows, cols, vals) of a scipy sparse matrix in column-major storage order, duplicates summed in storage order, stored zeros kept."""
    C = S.tocsc()
    r = np.asarray(C.indices, dtype=np.int64)[:C.indptr[-1]]
    c = np.repeat(np.arange(C.shape[1], dtype=np.int64), np.diff(C.indptr))
    v = np.asarray(C.data)[:C.indptr[-1]].copy()
    order = np.lexsort((r, c))
    r, c, v = r[order], c[order], v[order]
    first = np.ones(r.size, dtype=bool)
    first[1:] = (r[1:] != r[:-1]) | (c[1:] != c[:-1])
    out = v[first].copy()
    with np.errstate(all="ignore"):
        np.add.at(out, (np.cumsum(first) - 1)[~first], v[~first])
    return r[first], c[first], out


def tile(trip, I):
    """Entries of chunk ``I`` (1-based inclusive ranges) with local indices, column-major order."""
    r, c, v = trip
    (r0, r1), (c0, c1) = I
    k = (r >= r0 - 1) & (r <= r1 - 1) & (c >= c0 - 1) & (c <= c1 - 1)
    return r[k] - (r0 - 1), c[k] - (c0 - 1), v[k]


def tile_matvec(t, shape, x: np.ndarray, trans: bool) -> np.ndarray:
    """``localpart(A)*x`` (``_spmatmul!``: rows folded in column order) or ``localpart(A)'*x`` (columns folded in storage order)."""
    r, c, v = t
    m, n = shape
    if trans:
        key, other, nout = c, r, n
    else:
        key, other, nout = r, c, m
    order = np.lexsort((c, key))                                   # by output index, then column (= storage order within a column)
    key, other, vv = key[order], other[order], v[order]
    lens = np.bincount(key, minlength=nout).astype(np.int64)
    starts = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int64)
    vc, xc = _carrier(np.ascontiguousarray(vv)), _carrier(np.ascontiguousarray(x))
    with np.errstate(all="ignore"):
        terms = vc * xc[other]
    out = fold_groups(starts, lens, terms)
    return out.view(v.dtype) if v.dtype in _U else out


def mul_model(trip, dims, cuts, x, trans: bool, alpha=1, beta=0, y0=None):
    """The reference's ``mul!(y, A, x, α, β)`` with SparseArrays' tile products: ``cuts`` are the layout's (1-based) cuts of A; returns
    the dense result vector."""
    dt = np.asarray(trip[2]).dtype
    rc, cc = cuts
    ocuts, icuts = (cc, rc) if trans else (rc, cc)
    nout = dims[1] if trans else dims[0]
    y = np.zeros(nout, dtype=dt) if y0 is None else np.asarray(y0, dtype=dt).copy()
    a, b = _carrier(np.asarray([alpha], dtype=dt)), _carrier(np.asarray([beta], dtype=dt))
    for i in range(len(ocuts) - 1):
        lo, hi = ocuts[i] - 1, ocuts[i + 1] - 1
        with np.errstate(all="ignore"):
            acc = _carrier(y[lo:hi].copy())
            if beta == 0:
                acc = np.zeros_like(acc)
            elif beta != 1:
                acc = acc * b[0]
            for j in range(len(icuts) - 1):
                jlo, jhi = icuts[j] - 1, icuts[j + 1] - 1
                I = ((jlo + 1, jhi), (lo + 1, hi)) if trans else ((lo + 1, hi), (jlo + 1, jhi))
                shape = (I[0][1] - I[0][0] + 1, I[1][1] - I[1][0] + 1)
                R = _carrier(tile_matvec(tile(trip, I), shape, np.asarray(x, dtype=dt)[jlo:jhi], trans))
                acc = acc + (R * a[0] if alpha != 1 else R)
        y[lo:hi] = acc.view(dt) if dt in _U else acc
    return y


def same_bits(got: np.ndarray, want: np.ndarray) -> bool:
    """Bit-identical, except that NaN payloads are not compared (every NaN equals every NaN)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return bool(np.array_equal(got, want))
    gn, wn = np.isnan(got), np.isnan(want)
    u = np.uint32 if got.dtype.itemsize == 4 else np.uint64
    return bool(np.array_equal(gn, wn) and np.array_equal(got[~gn].view(u), want[~wn].view(u)))


def csc_to_csr(m: int, colptr: np.ndarray, rowval: np.ndarray, nzval: np.ndarray):
    """The row-major copy K19 must produce: rows ascending, columns ascending within each row (a stable sort by row of the column-major
    entries)."""
    n = len(colptr) - 1
    cols = np.repeat(np.arange(n, dtype=np.int64), np.diff(colptr))
    order = np.argsort(np.asarray(rowval, dtype=np.int64), kind="stable")
    rowptr = np.zeros(m + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum(np.bincount(np.asarray(rowval, dtype=np.int64), minlength=m))
    return rowptr, cols[order].astype(np.int32), np.asarray(nzval)[order]
