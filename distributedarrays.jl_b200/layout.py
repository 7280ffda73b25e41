"""Layout math of a DArray: which block of the global array each worker (GPU) owns.

Host-side integer logic, bit-exact with the reference (DistributedArrays.jl v0.6.9):
``defaultdist`` (src/darray.jl:251-296), ``chunk_idxs`` (:299-307), ``locate`` (:448-456), the layout derived from
a grid of chunks (``DArray(refs)``, :183-216) and the slab/chunk intersection algebra of ``setindex!(::Array,
::SubDArray)`` (:798-820) restricted to unit ranges.  Indices are 1-based inclusive ranges ``(lo, hi)`` exactly as the
reference stores them, so that ``d.indices`` / ``d.cuts`` can be compared verbatim with the reference's.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

Range = Tuple[int, int]


def _distinct_primes_desc(n: int) -> List[int]:
    ps, q = [], 2
    while q * q <= n:
        if n % q == 0:
            ps.append(q)
            while n % q == 0:
                n //= q
        q += 1 if q == 2 else 2
    if n > 1:
        ps.append(n)
    return ps[::-1]


def defaultdist(dims: Sequence[int], npids: int) -> Tuple[int, ...]:
    """Grid shape for ``npids`` workers (reference src/darray.jl:251-276): the largest remaining prime factor of the
    worker count goes to the currently largest dimension, ties to the highest dimension."""
    rem_dims = [int(d) for d in dims]
    grid = [1] * len(rem_dims)
    primes = _distinct_primes_desc(npids)
    left, k = npids, 0
    while left > 1:
        if left % primes[k]:
            k += 1
            if k == len(primes):
                break
        fac = primes[k]
        big = max(rem_dims)
        where = len(rem_dims) - 1 - rem_dims[::-1].index(big)  # findlast
        if rem_dims[where] >= fac:
            rem_dims[where] //= fac
            grid[where] *= fac
        left //= fac
    return tuple(grid)


def cuts_for(sz: int, nc: int) -> List[int]:
    """First index of each of ``nc`` chunks of a dimension of size ``sz`` plus the end sentinel
    (reference src/darray.jl:279-296); the first ``sz % nc`` chunks are one longer."""
    if sz < nc:
        return list(range(1, sz + 2)) + [0] * (nc - sz)
    q, r = divmod(sz, nc)
    return [i * q + min(i, r) + 1 for i in range(nc + 1)]


def chunk_idxs(dims: Sequence[int], grid: Sequence[int]):
    """(indices, cuts) as in reference src/darray.jl:299-307.  ``indices`` is a list in column-major grid order."""
    cuts = [cuts_for(int(d), int(g)) for d, g in zip(dims, grid)]
    idx = []
    for lin in range(int(np.prod(grid)) if len(grid) else 1):
        c = unravel(lin, grid)
        # Julia normalises an empty UnitRange a:b (b < a-1) to a:a-1
        idx.append(tuple((cuts[k][c[k]], max(cuts[k][c[k]] - 1, cuts[k][c[k] + 1] - 1)) for k in range(len(dims))))
    return idx, cuts


def unravel(lin: int, shape: Sequence[int]) -> Tuple[int, ...]:
    """0-based column-major multi-index."""
    out = []
    for s in shape:
        out.append(lin % s)
        lin //= s
    return tuple(out)


def ravel(idx: Sequence[int], shape: Sequence[int]) -> int:
    lin, mul = 0, 1
    for i, s in zip(idx, shape):
        lin += i * mul
        mul *= s
    return lin


def rlen(r: Range) -> int:
    return max(0, r[1] - r[0] + 1)


def shape_of(idx: Sequence[Range]) -> Tuple[int, ...]:
    return tuple(rlen(r) for r in idx)


@dataclass
class Layout:
    """The metadata fields of the reference's ``DArray`` struct (src/darray.jl:25-31) minus id/localpart."""

    dims: Tuple[int, ...]
    grid: Tuple[int, ...]            # size(pids)
    pids: List[int]                  # vec(pids), column-major == procs(d)
    indices: List[Tuple[Range, ...]]  # vec(indices)
    cuts: List[List[int]]

    @property
    def ndim(self) -> int:
        return len(self.dims)

    def chunk_of_pid(self, pid: int) -> int:
        """``localpartindex`` (src/darray.jl:309-318): 0-based chunk number of ``pid`` or -1."""
        try:
            return self.pids.index(pid)
        except ValueError:
            return -1

    def localindices(self, pid: int) -> Tuple[Range, ...]:
        """src/darray.jl:394-400."""
        c = self.chunk_of_pid(pid)
        return self.indices[c] if c >= 0 else tuple((1, 0) for _ in self.dims)

    def locate(self, *I: int) -> Tuple[int, ...]:
        """1-based grid index of the chunk holding element ``I`` (src/darray.jl:448-456)."""
        out = []
        for c, i in zip(self.cuts, I):
            fi = int(np.searchsorted(np.asarray(c), i, side="right"))
            if fi >= len(c):
                raise ValueError("ArgumentError: element not contained in array")
            out.append(fi)
        return tuple(out)

    def same_as(self, other: "Layout") -> bool:
        return self.dims == other.dims and self.grid == other.grid and self.pids == other.pids and self.indices == other.indices


def make_layout(dims: Sequence[int], pids: Sequence[int], dist: Optional[Sequence[int]] = None) -> Layout:
    """``DArray(init, dims, procs[, dist])`` (src/darray.jl:159-173)."""
    dims = tuple(int(d) for d in dims)
    if len(pids) == 0:
        raise ValueError("ArgumentError: no processors given")
    grid = tuple(int(g) for g in dist) if dist is not None else defaultdist(dims, len(pids))
    if len(grid) != len(dims):
        raise ValueError("ArgumentError: dist must have one entry per dimension")
    n = int(np.prod(grid))
    if n > len(pids):
        raise ValueError("ArgumentError: dist needs more workers than given")
    idx, cuts = chunk_idxs(dims, grid)
    return Layout(dims, grid, list(pids)[:n], idx, cuts)


def layout_from_chunk_shapes(shapes: Sequence[Sequence[int]], grid: Sequence[int], pids: Sequence[int]) -> Layout:
    """``DArray(refs)`` (src/darray.jl:183-216): irregular layout derived from the chunk sizes, given in
    column-major grid order."""
    grid = tuple(int(g) for g in grid)
    nd = len(grid)
    idx = []
    for lin in range(len(shapes)):
        c = unravel(lin, grid)
        rng = []
        for x in range(nd):
            start = 1
            for j in range(c[x]):
                prev = list(c)
                prev[x] = j
                start += int(shapes[ravel(prev, grid)][x])
            rng.append((start, start + int(shapes[lin][x]) - 1))
        idx.append(tuple(rng))
    cuts = [[1] + sorted({i[x][1] + 1 for i in idx}) for x in range(nd)]
    dims = tuple(c[-1] - 1 for c in cuts)
    return Layout(dims, grid, list(pids), idx, cuts)


def default_procs(dims: Sequence[int], workers: Sequence[int]) -> List[int]:
    """``workers()[1:min(nworkers(), maximum(dims))]`` (src/darray.jl:174, 545)."""
    return list(workers)[: min(len(workers), max(int(d) for d in dims))]


@dataclass
class SlabPiece:
    chunk: int                       # 0-based chunk number (owner = layout.pids[chunk])
    src: Tuple[Range, ...]           # 1-based ranges inside the owner's localpart
    dst: Tuple[Range, ...]           # 1-based ranges inside the dense destination array
    whole_chunk: bool                # reference fetches chunk(d, pid) instead of a sub-slab (src/darray.jl:809-811)


def slab_plan(layout: Layout, J: Sequence[Range]) -> List[SlabPiece]:
    """Which chunks a unit-range view ``d[J...]`` touches and where each piece lands
    (``K = J ∩ K_c`` and the index bookkeeping of reference src/darray.jl:804-815)."""
    out = []
    for c, Kc in enumerate(layout.indices):
        K = tuple((max(j[0], k[0]), min(j[1], k[1])) for j, k in zip(J, Kc))
        if any(rlen(r) == 0 for r in K):
            continue
        src = tuple((k[0] - kc[0] + 1, k[1] - kc[0] + 1) for k, kc in zip(K, Kc))
        dst = tuple((k[0] - j[0] + 1, k[1] - j[0] + 1) for k, j in zip(K, J))
        out.append(SlabPiece(c, src, dst, all(a == b for a, b in zip(K, Kc))))
    return out


def contains(outer: Sequence[Range], inner: Sequence[Range]) -> bool:
    """``checkbounds_indices(Bool, lidcs, J)`` for unit ranges (makelocal's locality test, src/darray.jl:356-357)."""
    return all(rlen(j) == 0 or (o[0] <= j[0] and j[1] <= o[1]) for o, j in zip(outer, inner))


def collapse_for_region(shape: Sequence[int], region: Sequence[int]):
    """Split a column-major chunk shape into maximal runs of kept / reduced dims.  Returns a list of
    (is_reduced, extent) runs, first dim first.  A reduction over ``region`` (1-based dims) is then a sequence of
    (inner, reduce, outer) passes, one per reduced run."""
    runs = []
    for k, s in enumerate(shape):
        red = (k + 1) in region
        if runs and runs[-1][0] == red:
            runs[-1][1] *= int(s)
        else:
            runs.append([red, int(s)])
    return [(r, e) for r, e in runs]


def reduction_passes(shape: Sequence[int], region: Sequence[int]):
    """Yield the ``(inner, reduce, outer)`` kernel passes of a reduction of a column-major chunk over ``region`` (1-based dims):
    one per maximal run of reduced dims, last run first, so that ``inner`` is always the untouched prefix.  Each pass sees the
    extents the passes before it left (their runs collapsed to 1)."""
    runs = collapse_for_region(shape, set(region))
    ext = [e for _, e in runs]
    for ri in range(len(runs) - 1, -1, -1):
        if runs[ri][0]:
            yield int(np.prod(ext[:ri])), ext[ri], int(np.prod(ext[ri + 1:]))
            ext[ri] = 1
