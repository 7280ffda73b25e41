"""``sort(d::DVector; sample=...)``: the reference's samplesort (src/sort.jl) with every data-sized step on the GPU.

Reference step                                                   here
---------------------------------------------------------------  ------------------------------------------------------------------
``sort(localpart(d))`` on every worker (:8, :22)                  K11 ``dab_sort`` (LSD radix sort of the chunk)
``sorted[collect(1:div(llp,ss):llp)]`` sample, ss = min(512,llp)  strided ``dab_copy_box`` gather + D2H of <= 1023 keys per worker
sort the samples, pick ``np`` boundaries (:66-88, :127-155)        host (a few hundred keys; identical index arithmetic)
scan each sorted chunk for the first ``x > boundaries[i+1]``       ``dab_sorted_split`` (binary searches on the device)
``put!`` piece i into worker i's RemoteChannel (:42-48)            one grouped NCCL send/recv (device-to-device inside a rank)
``sort!(lp_sorting)`` of what a worker received (:52-61)           K11 again
``DArray(local_sorted_refs)`` without the empty parts (:163-169)   irregular layout from the received sizes

The result is bit-identical to the reference's for NaN-free input (a sorted vector has one representation once -0.0 < +0.0 is
fixed); chunk sizes follow from the same boundaries, so the layout matches too.  NaNs sort last; inside the NaN block the
reference keeps input order, the radix sort orders by payload.

``sort(d; by = f)`` (``:by`` is accepted at src/sort.jl:111 and travels in ``kwargs...`` to every local sort, :8, :22, :61, and to the
sort of the gathered samples, :77; the split compares ``by(x) > by(boundaries[i+1])``, :32): ``f`` is traced like a broadcast
closure, ``keys = f.(chunk)`` is ONE fused elementwise kernel, ``dab_sort_by_key`` orders the values stably by those keys (K11 on
packed key|position words), the split runs on ``f.(sorted chunk)``, and the few hundred samples / boundaries get their keys from the
same kernel so that host and device agree bit for bit on ``f``.

``sortperm(d; sample, by)`` (no reference method) runs the same samplesort (``_samplesort``) with K21 ``dab_sort_pairs`` as both local
sorts: every key carries its 1-based global index, the Int64 index plane travels with the keys by the same exchange plan, and the result
holds the indices.  Stable (equal keys and all NaNs keep ascending index order), in ``sort``'s layout.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List

import numpy as np

from . import _lib
from ._darray import B200Array, DArray, dab_dtype
from .layout import layout_from_chunk_shapes
from .runtime import grouped_exchange

_SORT_DTYPES = (np.dtype(np.float32), np.dtype(np.float64), np.dtype(np.int32), np.dtype(np.int64))
SAMPLE_SIZE_ON_WORKER = 512                                    # src/sort.jl:69


class _SampleDefault:
    """``sample`` not given: ``true`` for a DVector; told apart from an explicit ``sample``, which is refused together with ``dims``."""

    def __repr__(self):
        return "true"


_SAMPLE_DEFAULT = _SampleDefault()


def _typemin(dt):
    return -np.inf if dt.kind == "f" else np.iinfo(dt).min


def _typemax(dt):
    return np.inf if dt.kind == "f" else np.iinfo(dt).max


def _host_sort(v: np.ndarray) -> np.ndarray:
    """isless order for the (tiny) sample vector."""
    if v.dtype.kind != "f":
        return np.sort(v, kind="stable")
    nan = np.isnan(v)
    body = v[~nan]
    return np.concatenate([body[np.lexsort((~np.signbit(body), body))], v[nan]])


def boundaries_from_samples(samples: np.ndarray, nparts: int, dt: np.dtype) -> np.ndarray:
    """src/sort.jl:78-85 and :149-153."""
    s = _host_sort(np.asarray(samples).astype(dt)).copy()
    if len(s) == 0:
        raise _lib.ArgumentError(_lib.ERR_ARG, "sort: empty sample")
    s[0] = _typemin(dt)
    step = len(s) // nparts
    b = [s[(x - 1) * step] for x in range(1, nparts + 1)]
    b.append(_typemax(dt))
    return np.asarray(b, dtype=dt)


def uniform_sample(lb, ub, nparts: int, dt: np.dtype) -> np.ndarray:
    """The ``sample::Tuple`` branch, src/sort.jl:127-145."""
    if not lb <= ub:
        raise AssertionError("AssertionError: lb <= ub")
    if isinstance(lb, np.float32) and isinstance(ub, np.float32):
        part = np.float32(abs(ub - lb)) / np.float32(nparts)
        vals = [np.float32(lb + np.float32(n) * part) for n in range(nparts)]
    else:
        if dt.kind == "f" or not (isinstance(lb, (int, np.integer)) and isinstance(ub, (int, np.integer))):
            part = abs(float(ub) - float(lb)) / nparts
        else:  # abs(ub - lb) in T's wrap-around machine arithmetic (a full-range Int sample overflows, as in the reference)
            bits = 8 * dt.itemsize
            diff = (int(ub) - int(lb) + (1 << (bits - 1))) % (1 << bits) - (1 << (bits - 1))
            part = float(diff if diff == -(1 << (bits - 1)) else abs(diff)) / nparts
        vals = [float(lb) + n * part for n in range(nparts)]
    if np.isnan(part) or np.isinf(part):
        raise _lib.ArgumentError(_lib.ERR_ARG, "lower and upper bounds must not be infinities")
    if dt.kind != "f":
        vals = [np.rint(v) for v in vals]
    return np.asarray(vals).astype(dt)


def _sort_chunk(rt, src_ptr: int, n: int, dt: np.dtype, out: B200Array):
    tmp = B200Array.empty(rt, (n,), dt, temp=True) if n > 1024 or src_ptr == out.ptr else None
    _lib.call("dab_sort", rt.ctx, dab_dtype(dt), C.c_void_p(src_ptr), C.c_void_p(out.ptr), C.c_void_p(tmp.ptr if tmp else None), n)
    if tmp is not None:
        tmp.free()


class _KeyFn:
    """``by`` traced once for the element type of ``d``: the expression tree, the key dtype, and the launches that use it."""

    def __init__(self, rt, by, dt: np.dtype):
        from . import _broadcast as bc
        self.rt, self.bc, self.vtag = rt, bc, bc.tag_of(dt)
        e = bc.trace(by, [self.vtag])
        if e.jt == "bool":
            e = bc.convert(e, "i32")                            # false < true: order Bool keys as 0 / 1
        self.expr = e
        self.kdt = np.dtype(bc._NPT[e.jt])                      # Float32 Float64 Int32 Int64: the key types dab_sort_by_key serves

    def keys_of(self, vals: B200Array) -> B200Array:
        """``by.(vals)`` on the device (one fused elementwise launch), as a temporary."""
        keys = B200Array.empty(self.rt, vals.shape, self.kdt, temp=True)
        self.bc.run_local(self.rt, self.expr, keys, [self.bc.LocalArg(arr=vals, tag=self.vtag)])
        return keys

    def keys_of_host(self, vals: np.ndarray) -> np.ndarray:
        """``by.(vals)`` for a small host vector (samples, boundaries), computed by the same kernel as the chunks' keys."""
        vals = np.ascontiguousarray(vals)
        if vals.size == 0:
            return np.empty(0, dtype=self.kdt)
        dv = B200Array.from_numpy(self.rt, vals)
        dk = self.keys_of(dv)
        out = dk.to_numpy()
        dk.free()
        dv.free()
        return out

    def sort_chunk(self, src: B200Array, out: B200Array):
        """``out = sort(src; by)``: values ordered stably by their keys."""
        n = src.size
        if n == 0:
            return
        keys = self.keys_of(src)
        need = C.c_size_t()
        _lib.check(_lib.lib().dab_sort_by_key_scratch_bytes(dab_dtype(self.kdt), n, C.byref(need)))
        scratch = B200Array.empty(self.rt, (need.value,), np.uint8, temp=True)
        _lib.call("dab_sort_by_key", self.rt.ctx, dab_dtype(self.kdt), C.c_void_p(keys.ptr), src.dtype.itemsize, C.c_void_p(src.ptr),
                  C.c_void_p(out.ptr), C.c_void_p(scratch.ptr), need.value, n)
        scratch.free()
        keys.free()


def key_order(keys: np.ndarray) -> np.ndarray:
    """Permutation of a stable ``isless`` sort of a (tiny) host key vector: -0.0 before +0.0, NaNs last in input order."""
    k = np.asarray(keys)
    if k.dtype.kind != "f":
        return np.argsort(k, kind="stable")
    nan = np.isnan(k)
    return np.lexsort((~np.signbit(k) & ~nan, np.where(nan, 0, k), nan))


def boundaries_from_samples_by(samples: np.ndarray, sample_keys: np.ndarray, nparts: int, dt: np.dtype) -> np.ndarray:
    """src/sort.jl:77-85 with ``by``: ``sort!(samples; by)`` is a stable sort by the samples' keys; the rest as without ``by``."""
    s = np.asarray(samples).astype(dt)[key_order(sample_keys)].copy()
    if len(s) == 0:
        raise _lib.ArgumentError(_lib.ERR_ARG, "sort: empty sample")
    s[0] = _typemin(dt)
    step = len(s) // nparts
    b = [s[(x - 1) * step] for x in range(1, nparts + 1)]
    b.append(_typemax(dt))
    return np.asarray(b, dtype=dt)


def sort_exchange_plan(pids, sizes, rank_of, my_rank: int):
    """Who ships which piece where: piece j of source worker p (``sizes[p][j]`` keys, the run ending at split point j of p's sorted
    chunk) goes to worker ``pids[j]`` and lands at offset ``sum of the earlier sources' pieces`` of its receive buffer (the
    reference appends in arrival order and sorts afterwards, src/sort.jl:42-61; source order is used here).  Pure function of
    the size matrix, so every rank derives matching send/recv lists in the same (j, p) order."""
    plan = {"local": [], "sends": [], "recvs": []}
    for j in range(len(pids)):
        drank = rank_of(pids[j])
        off = 0
        for p in pids:
            n = sizes[p][j]
            if n:
                srank = rank_of(p)
                if srank == my_rank and drank == my_rank:
                    plan["local"].append((j, p, off, n))
                elif srank == my_rank:
                    plan["sends"].append((j, p, n, drank))
                elif drank == my_rank:
                    plan["recvs"].append((j, p, off, n, srank))
            off += n
    return plan


def sort(d: DArray, sample=_SAMPLE_DEFAULT, by=None, alg=None, dims=None, **kwargs) -> DArray:  # noqa: A001 - mirrors Base.sort
    """``sort(d::DVector; sample=true, alg, by)`` (reference src/sort.jl:107-170).  ``sample``: True (<= 512 sampled keys per
    worker balance the parts), False (uniform between min(d) and max(d)), a ``(min, max)`` tuple, or an array used as the sample.
    ``by``: a traceable key function (same closures as broadcast / map); values are ordered stably by ``by(x)``.
    ``alg`` is accepted and ignored: a keys-only sort has one result whatever the algorithm, and the keyed sort is stable like
    Julia's default.  Called on the slice of ``mapslices(sort, D; dims)`` it stands for the per-slice sort (``dab_sort_slices``).

    ``sort(A; dims=d)`` (1-based ``d``) sorts every fibre of ``A`` along ``d``: the values and the layout of ``mapslices(sort, A, dims=d)``,
    bit for bit.  With ``by = f`` the values of every fibre are put in the stable ``isless`` order of their keys ``f.(A)`` (K26,
    ``dab_sortperm_slices``), in the same layout.  A DVector with ``dims=1`` is ``sort(v)``.  Only ``by`` and ``alg`` go with ``dims``."""
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray):
        refuse("sort")
    from ._broadcast import Expr
    if isinstance(d, Expr):
        from . import _slices
        if _slices.tracing():
            return _slices.sort_of_slice(d, by, kwargs if dims is None else dict(kwargs, dims=dims))
    if dims is not None:
        return _sort_dims(d, dims, by, sample, kwargs, perm=False)
    sample = True if sample is _SAMPLE_DEFAULT else sample
    if isinstance(d, DArray) and d.dtype.kind == "c" and by is None:
        raise TypeError(f"MethodError: no method matching isless(::{d.dtype}, ::{d.dtype}) -- complex numbers are not ordered")
    return sort_with_boundaries(d, sample, by, alg, **kwargs)[0]


def sort_with_boundaries(d: DArray, sample=True, by=None, alg=None, **kwargs):
    """``sort`` plus the ``boundaries`` vector it partitioned with (what compute_boundaries returns, src/sort.jl:66-88)."""
    kf, pids = _check_args(d, sample, by, kwargs, "sort")
    presample = _presample(d, sample, len(pids), d.dtype)
    return _samplesort(d, d.chunks, d.dtype, presample, kf, perm=False)


def sortperm(d: DArray, sample=_SAMPLE_DEFAULT, by=None, alg=None, dims=None, **kwargs) -> DArray:
    """``sortperm(d::DVector; sample=true, by)``: the DVector of Int64 with ``d[p]`` sorted -- Julia's ``sortperm(Array(d))``, 1-based
    global indices in ``isless`` order, STABLE (equal keys, and all NaNs, keep ascending index order).  The samplesort of ``sort``
    with K21 (``dab_sort_pairs``) carrying every key's global index: chunk j of the result indexes the elements in chunk j of
    ``sort(d; sample)``, the layout is the same.  (Only when the reference's scan would leave NaNs ahead of larger keys, so that
    ``sort(d)`` itself is out of ``isless`` order, are the NaNs moved to the last receiving piece and the chunk sizes differ.)
    ``by = f``: ``sortperm(f.(d))``, with ``sample`` in key space.  ``alg`` is accepted and ignored (one stable result).

    ``sortperm(A; dims=d)`` (1-based ``d``): a ``DArray{Int64}`` of ``A``'s dims in which every fibre along ``d`` holds, at rank r, the
    1-based global column-major LINEAR index into ``A`` of the fibre element of rank r -- Julia >= 1.9's ``sortperm(A; dims)``, the
    ``LinearIndices(A)`` convention of ``findmax(A; dims)``.  Stable ``isless`` order: equal keys keep ascending index order, -0.0 sorts
    before +0.0, NaNs go last in input order.  ``by = f`` is ``sortperm(f.(A); dims)`` (a Bool key orders as 0 / 1).  The layout is
    ``sort(A; dims)``'s (that of ``mapslices(sort, A, dims=d)``), so ``A[sortperm(A; dims)]`` equals ``sort(A; dims)`` element for
    element -- except inside a run of NaNs with different payloads, which ``sort`` orders by bits and ``sortperm`` keeps in input
    order.  A DVector with ``dims=1`` is ``sortperm(v)``.  Only ``by`` and ``alg`` go with ``dims``."""
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray):
        refuse("sortperm")
    if dims is not None:
        return _sort_dims(d, dims, by, sample, kwargs, perm=True)
    sample = True if sample is _SAMPLE_DEFAULT else sample
    if isinstance(d, DArray) and d.dtype.kind == "c" and by is None:
        raise TypeError(f"MethodError: no method matching isless(::{d.dtype}, ::{d.dtype}) -- complex numbers are not ordered")
    kf, pids = _check_args(d, sample, by, kwargs, "sortperm")
    if d.size == 0:
        raise _lib.ArgumentError(_lib.ERR_EMPTY, "sortperm: empty DVector")
    kdt = d.dtype if kf is None else kf.kdt
    if kf is None:
        return _samplesort(d, d.chunks, kdt, _presample(d, sample, len(pids), kdt), None, perm=True)[0]
    if sample is not False:
        presample = _presample(None, sample, len(pids), kdt)   # a bad sample raises before the keys are computed
    keys = DArray(d.layout, kdt, {pid: kf.keys_of(ch) for pid, ch in d.chunks.items()}, d.rt)
    try:
        if sample is False:
            presample = _presample(keys, False, len(pids), kdt)
        return _samplesort(keys, keys.chunks, kdt, presample, None, perm=True)[0]
    finally:
        keys.close()


def _check_args(d: DArray, sample, by, kwargs, what: str):
    """The argument checks of ``sort`` / ``sortperm``, all before any launch: (traced key function or None, pids)."""
    if kwargs:
        raise _lib.ArgumentError(_lib.ERR_ARG, "Only `alg`, `by` and `sample` are supported as keyword arguments")
    if d.ndim != 1:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, f"{what} is defined for a DVector")
    dt = d.dtype
    if dt not in _SORT_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}: eltype {dt} (served: Float32 Float64 Int32 Int64)")
    kf = _KeyFn(d.rt, by, dt) if by is not None else None      # traced before any launch: an untraceable `by` raises here
    pids = list(d.layout.pids)
    if len(pids) > 256:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} over more than 256 workers")
    if sample is True and any(hi < lo for ((lo, hi),) in d.layout.indices):
        raise ZeroDivisionError("DivideError: integer division error")            # div(llp, 0) on an empty localpart, src/sort.jl:9
    return kf, pids


def _presample(d, sample, nparts: int, dt: np.dtype):
    """The sample of the boundaries that do not need the sorted chunks (src/sort.jl:118-155), or None for ``sample = true``.
    ``sample = false`` reads minimum(d) and maximum(d); the other forms launch nothing."""
    if sample is False:
        from ._mapreduce import maximum, minimum
        sample = (minimum(d), maximum(d))
    if isinstance(sample, tuple):
        if len(sample) != 2:
            raise _lib.ArgumentError(_lib.ERR_ARG, "keyword arg `sample` must be Boolean, Tuple(Min,Max) or an actual sample of data")
        return uniform_sample(sample[0], sample[1], nparts, dt)
    if isinstance(sample, (np.ndarray, list)):
        return np.asarray(sample)
    if sample is not True:
        raise _lib.ArgumentError(_lib.ERR_ARG, f"keyword arg `sample` must be Boolean, Tuple(Min,Max) or an actual sample of data : {sample}")
    return None


def _sort_pairs(rt, keys_ptr: int, keys_out: B200Array, vals_ptr, base: int, vals_out: B200Array, n: int, dt: np.dtype):
    """K21 on one chunk: keys_out / vals_out = keys / vals (``vals_ptr`` None: base + i) in the stable isless order of the keys."""
    need = C.c_size_t()
    _lib.check(_lib.lib().dab_sort_pairs_scratch_bytes(dab_dtype(dt), n, C.byref(need)))
    scratch = B200Array.empty(rt, (need.value,), np.uint8, temp=True)
    _lib.call("dab_sort_pairs", rt.ctx, dab_dtype(dt), C.c_void_p(keys_ptr), C.c_void_p(keys_out.ptr), C.c_void_p(vals_ptr), base,
              C.c_void_p(vals_out.ptr), C.c_void_p(scratch.ptr), need.value, n)
    scratch.free()


def _nan_count(rt, s: B200Array) -> int:
    """count(isnan, s) on the device (one reduce launch)."""
    slot = B200Array.empty(rt, (16,), np.uint8, temp=True)
    _lib.call("dab_reduce", rt.ctx, dab_dtype(s.dtype), _lib.COUNT, _lib.MAP_ISNAN, None, C.c_void_p(s.ptr), s.size, C.c_void_p(slot.ptr))
    n = int(slot.to_numpy()[:8].view(np.int64)[0])
    slot.free()
    return n


def _samplesort(d: DArray, src: Dict[int, B200Array], dt: np.dtype, presample, kf, perm: bool):
    """The samplesort of ``d``'s layout over the chunks ``src`` (keys of dtype ``dt``).  ``perm``: every key carries its 1-based
    global index (K21) and the result holds the indices instead of the keys."""
    rt = d.rt
    pids = list(d.layout.pids)
    nparts = len(pids)
    isz = dt.itemsize

    # ---- sort(localpart(d)) on every worker (sortperm: with the chunk's global indices)
    srt: Dict[int, B200Array] = {}
    idx: Dict[int, B200Array] = {}
    for pid, ch in src.items():
        out = B200Array.empty(rt, (ch.size,), dt, temp=True)
        if perm:
            idx[pid] = B200Array.empty(rt, (ch.size,), np.int64, temp=True)
            ((lo, _),) = d.layout.indices[pids.index(pid)]
            _sort_pairs(rt, ch.ptr, out, None, lo, idx[pid], ch.size, dt)
        elif kf is None:
            _sort_chunk(rt, ch.ptr, ch.size, dt, out)
        else:
            kf.sort_chunk(ch, out)
        srt[pid] = out

    # ---- boundaries
    if presample is not None:
        boundaries = boundaries_from_samples(presample, nparts, dt)
    else:
        # every worker's samples sorted[1:step:llp] (src/sort.jl:9-14) gathered on every rank: strided device gather into one staging
        # row per local worker, then ONE small all-gather through the exchange arena (no pickled host collective)
        wpr = rt.workers_per_rank
        SLOT = 1024                                             # <= 1023 samples per worker
        stage = B200Array.empty(rt, (wpr * SLOT,), dt, temp=True)
        counts = {}
        for k, pid in enumerate(pids):
            ((lo, hi),) = d.layout.indices[k]
            llp = max(0, hi - lo + 1)
            ss = SAMPLE_SIZE_ON_WORKER if llp > SAMPLE_SIZE_ON_WORKER else llp
            if ss == 0:
                raise ZeroDivisionError("DivideError: integer division error")        # div(llp, 0), src/sort.jl:9
            counts[pid] = len(range(0, llp, llp // ss))
        for pid, s in srt.items():
            llp = s.size
            step = llp // (SAMPLE_SIZE_ON_WORKER if llp > SAMPLE_SIZE_ON_WORKER else llp)
            cnt = counts[pid]
            # sorted[1:step:llp]: row 0 of the (step x cnt) column-major view of the sorted chunk
            _lib.call("dab_copy_box", rt.ctx, isz, C.c_void_p(stage.ptr + ((pid - 1) % wpr) * SLOT * isz), _lib.sz4((1, cnt)), _lib.sz4((0, 0, 0, 0)),
                      C.c_void_p(s.ptr), _lib.sz4((step, cnt)), _lib.sz4((0, 0, 0, 0)), _lib.sz4((1, cnt)))
        rows = rt.allgather_small(dev_ptr=stage.ptr, nbytes=wpr * SLOT * isz, dtype=dt)
        stage.free()
        everyone = {pid: rows[rt.rank_of(pid)][((pid - 1) % wpr) * SLOT:((pid - 1) % wpr) * SLOT + counts[pid]] for pid in pids}
        samples = np.concatenate([everyone[p] for p in pids])
        if kf is None:
            boundaries = boundaries_from_samples(samples, nparts, dt)
        else:                                                   # sort!(samples; by) (src/sort.jl:77): every rank holds the same samples
            boundaries = boundaries_from_samples_by(samples, kf.keys_of_host(samples), nparts, dt)

    # ---- split every sorted chunk at the boundaries (src/sort.jl:26-40): sizes[src pid][destination index]
    sizes_mine: Dict[int, List[int]] = {}
    ends: Dict[int, List[int]] = {}
    # with `by` the scan compares by(x) > by(boundaries[i+1]) (src/sort.jl:32): the same search on the keys of the sorted chunk
    bnd = np.ascontiguousarray(boundaries[1:] if kf is None else kf.keys_of_host(boundaries[1:]))
    split_dt = dt if kf is None else kf.kdt
    for pid, s in srt.items():
        cnt = (C.c_ulonglong * nparts)()
        ks = s if kf is None or s.size == 0 else kf.keys_of(s)
        _lib.call("dab_sorted_split", rt.ctx, dab_dtype(split_dt), C.c_void_p(ks.ptr), s.size, C.c_void_p(bnd.ctypes.data), nparts, cnt)
        if ks is not s:
            ks.free()                                           # dab_sorted_split returned with the counts: the keys are no longer read
        e, prev = [], 0
        for i in range(nparts):
            prev = max(prev, int(cnt[i]))                   # the scan for piece i starts where piece i-1 ended
            e.append(prev)
        ends[pid] = e
        sizes_mine[pid] = [e[0]] + [e[i] - e[i - 1] for i in range(1, nparts)]
        if perm:                                                # sortperm: the chunk's NaN count rides along as one more column
            sizes_mine[pid].append(_nan_count(rt, s) if dt.kind == "f" and s.size else 0)
    # the size matrix (source worker x destination) on every rank: one small all-gather through the exchange arena
    wpr = rt.workers_per_rank
    ncol = nparts + 1 if perm else nparts
    mine_arr = np.zeros((wpr, ncol), dtype=np.int64)
    for pid, row in sizes_mine.items():
        mine_arr[(pid - 1) % wpr] = row
    allrows = rt.allgather_small(mine_arr.reshape(-1))
    sizes: Dict[int, List[int]] = {}
    for pid in pids:
        r, w = rt.rank_of(pid), (pid - 1) % wpr
        sizes[pid] = [int(v) for v in allrows[r].reshape(wpr, ncol)[w]]
    if perm:
        # The reference scan leaves a chunk's NaNs (the tail of its sorted keys) in its last non-empty piece, which can lie ahead of
        # larger keys of other chunks.  sortperm moves them to the last piece that receives anything, J: the result stays in isless
        # order, and when sort's result is (every NaN chunk already ends in J) nothing moves and the layout is sort's.
        nan = {p: sizes[p].pop() for p in pids}
        J = max((max(j for j in range(nparts) if sizes[p][j]) for p in pids if any(sizes[p])), default=0)
        for p in pids:
            if nan[p]:
                last = max(j for j in range(nparts) if sizes[p][j])
                sizes[p][last] -= nan[p]
                sizes[p][J] += nan[p]
                if p in ends:
                    ends[p] = [int(x) for x in np.cumsum(sizes[p])]

    # ---- ship piece i to worker i (sortperm: the index plane travels with the keys, by the same plan)
    totals = [sum(sizes[p][j] for p in pids) for j in range(nparts)]
    # a worker that receives ONE non-empty piece already holds its sorted result: the piece lands straight in the result chunk and the
    # second sort (``sort!(lp_sorting)``, src/sort.jl:61) has nothing to do; several pieces are concatenated and sorted again
    recv: Dict[int, B200Array] = {}
    recv_idx: Dict[int, B200Array] = {}
    single_run: Dict[int, bool] = {}
    for j, pid in enumerate(pids):
        if rt.is_local(pid) and totals[j]:
            single_run[j] = sum(1 for p in pids if sizes[p][j]) == 1
            recv[j] = B200Array.empty(rt, (totals[j],), dt, temp=perm or not single_run[j])
            if perm:
                recv_idx[j] = B200Array.empty(rt, (totals[j],), np.int64, temp=not single_run[j])
    plan = sort_exchange_plan(pids, sizes, rt.rank_of, rt.rank)
    planes = [(srt, recv, isz)] + ([(idx, recv_idx, 8)] if perm else [])
    sends, recvs = [], []
    for sbufs, rbufs, es in planes:
        for j, p, off, n in plan["local"]:
            _lib.call("dab_d2d", rt.ctx, C.c_void_p(rbufs[j].ptr + off * es), C.c_void_p(sbufs[p].ptr + (ends[p][j] - n) * es), n * es)
        sends += [(sbufs[p].ptr + (ends[p][j] - n) * es, n * es, peer) for j, p, n, peer in plan["sends"]]
        recvs += [(rbufs[j].ptr + off * es, n * es, peer) for j, p, off, n, peer in plan["recvs"]]
    grouped_exchange(rt, sends, recvs)
    for s in list(srt.values()) + list(idx.values()):
        s.free()

    # ---- sort!(lp_sorting) on every receiver and DArray(local_sorted_refs) without the empty parts (src/sort.jl:52-61, 163-169)
    keep = [j for j in range(nparts) if totals[j] > 0]
    if not keep:
        raise _lib.ArgumentError(_lib.ERR_EMPTY, "sort: empty DVector")
    chunks: Dict[int, B200Array] = {}
    for j, buf in recv.items():
        if perm:
            # pieces arrive in source-worker order, which is global index order: the stable pair sort keeps equal keys in index order
            if single_run[j]:
                chunks[pids[j]] = recv_idx[j]
            else:
                chunks[pids[j]] = B200Array.empty(rt, (totals[j],), np.int64)
                _sort_pairs(rt, buf.ptr, buf, recv_idx[j].ptr, 0, chunks[pids[j]], totals[j], dt)
                recv_idx[j].free()
            buf.free()
            continue
        if single_run[j]:
            chunks[pids[j]] = buf
            continue
        out = B200Array.empty(rt, (totals[j],), dt)
        if kf is None:
            _sort_chunk(rt, buf.ptr, totals[j], dt, out)
        else:
            kf.sort_chunk(buf, out)
        buf.free()
        chunks[pids[j]] = out
    layout = layout_from_chunk_shapes([(totals[j],) for j in keep], (len(keep),), [pids[j] for j in keep])
    return DArray(layout, np.int64 if perm else dt, chunks, rt), boundaries


# ---- sort(A; dims) / sortperm(A; dims): segmented sorts of the fibres along one dimension ----------------------------------------------

_CHUNK_LIMIT_LONG = 0xFFFFF000                                 # K21's bound, which K26's long-fibre passes inherit


def check_dims(dims, ndim: int, what: str) -> int:
    """``dims`` of ``sort`` / ``sortperm``: a Python or NumPy integer (not a Bool) in ``1:ndim``."""
    if isinstance(dims, (bool, np.bool_)) or not isinstance(dims, (int, np.integer)) or not 1 <= int(dims) <= ndim:
        raise _lib.ArgumentError(_lib.ERR_ARG, f"{what}: dims = {dims!r} is not a dimension of a {ndim}-dimensional DArray (an integer in 1:{ndim})")
    return int(dims)


def _check_dims_args(A, dims, by, sample, kwargs, what: str):
    """Every refusal of ``sort`` / ``sortperm`` with ``dims``, before anything is allocated or launched: (dim, traced ``by`` or None)."""
    from ._darray import SubDArray, refuse_float16
    if isinstance(A, SubDArray):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(view; dims) is not served: make it a DArray first (DArray(view))")
    if sample is not _SAMPLE_DEFAULT or kwargs:
        given = (["sample"] if sample is not _SAMPLE_DEFAULT else []) + sorted(kwargs)
        raise _lib.ArgumentError(_lib.ERR_ARG, f"Only `alg`, `by` and `dims` are supported as keyword arguments with `dims` (got {', '.join(given)})")
    dim = check_dims(dims, A.ndim, what)
    dt = A.dtype
    if dt.kind == "c":
        if by is None:
            raise TypeError(f"MethodError: no method matching isless(::{dt}, ::{dt}) -- complex numbers are not ordered")
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}(A; dims, by) of a {dt} DArray is not served (no complex values are moved)")
    refuse_float16(what, A)
    if dt not in _SORT_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}: eltype {dt} (served: Float32 Float64 Int32 Int64)")
    kf = _KeyFn(A.rt, by, dt) if by is not None else None       # traced before any launch: an untraceable `by` raises here
    if kf is not None and kf.kdt not in _SORT_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what}: keys of type {kf.kdt} (served: Float32 Float64 Int32 Int64)")
    if A.ndim > 8:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} with dims over more than 8 dimensions is not served")
    return dim, kf


def _sort_dims(A, dims, by, sample, kwargs, perm: bool) -> DArray:
    """``sort(A; dims, by)`` / ``sortperm(A; dims, by)``.  Checks, then the working layout of ``mapslices(..., dims)`` (A's own when the
    dimension is whole on every worker, else the reference's redistribution ``p``), then one K26 launch per local chunk."""
    what = "sortperm" if perm else "sort"
    dim, kf = _check_dims_args(A, dims, by, sample, kwargs, what)
    if A.ndim == 1:                                             # a DVector: the samplesort, in its own layout
        return sortperm(A, by=by) if perm else sort(A, by=by)
    if not perm and kf is None:                                 # mapslices(sort, A, dims): K13 and the reference's redistribution
        from ._slices import mapslices
        return mapslices(sort, A, dims=dim)
    from . import _slices
    from .layout import make_layout, rlen, shape_of
    p = _slices.redistribution_grid(A.dims, A.layout.grid, (dim,), len(A.layout.pids))
    L = A.layout if p is None else make_layout(A.dims, list(A.layout.pids), p)
    if any(rlen(r) == 0 for I in L.indices for r in I):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} with dims over a DArray with an empty localpart is not served")
    shapes = [shape_of(I) for I in L.indices]
    if A.dims[dim - 1] > _lib.SORTPERM_SLICES_SMEM_LEN and any(int(np.prod(s)) >= _CHUNK_LIMIT_LONG for s in shapes):
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"{what} with dims: chunks of 2^32 - 4096 or more elements with fibres longer "
                                    f"than {_lib.SORTPERM_SLICES_SMEM_LEN} are not served")
    layout = layout_from_chunk_shapes(shapes, L.grid, L.pids)
    rt = A.rt
    W = A if p is None else _slices._redistribute(A, p)
    odt = np.dtype(np.int64) if perm else A.dtype
    chunks: Dict[int, B200Array] = {}
    try:
        for pid, ch in W.chunks.items():
            I = L.indices[L.pids.index(pid)]
            out = B200Array.empty(rt, ch.shape, odt)
            chunks[pid] = out
            keys = kf.keys_of(ch) if kf is not None else ch
            try:
                sortperm_slices_chunk(rt, keys, [r[0] - 1 for r in I], A.dims, dim, out if perm else None, None if perm else (ch, out))
            finally:
                if keys is not ch:
                    keys.free()
    except BaseException:
        for out in chunks.values():
            out.free()
        raise
    finally:
        if W is not A:
            W.close()
    return DArray(layout, odt, chunks, rt)


def sortperm_slices_chunk(rt, keys: B200Array, lo, gdims, dim: int, perm_out, vals):
    """One K26 launch: ``perm_out`` (Int64, the chunk's shape) gets the global indices; with ``vals = (src, dst)`` the values of ``src`` go
    to ``dst`` in the same order (then ``perm_out`` may be None: the indices go to a temporary)."""
    N = keys.ndim
    SZ = C.c_size_t * N
    tmp = B200Array.empty(rt, keys.shape, np.int64, temp=True) if perm_out is None else None
    P = perm_out if perm_out is not None else tmp
    try:
        src, dst = vals if vals is not None else (None, None)
        _lib.call("dab_sortperm_slices", rt.ctx, dab_dtype(keys.dtype), C.c_void_p(keys.ptr), N, SZ(*keys.shape), SZ(*lo), SZ(*gdims), dim,
                  C.c_void_p(P.ptr), src.dtype.itemsize if src is not None else 0, C.c_void_p(src.ptr if src is not None else None),
                  C.c_void_p(dst.ptr if dst is not None else None))
    finally:
        if tmp is not None:
            tmp.free()
