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


def sort(d: DArray, sample=True, by=None, alg=None, **kwargs) -> DArray:  # noqa: A001 - mirrors Base.sort
    """``sort(d::DVector; sample=true, alg, by)`` (reference src/sort.jl:107-170).  ``sample``: True (<= 512 sampled keys per
    worker balance the parts), False (uniform between min(d) and max(d)), a ``(min, max)`` tuple, or an array used as the sample.
    ``by``: a traceable key function (same closures as broadcast / map); values are ordered stably by ``by(x)``.
    ``alg`` is accepted and ignored: a keys-only sort has one result whatever the algorithm, and the keyed sort is stable like
    Julia's default.  Called on the slice of ``mapslices(sort, D; dims)`` it stands for the per-slice sort (``dab_sort_slices``)."""
    from ._sparse import SparseDArray, refuse
    if isinstance(d, SparseDArray):
        refuse("sort")
    from ._broadcast import Expr
    if isinstance(d, Expr):
        from . import _slices
        if _slices.tracing():
            return _slices.sort_of_slice(d, by, kwargs)
    if isinstance(d, DArray) and d.dtype.kind == "c" and by is None:
        raise TypeError(f"MethodError: no method matching isless(::{d.dtype}, ::{d.dtype}) -- complex numbers are not ordered")
    return sort_with_boundaries(d, sample, by, alg, **kwargs)[0]


def sort_with_boundaries(d: DArray, sample=True, by=None, alg=None, **kwargs):
    """``sort`` plus the ``boundaries`` vector it partitioned with (what compute_boundaries returns, src/sort.jl:66-88)."""
    if kwargs:
        raise _lib.ArgumentError(_lib.ERR_ARG, "Only `alg`, `by` and `sample` are supported as keyword arguments")
    if d.ndim != 1:
        raise _lib.DimensionMismatch(_lib.ERR_DIM_MISMATCH, "sort is defined for a DVector")
    dt = d.dtype
    if dt not in _SORT_DTYPES:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, f"sort: eltype {dt} (served: Float32 Float64 Int32 Int64)")
    rt = d.rt
    kf = _KeyFn(rt, by, dt) if by is not None else None         # traced before any launch: an untraceable `by` raises here
    pids = list(d.layout.pids)
    nparts = len(pids)
    if nparts > 256:
        raise _lib.UnsupportedError(_lib.ERR_UNSUPPORTED, "sort over more than 256 workers")
    isz = dt.itemsize
    if sample is True and any(hi < lo for ((lo, hi),) in d.layout.indices):
        raise ZeroDivisionError("DivideError: integer division error")            # div(llp, 0) on an empty localpart, src/sort.jl:9

    # ---- boundaries that do not need the sorted chunks (src/sort.jl:118-155)
    presample = None
    if sample is False:
        from ._mapreduce import maximum, minimum
        sample = (minimum(d), maximum(d))
    if isinstance(sample, tuple):
        if len(sample) != 2:
            raise _lib.ArgumentError(_lib.ERR_ARG, "keyword arg `sample` must be Boolean, Tuple(Min,Max) or an actual sample of data")
        presample = uniform_sample(sample[0], sample[1], nparts, dt)
    elif isinstance(sample, (np.ndarray, list)):
        presample = np.asarray(sample)
    elif sample is not True:
        raise _lib.ArgumentError(_lib.ERR_ARG, f"keyword arg `sample` must be Boolean, Tuple(Min,Max) or an actual sample of data : {sample}")

    # ---- sort(localpart(d)) on every worker
    srt: Dict[int, B200Array] = {}
    for pid, ch in d.chunks.items():
        out = B200Array.empty(rt, (ch.size,), dt, temp=True)
        if kf is None:
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
    # the size matrix (source worker x destination) on every rank: one small all-gather through the exchange arena
    wpr = rt.workers_per_rank
    mine_arr = np.zeros((wpr, nparts), dtype=np.int64)
    for pid, row in sizes_mine.items():
        mine_arr[(pid - 1) % wpr] = row
    allrows = rt.allgather_small(mine_arr.reshape(-1))
    sizes: Dict[int, List[int]] = {}
    for pid in pids:
        r, w = rt.rank_of(pid), (pid - 1) % wpr
        sizes[pid] = [int(v) for v in allrows[r].reshape(wpr, nparts)[w]]

    # ---- ship piece i to worker i
    totals = [sum(sizes[p][j] for p in pids) for j in range(nparts)]
    # a worker that receives ONE non-empty piece already holds its sorted result: the piece lands straight in the result chunk and the
    # second sort (``sort!(lp_sorting)``, src/sort.jl:61) has nothing to do; several pieces are concatenated and sorted again
    recv: Dict[int, B200Array] = {}
    single_run: Dict[int, bool] = {}
    for j, pid in enumerate(pids):
        if rt.is_local(pid) and totals[j]:
            single_run[j] = sum(1 for p in pids if sizes[p][j]) == 1
            recv[j] = B200Array.empty(rt, (totals[j],), dt, temp=not single_run[j])
    plan = sort_exchange_plan(pids, sizes, rt.rank_of, rt.rank)
    for j, p, off, n in plan["local"]:
        _lib.call("dab_d2d", rt.ctx, C.c_void_p(recv[j].ptr + off * isz), C.c_void_p(srt[p].ptr + (ends[p][j] - n) * isz), n * isz)
    sends = [(srt[p].ptr + (ends[p][j] - n) * isz, n * isz, peer) for j, p, n, peer in plan["sends"]]
    recvs = [(recv[j].ptr + off * isz, n * isz, peer) for j, p, off, n, peer in plan["recvs"]]
    grouped_exchange(rt, sends, recvs)
    for s in srt.values():
        s.free()

    # ---- sort!(lp_sorting) on every receiver and DArray(local_sorted_refs) without the empty parts (src/sort.jl:52-61, 163-169)
    keep = [j for j in range(nparts) if totals[j] > 0]
    if not keep:
        raise _lib.ArgumentError(_lib.ERR_EMPTY, "sort: empty DVector")
    chunks: Dict[int, B200Array] = {}
    for j, buf in recv.items():
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
    return DArray(layout, dt, chunks, rt), boundaries
