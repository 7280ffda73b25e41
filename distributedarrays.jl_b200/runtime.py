"""Process / device runtime: the stand-in for Julia's ``Distributed`` worker pool on this path.

One OS process per GPU (launched by ``torchrun``; RANK / LOCAL_RANK / WORLD_SIZE from the environment), exactly like the
reference's one Julia process per worker (test/runtests.jl:10-15).  ``torch.distributed`` is plumbing only: it ships
the 128-byte NCCL id and the CUDA IPC handles between ranks and provides host barriers.  All data-path traffic goes
through ``libdab200.so`` (NCCL / peer loads over NVLink).

Workers are numbered 1..P like ``workers()``.  ``P = world_size * workers_per_rank``; worker ``w`` lives on rank
``(w-1) // workers_per_rank``.  ``workers_per_rank > 1`` puts several chunks on one GPU -- used to exercise multi-chunk
layouts (grids, fibres, halo reads) on a single-GPU box; the production mapping is one worker per GPU.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, NamedTuple, Optional, Sequence

import numpy as np

from . import _lib

_RT: Optional["Runtime"] = None


class Runtime:
    def __init__(self, workers_per_rank: int = 1, device: Optional[int] = None, use_dist: Optional[bool] = None):
        L = _lib.lib()
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.workers_per_rank = int(workers_per_rank)
        n = C.c_int32(0)
        _lib.check(L.dab_device_count(C.byref(n)))
        if n.value < 1:
            raise _lib.DabError(_lib.ERR_CUDA, "no CUDA device visible: the DArray hot path has no CPU fallback")
        self.device = int(device) if device is not None else self.local_rank % n.value
        ctx = C.c_void_p()
        _lib.check(L.dab_init(self.device, C.byref(ctx)))
        self.ctx = ctx
        self.dist = None
        self._ipc_cache = {}
        self.last_kernel = None  # which entry point served the last local broadcast launch (diagnostics)
        self.fused_combine = False
        self._arena = None
        if use_dist is None:
            use_dist = self.world > 1
        if use_dist and self.world > 1:
            self._init_dist()

    # ---- torch.distributed plumbing ----------------------------------------------------------------------
    def _init_dist(self):
        import torch
        import torch.distributed as dist

        if not dist.is_initialized():
            torch.cuda.set_device(self.device)
            dist.init_process_group(backend="cpu:gloo,cuda:nccl", rank=self.rank, world_size=self.world)
        self.dist = dist
        ident = np.zeros(128, dtype=np.uint8)
        if self.rank == 0:
            _lib.check(_lib.lib().dab_comm_unique_id(ident.ctypes.data_as(C.c_void_p)))
        box = [ident.tobytes()]
        dist.broadcast_object_list(box, src=0)
        buf = C.create_string_buffer(box[0], 128)
        _lib.call("dab_comm_init_rank", self.ctx, buf, self.rank, self.world)
        # mailboxes for the fused reduce + combine kernel (peer stores over NVLink instead of ncclAllGather + D2H);
        # DAB_FUSED_COMBINE=0 keeps the NCCL path (A/B measurements, debugging)
        if os.environ.get("DAB_FUSED_COMBINE", "1") != "0":
            h = C.create_string_buffer(64)
            _lib.call("dab_mailbox_create", self.ctx, h)
            allh = [None] * self.world
            dist.all_gather_object(allh, h.raw)
            _lib.call("dab_mailbox_attach", self.ctx, C.create_string_buffer(b"".join(allh), 64 * self.world), self.rank, self.world)
            self.fused_combine = True
            dist.barrier()

    def barrier(self):
        """Stream sync + host barrier: the fence before one-sided (peer) reads of other workers' chunks."""
        self.sync()
        if self.dist is not None:
            self.dist.barrier()

    def device_barrier(self):
        """Stream-ordered barrier across the ranks (``dab_peer_barrier``): later launches on this rank's stream start only after every
        rank's earlier launches have completed -- the fence around one-sided peer reads / puts, without a host synchronisation.  Falls
        back to the host barrier when the peer mailboxes are not attached (``DAB_FUSED_COMBINE=0``)."""
        if self.world == 1:
            return
        if self.fused_combine:
            _lib.call("dab_peer_barrier", self.ctx)
        else:
            self.barrier()

    def arena(self, bank_bytes: int = 8 << 20):
        """The exchange arena: two banks of device memory per rank, mapped by every other rank over CUDA IPC (collective on first use).
        Small cross-worker payloads (tile results of ``mul!``, partial slabs of ``mapreducedim_between!``) are PUT straight into the
        consumer's bank with device-to-device copies over NVLink and ordered by ``device_barrier`` -- no NCCL launch, no host sync.
        Banks alternate per exchange, so a producer can fill the next bank while the consumer still reads the previous one."""
        if self._arena is None:
            bank_bytes = int(os.environ.get("DAB_ARENA_KB", bank_bytes >> 10)) << 10   # DAB_ARENA_KB=1 forces the NCCL fallbacks (tests)
            ptr = self.alloc(2 * bank_bytes + 256)
            base = (ptr + 255) & ~255
            if self.world > 1:
                handles = self.allgather_object((self.ipc_handle(ptr), base - ptr))
                peers = [base if r == self.rank else self.ipc_open(h) + off for r, (h, off) in enumerate(handles)]
            else:
                peers = [base]
            self._arena = {"alloc": ptr, "peers": peers, "bank_bytes": bank_bytes, "turn": 0}
        return self._arena

    def arena_next_bank(self) -> int:
        """Byte offset of the bank the next exchange uses (every rank calls this once per exchange, in the same order)."""
        a = self.arena()
        off = (a["turn"] & 1) * a["bank_bytes"]
        a["turn"] += 1
        return off

    def allgather_small(self, arr: Optional[np.ndarray] = None, dev_ptr: int = 0, nbytes: int = 0, dtype=np.uint8) -> List[np.ndarray]:
        """All-gather of one small fixed-size payload per rank WITHOUT a host collective: every rank PUTs its payload (a host array,
        or ``nbytes`` at ``dev_ptr`` on the device) into slot ``rank`` of every peer's exchange-arena bank, a device-side barrier makes
        the puts visible, one D2H copy brings the whole bank to the host.  ~50 us instead of the milliseconds of a pickled
        ``all_gather_object``.  Payloads must have the same size on every rank; falls back to the object gather when they do not fit."""
        if arr is not None:
            arr = np.ascontiguousarray(arr)
            nbytes, dtype = arr.nbytes, arr.dtype
        if self.world == 1:
            if arr is not None:
                return [arr.copy()]
            out = np.empty(nbytes, dtype=np.uint8)
            _lib.call("dab_d2h", self.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(dev_ptr), nbytes)
            self.sync()
            return [out.view(dtype)]
        slot = (nbytes + 255) & ~255
        if not self.fused_combine or slot * self.world > self.arena()["bank_bytes"]:
            if arr is None:
                arr = np.empty(nbytes, dtype=np.uint8)
                _lib.call("dab_d2h", self.ctx, C.c_void_p(arr.ctypes.data), C.c_void_p(dev_ptr), nbytes)
                self.sync()
                arr = arr.view(dtype)
            return self.allgather_object(arr)
        bank = self.arena_next_bank()
        peers = self.arena()["peers"]
        tmp = 0
        if arr is not None:
            tmp = self.alloc_temp(max(nbytes, 16))
            _lib.call("dab_h2d", self.ctx, C.c_void_p(tmp), C.c_void_p(arr.ctypes.data), nbytes)
            self.sync()                                    # arr may be a temporary of the caller
            dev_ptr = tmp
        for r in range(self.world):
            if nbytes:
                _lib.call("dab_d2d", self.ctx, C.c_void_p(peers[r] + bank + self.rank * slot), C.c_void_p(dev_ptr), nbytes)
        self.device_barrier()
        host = np.empty(slot * self.world, dtype=np.uint8)
        _lib.call("dab_d2h", self.ctx, C.c_void_p(host.ctypes.data), C.c_void_p(peers[self.rank] + bank), slot * self.world)
        self.sync()
        if tmp:
            self.free_temp(tmp)
        return [host[r * slot:r * slot + nbytes].view(dtype) for r in range(self.world)]

    def allgather_object(self, obj) -> list:
        if self.dist is None:
            return [obj]
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    # ---- workers -------------------------------------------------------------------------------------------
    @property
    def nworkers(self) -> int:
        return self.world * self.workers_per_rank

    def workers(self) -> List[int]:
        return list(range(1, self.nworkers + 1))

    def rank_of(self, pid: int) -> int:
        return (pid - 1) // self.workers_per_rank

    def is_local(self, pid: int) -> bool:
        return self.rank_of(pid) == self.rank

    def local_workers(self) -> List[int]:
        return [p for p in self.workers() if self.is_local(p)]

    def myid(self) -> int:
        """The first worker of this rank (the only one when workers_per_rank == 1)."""
        return self.rank * self.workers_per_rank + 1

    # ---- device helpers ------------------------------------------------------------------------------------
    def sync(self):
        _lib.call("dab_sync", self.ctx)

    def alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        _lib.call("dab_alloc", self.ctx, int(nbytes), C.byref(p))
        return int(p.value)

    def free(self, ptr: int):
        if ptr and self.ctx:
            _lib.call("dab_free", self.ctx, C.c_void_p(ptr))

    def alloc_temp(self, nbytes: int) -> int:
        """Stream-ordered temporary (cudaMallocAsync pool): no synchronisation, not IPC-exportable."""
        p = C.c_void_p()
        _lib.call("dab_alloc_async", self.ctx, int(nbytes), C.byref(p))
        return int(p.value)

    def free_temp(self, ptr: int):
        if ptr and self.ctx:
            _lib.call("dab_free_async", self.ctx, C.c_void_p(ptr))

    def set_option(self, key: str, value: int):
        """``dab_set_option``: e.g. ``set_option("ew_tma", 1)`` selects the TMA-staged elementwise kernel (same results)."""
        _lib.call("dab_set_option", self.ctx, key.encode(), int(value))

    def launches(self) -> int:
        n = C.c_uint64(0)
        _lib.call("dab_launch_count", self.ctx, C.byref(n))
        return int(n.value)

    def device_info(self):
        dev, sms, fr, tot = C.c_int32(), C.c_int32(), C.c_size_t(), C.c_size_t()
        _lib.call("dab_device_info", self.ctx, C.byref(dev), C.byref(sms), C.byref(fr), C.byref(tot))
        return {"device": dev.value, "sm_count": sms.value, "free_bytes": fr.value, "total_bytes": tot.value}

    # events on the ctx stream
    def event(self) -> int:
        e = C.c_void_p()
        _lib.call("dab_event_create", self.ctx, C.byref(e))
        return int(e.value)

    def record(self, ev: int):
        _lib.call("dab_event_record", self.ctx, C.c_void_p(ev))

    def elapsed_ms(self, e0: int, e1: int) -> float:
        ms = C.c_float()
        _lib.call("dab_event_elapsed_ms", self.ctx, C.c_void_p(e0), C.c_void_p(e1), C.byref(ms))
        return float(ms.value)

    def event_destroy(self, ev: int):
        _lib.call("dab_event_destroy", self.ctx, C.c_void_p(ev))

    # peer memory
    def ipc_handle(self, ptr: int) -> bytes:
        h = C.create_string_buffer(64)
        _lib.call("dab_ipc_get_handle", self.ctx, C.c_void_p(ptr), h)
        return h.raw

    def ipc_open(self, handle: bytes) -> int:
        if handle in self._ipc_cache:
            return self._ipc_cache[handle]
        p = C.c_void_p()
        _lib.call("dab_ipc_open", self.ctx, C.create_string_buffer(handle, 64), C.byref(p))
        self._ipc_cache[handle] = int(p.value)
        return int(p.value)

    def shutdown(self):
        global _RT
        if self.ctx:
            for p in self._ipc_cache.values():
                try:
                    _lib.call("dab_ipc_close", self.ctx, C.c_void_p(p))
                except _lib.DabError:
                    pass
            self._ipc_cache.clear()
            if self._arena is not None:
                try:
                    _lib.call("dab_free", self.ctx, C.c_void_p(self._arena["alloc"]))
                except _lib.DabError:
                    pass
                self._arena = None
            _lib.lib().dab_shutdown(self.ctx)
            self.ctx = None
        if self.dist is not None:
            try:
                if self.dist.is_initialized():
                    self.dist.destroy_process_group()
            except Exception:
                pass
            self.dist = None
        if _RT is self:
            _RT = None


# ---- how a rank reads from or ships to its peers ------------------------------------------------------------------------------
# Every operation with a cross-rank step goes through these helpers.  They take the runtime as an argument, so that a test can
# drive them with a stand-in.  All of them are collective: every rank calls them in the same order with arguments derived from
# the layouts alone.  DESIGN.md §5 lists which operations use which fence kind.


def fence(rt, kind: str):
    """``"host"``: ``barrier`` (stream sync + host barrier).  ``"device"``: ``device_barrier`` (stream-ordered, no host sync)."""
    if kind == "host":
        rt.barrier()
    elif kind == "device":
        rt.device_barrier()
    else:
        raise ValueError(f"fence kind {kind!r}: expected 'host' or 'device'")


def open_remote_reads(rt, arrays: Sequence, kind: str) -> bool:
    """Opening half of a one-sided read of other ranks' chunks of the DArrays ``arrays``: shares the CUDA-IPC handles not
    shared yet and fences the producers, so that every earlier write to those chunks has landed before a peer reads them.
    It opens one-sided WRITES the same way (``d[mask]`` stores into other ranks' chunks of its result): every owner has
    allocated the chunk and finished with it before a peer stores into it.  Nothing happens on one rank or for an empty
    list.  Returns whether it fenced; pass that to ``close_remote_reads``."""
    if rt.world == 1 or not arrays:
        return False
    for a in arrays:
        if a._handles is None:
            a.share()
    fence(rt, kind)
    return True


def close_remote_reads(rt, fenced: bool, kind: str):
    """Closing half of ``open_remote_reads``, with the same fence kind: the owners of the chunks that were read may not
    overwrite or free them before every reader's copy has run (freed blocks go straight back to the allocator cache).  The
    reference's ``remotecall_fetch`` is synchronous for the same reason.  After one-sided writes the closing fence is what
    makes the peers' stores visible to the chunks' owners."""
    if fenced:
        if kind == "host":
            rt.sync()
        fence(rt, kind)


def grouped_exchange(rt, sends: Sequence, recvs: Sequence):
    """One grouped NCCL point-to-point exchange of ``(device pointer, bytes, peer rank)`` transfers: every send in list order,
    then every receive in list order.  NCCL matches the grouped calls between two ranks in the order they are issued, so both
    sides must list a pair's transfers in the same order (the exchange plans do).  Two empty lists issue nothing."""
    if not sends and not recvs:
        return
    _lib.call("dab_group_start", rt.ctx)
    for ptr, nb, peer in sends:
        _lib.call("dab_send", rt.ctx, C.c_void_p(ptr), nb, peer)
    for ptr, nb, peer in recvs:
        _lib.call("dab_recv", rt.ctx, C.c_void_p(ptr), nb, peer)
    _lib.call("dab_group_end", rt.ctx)


class Stacks(NamedTuple):
    tables: Dict[int, Dict[int, int]]  # rank -> {result chunk: byte offset of its stack}, for every rank
    use_arena: bool
    bank: int                          # byte offset of the arena bank of this exchange (0 without the arena)
    base: int                          # device address of this rank's stacks
    temp: int                          # the private stack buffer the caller frees with ``free_temp`` (0 with the arena)


def exchange_stacks(rt, owners: Sequence[int], nbytes: Sequence[int]) -> Stacks:
    """Where the consumers of an exchange collect what they receive: one stack per result chunk ``c``, of ``nbytes[c]`` bytes
    rounded up to 256, on rank ``owners[c]``; each rank's stacks lie back to back in chunk order.  Every rank derives the same
    tables, so a producer knows the offset of a stack inside its consumer's buffer.  With several ranks, and every rank's
    stacks fitting one bank, the stacks sit in the exchange arena; otherwise in a private temporary.  ``deliver`` fills them."""
    tables: Dict[int, Dict[int, int]] = {r: {} for r in range(rt.world)}
    totals = [0] * rt.world
    for c, (r, nb) in enumerate(zip(owners, nbytes)):
        tables[r][c] = totals[r]
        totals[r] += (nb + 255) & ~255
    if rt.world > 1 and max(totals) <= rt.arena()["bank_bytes"]:
        bank = rt.arena_next_bank()
        return Stacks(tables, True, bank, rt.arena()["peers"][rt.rank] + bank, 0)
    temp = rt.alloc_temp(max(totals[rt.rank], 16))
    return Stacks(tables, False, 0, temp, temp)


def deliver(rt, st: Stacks, sends: Sequence, recvs: Sequence):
    """Moves slabs into the exchange stacks ``st`` of their consumers.  ``sends``: ``(source pointer, bytes, consumer rank, result chunk,
    byte offset in that chunk's stack)``; ``recvs``: ``(producer rank, result chunk, byte offset, bytes)``, used without the arena only.
    Sends to this rank's own stacks are device copies, issued first and in list order.  With the arena every other send is a put into
    its consumer's bank, and every rank then fences the device once, also a rank with nothing to send.  Without it the other sends and
    the receives go to one ``grouped_exchange`` in list order, so both sides must derive their lists from the same plan.  Zero-byte
    entries are skipped on both sides."""
    mine = st.tables[rt.rank]
    remote = []
    for src, nb, dst, c, off in sends:
        if nb and dst == rt.rank:
            _lib.call("dab_d2d", rt.ctx, C.c_void_p(st.base + mine[c] + off), C.c_void_p(src), nb)
        elif nb:
            remote.append((src, nb, dst, c, off))
    if st.use_arena:
        peers = rt.arena()["peers"]
        for src, nb, dst, c, off in remote:
            _lib.call("dab_d2d", rt.ctx, C.c_void_p(peers[dst] + st.bank + st.tables[dst][c] + off), C.c_void_p(src), nb)
        fence(rt, "device")                                   # every producer's puts have landed
    else:
        grouped_exchange(rt, [(src, nb, dst) for src, nb, dst, _, _ in remote],
                         [(st.base + mine[c] + off, nb, src) for src, c, off, nb in recvs if nb])


def init(workers_per_rank: int = 1, device: Optional[int] = None, use_dist: Optional[bool] = None) -> Runtime:
    """``addprocs`` analogue: create (or re-create) the process-wide runtime."""
    global _RT
    if _RT is not None:
        if _RT.workers_per_rank == workers_per_rank and (device is None or device == _RT.device):
            return _RT
        _RT.shutdown()
    _RT = Runtime(workers_per_rank, device, use_dist)
    return _RT


def runtime() -> Runtime:
    global _RT
    if _RT is None:
        _RT = Runtime()
    return _RT


def nworkers() -> int:
    return runtime().nworkers


def workers() -> List[int]:
    return runtime().workers()


def myid() -> int:
    return runtime().myid()
