"""CPU tests of the cross-rank protocol helpers in ``runtime.py`` (remote-read bracket, grouped exchange, exchange stacks), driven
with a stand-in runtime at world 2 that records every fence, share and C-ABI call.  No GPU and no second process: on one GPU every
``world > 1`` branch of the operations is skipped, so this is where a slip in the protocol shows up without a multi-GPU machine."""
import ctypes as C

import numpy as np
import pytest

PEERS = [1 << 40, 2 << 40]  # arena base of each rank, as mapped on this rank


class StandIn:
    """What the helpers use of ``Runtime``, with a log instead of a device."""

    def __init__(self, world=2, rank=0, wpr=1, bank_bytes=8 << 20):
        self.world, self.rank, self.workers_per_rank, self.ctx = world, rank, wpr, "ctx"
        self.bank_bytes, self.turn, self.log = bank_bytes, 0, []

    def rank_of(self, pid):
        return (pid - 1) // self.workers_per_rank

    def sync(self):
        self.log.append("sync")

    def barrier(self):
        self.log.append("barrier")

    def device_barrier(self):
        self.log.append("device_barrier")

    def arena(self):
        assert self.world > 1, "arena() allocates device memory: never at world 1"
        return {"bank_bytes": self.bank_bytes, "peers": PEERS}

    def arena_next_bank(self):
        self.log.append("arena_next_bank")
        off = (self.turn & 1) * self.bank_bytes
        self.turn += 1
        return off

    def alloc_temp(self, nbytes):
        self.log.append(("alloc_temp", nbytes))
        return 0x5000


class Shared:
    def __init__(self, rt, name, handles):
        self.rt, self.name, self._handles = rt, name, handles

    def share(self):
        self.rt.log.append(("share", self.name))
        self._handles = {}
        return self


@pytest.fixture()
def lib_calls(dab, monkeypatch):
    """Replaces ``_lib.call`` by a recorder: (name, arguments with pointers as integers)."""
    import sys
    calls = []

    def record(name, ctx, *args):
        calls.append((name,) + tuple(a.value if isinstance(a, C.c_void_p) else a for a in args))

    monkeypatch.setattr(sys.modules["darray_b200._lib"], "call", record)
    return calls


def test_remote_reads_at_world_1_do_nothing(dab):
    from darray_b200.runtime import close_remote_reads, open_remote_reads
    for kind in ("host", "device"):
        rt = StandIn(world=1)
        assert open_remote_reads(rt, [Shared(rt, "a", None)], kind) is False
        close_remote_reads(rt, False, kind)
        assert rt.log == []


def test_remote_reads_share_only_unshared_arrays_and_fence_once(dab):
    from darray_b200.runtime import open_remote_reads
    rt = StandIn()
    arrays = [Shared(rt, "a", None), Shared(rt, "b", {1: b"h"}), Shared(rt, "c", None)]
    assert open_remote_reads(rt, arrays, "host") is True
    assert rt.log == [("share", "a"), ("share", "c"), "barrier"]


def test_remote_reads_of_no_array_open_no_fence(dab):
    from darray_b200.runtime import close_remote_reads, open_remote_reads
    for kind in ("host", "device"):
        rt = StandIn()
        fenced = open_remote_reads(rt, [], kind)
        close_remote_reads(rt, fenced, kind)
        assert fenced is False and rt.log == []


@pytest.mark.parametrize("kind, opening, closing", [("host", ["barrier"], ["sync", "barrier"]),
                                                     ("device", ["device_barrier"], ["device_barrier"])])
def test_remote_read_fence_kinds(dab, lib_calls, kind, opening, closing):
    from darray_b200.runtime import close_remote_reads, open_remote_reads
    rt = StandIn(rank=1)
    fenced = open_remote_reads(rt, [Shared(rt, "a", {})], kind)
    assert rt.log == opening
    del rt.log[:]
    close_remote_reads(rt, fenced, kind)
    assert rt.log == closing and lib_calls == []


def test_unknown_fence_kind_is_an_error(dab):
    from darray_b200.runtime import open_remote_reads
    with pytest.raises(ValueError):
        open_remote_reads(StandIn(), [Shared(None, "a", {})], "stream")


def test_grouped_exchange_order(dab, lib_calls):
    from darray_b200.runtime import grouped_exchange
    rt = StandIn()
    grouped_exchange(rt, [], [])
    assert lib_calls == []
    grouped_exchange(rt, [(0x100, 8, 1), (0x200, 0, 1)], [(0x300, 16, 1), (0x400, 24, 1)])
    assert lib_calls == [("dab_group_start",), ("dab_send", 0x100, 8, 1), ("dab_send", 0x200, 0, 1), ("dab_recv", 0x300, 16, 1),
                         ("dab_recv", 0x400, 24, 1), ("dab_group_end",)]
    del lib_calls[:]
    grouped_exchange(rt, [], [(0x300, 16, 1)])
    assert lib_calls == [("dab_group_start",), ("dab_recv", 0x300, 16, 1), ("dab_group_end",)]
    assert rt.log == []


def _reducedim_stacks(dab, shape, nprocs, region, wpr, isz):
    """(owners, bytes) of the result chunks of ``mapreduce(...; dims=region)``, as ``mapreducedim`` computes them."""
    from darray_b200._mapreduce import plan_reducedim
    from darray_b200.layout import shape_of
    Rlayout, fibres = plan_reducedim(dab.make_layout(shape, list(range(1, nprocs + 1))), region)
    return ([(p - 1) // wpr for p in Rlayout.pids],
            [int(np.prod(shape_of(ix))) * len(f) * isz for ix, f in zip(Rlayout.indices, fibres)])


def _matvec_stacks(dab, n, ypids, gj, wpr, isz):
    """(owners, bytes) of the chunks of ``y`` in ``mul!(y, A, x)`` with ``gj`` tiles per chunk, as ``mul_`` computes them."""
    from darray_b200.layout import rlen
    ylay = dab.make_layout((n,), ypids, [len(ypids)])
    return [(p - 1) // wpr for p in ypids], [rlen(ix[0]) * gj * isz for ix in ylay.indices]


# Offsets and per-rank totals the two stack tables of mapreducedim and mul! gave before they were merged.
STACK_CASES = [
    ("reducedim", ((1000, 600), 8, (1,), 4, 8), {0: {0: 0}, 1: {1: 0}}, [9728, 9728]),
    ("reducedim", ((700, 12), 8, (2,), 4, 4), {0: {0: 0, 1: 512, 2: 1024, 3: 1536}, 1: {4: 0, 5: 512, 6: 1024, 7: 1536}}, [2048, 2048]),
    ("reducedim", ((6, 5, 8), 8, (1, 3), 4, 8), {0: {0: 0, 1: 256}, 1: {}}, [512, 0]),
    ("reducedim", ((300, 7), 4, (2,), 2, 8), {0: {0: 0, 1: 768}, 1: {2: 0, 3: 768}}, [1536, 1536]),
    ("matvec", (1001, [1, 2, 3, 4, 5, 6, 7, 8], 3, 4, 8), {0: {0: 0, 1: 3072, 2: 6144, 3: 9216}, 1: {4: 0, 5: 3072, 6: 6144, 7: 9216}},
     [12288, 12288]),
    ("matvec", (1000, [1, 2, 3, 4], 2, 2, 4), {0: {0: 0, 1: 2048}, 1: {2: 0, 3: 2048}}, [4096, 4096]),
    ("matvec", (17, [1, 2], 5, 2, 4), {0: {0: 0, 1: 256}, 1: {}}, [512, 0]),
]


@pytest.mark.parametrize("kind, args, tables, totals", STACK_CASES)
@pytest.mark.parametrize("rank", [0, 1])
def test_exchange_stacks_tables_and_placement(dab, kind, args, tables, totals, rank):
    from darray_b200.runtime import exchange_stacks
    owners, nbytes = (_reducedim_stacks if kind == "reducedim" else _matvec_stacks)(dab, *args)
    # every rank's stacks fit one bank: the arena, one bank per exchange, alternating
    rt = StandIn(rank=rank, bank_bytes=max(totals))
    for bank in (0, max(totals)):
        st = exchange_stacks(rt, owners, nbytes)
        assert st.tables == tables
        assert st.use_arena and st.bank == bank and st.base == PEERS[rank] + bank and st.temp == 0
    assert rt.log == ["arena_next_bank", "arena_next_bank"]
    # one rank's stacks do not fit: a private temporary of max(total, 16) bytes on every rank, no bank taken
    rt = StandIn(rank=rank, bank_bytes=max(totals) - 1)
    st = exchange_stacks(rt, owners, nbytes)
    assert st.tables == tables
    assert not st.use_arena and st.base == st.temp == 0x5000
    assert rt.log == [("alloc_temp", max(totals[rank], 16))]


def test_exchange_stacks_at_world_1_never_touch_the_arena(dab):
    from darray_b200.runtime import exchange_stacks
    owners, nbytes = _matvec_stacks(dab, 1001, [1, 2, 3, 4, 5, 6, 7, 8], 3, 8, 8)
    rt = StandIn(world=1)
    st = exchange_stacks(rt, owners, nbytes)
    assert st.tables == {0: {0: 0, 1: 3072, 2: 6144, 3: 9216, 4: 12288, 5: 15360, 6: 18432, 7: 21504}}
    assert not st.use_arena and st.temp == 0x5000 and rt.log == [("alloc_temp", 24576)]


# ---- deliver: slabs into the exchange stacks ------------------------------------------------------------------------------------------

TABLES = {0: {0: 0, 1: 512}, 1: {2: 0}}
# (source, bytes, consumer rank, result chunk, offset): a put, a local copy, a zero-byte put, a local copy
SENDS = [(0x100, 8, 1, 2, 16), (0x200, 16, 0, 1, 32), (0x300, 0, 1, 2, 0), (0x400, 24, 0, 0, 0)]
RECVS = [(1, 0, 8, 8), (1, 1, 0, 0), (1, 1, 16, 4)]                 # (producer rank, result chunk, offset, bytes)


def test_deliver_with_the_arena_puts_then_fences_once_on_every_rank(dab, lib_calls):
    from darray_b200.runtime import Stacks, deliver
    bank = 8 << 20
    rt = StandIn(rank=0)
    deliver(rt, Stacks(TABLES, True, bank, PEERS[0] + bank, 0), SENDS, RECVS)
    assert lib_calls == [("dab_d2d", PEERS[0] + bank + 512 + 32, 0x200, 16), ("dab_d2d", PEERS[0] + bank, 0x400, 24),
                         ("dab_d2d", PEERS[1] + bank + 16, 0x100, 8)]
    assert rt.log == ["device_barrier"]
    del lib_calls[:]
    rt = StandIn(rank=1)                                            # nothing to send: the fence is collective all the same
    deliver(rt, Stacks(TABLES, True, bank, PEERS[1] + bank, 0), [], [(0, 2, 16, 8)])
    assert lib_calls == [] and rt.log == ["device_barrier"]


def test_deliver_without_the_arena_is_one_grouped_exchange(dab, lib_calls):
    from darray_b200.runtime import Stacks, deliver
    rt = StandIn(rank=0)
    deliver(rt, Stacks(TABLES, False, 0, 0x5000, 0x5000), SENDS, RECVS)
    assert lib_calls == [("dab_d2d", 0x5000 + 512 + 32, 0x200, 16), ("dab_d2d", 0x5000, 0x400, 24), ("dab_group_start",),
                         ("dab_send", 0x100, 8, 1), ("dab_recv", 0x5000 + 8, 8, 1), ("dab_recv", 0x5000 + 512 + 16, 4, 1), ("dab_group_end",)]
    assert rt.log == []


def test_deliver_at_world_1_copies_only(dab, lib_calls):
    from darray_b200.runtime import Stacks, deliver
    rt = StandIn(world=1)
    deliver(rt, Stacks({0: {0: 0, 1: 256}}, False, 0, 0x5000, 0x5000), [(0x100, 8, 0, 1, 8), (0x200, 0, 0, 0, 0), (0x300, 4, 0, 0, 0)], [])
    assert lib_calls == [("dab_d2d", 0x5000 + 256 + 8, 0x100, 8), ("dab_d2d", 0x5000, 0x300, 4)] and rt.log == []


# ---- gather_fibres: the slabs of every fibre on the owner of its result chunk, run on both ranks of a world of 2 ------------------------


def _reducedim_case(dab, shape, nprocs, region, wpr, isz):
    from darray_b200._mapreduce import plan_reducedim
    from darray_b200.layout import shape_of
    L = dab.make_layout(shape, list(range(1, nprocs + 1)))
    R, fibres = plan_reducedim(L, region)
    plens = [int(np.prod(shape_of(ix))) for ix in R.indices]
    return L, R, fibres, [(plen * isz,) for plen in plens], wpr


def _findmax_case(dab, shape, dist, region, wpr, isz):
    """As ``_findmax._dims`` calls it: values and indices, a fibre of one member gathers nothing."""
    from darray_b200._mapreduce import plan_reducedim
    from darray_b200.layout import shape_of
    L = dab.make_layout(shape, list(range(1, int(np.prod(dist)) + 1)), dist)
    R, fibres = plan_reducedim(L, region)
    plens = [int(np.prod(shape_of(ix))) for ix in R.indices]
    return L, R, [m if len(m) > 1 else [] for m in fibres], [(plen * isz, plen * 8) for plen in plens], wpr


def _scan_case(dab, shape, dist, dims, wpr, isz):
    """As ``_scan._run`` calls it: the carry slabs of every chunk along ``dims``."""
    from darray_b200._scan import carry_plan
    from darray_b200.layout import shape_of
    L = dab.make_layout(shape, list(range(1, int(np.prod(dist)) + 1)), dist)
    k = dims - 1
    plens = [int(np.prod([s for a, s in enumerate(shape_of(ix)) if a != k])) for ix in L.indices]
    return L, L, carry_plan(L, dims), [(plen * isz,) for plen in plens], wpr


GATHER_CASES = [("reducedim", args, tables) for kind, args, tables, _ in STACK_CASES if kind == "reducedim"] + [
    ("findmax", ((14, 9), (2, 3), (2,), 3, 4), None),               # Float32 values of 3 x 7 per stack: a value plane of 84 bytes
    ("findmax", ((14, 9), (1, 3), (1,), 2, 8), None),               # reduced dim not cut: fibres of one member, nothing moves
    ("scan", ((30, 20), (2, 4), 2, 4, 8), None),
    ("scan", ((9, 12), (1, 4), 2, 2, 8), None),
]


def _slab(pid, p):
    return (pid << 24) | (p << 20)


def _gather_on_both_ranks(dab, lib_calls, case, arena):
    from darray_b200._mapreduce import gather_fibres
    L, R, fibres, plane_bytes, wpr = case
    runs = []
    for rank in (0, 1):
        rt = StandIn(rank=rank, wpr=wpr, bank_bytes=(8 << 20) if arena else -1)      # -1: not even empty stacks fit
        del lib_calls[:]
        slabs = {pid: tuple(_slab(pid, p) for p in range(len(plane_bytes[0]))) for pid in L.pids if rt.rank_of(pid) == rank}
        st, planes = gather_fibres(rt, L, R, fibres, plane_bytes, slabs)
        runs.append((rt, st, planes, list(lib_calls)))
    return runs


def _expected_writes(L, fibres, plane_bytes, planes):
    """Every (address, source, bytes) the owner's fold reads: slot s of plane p of result chunk rl holds member s's slab of plane p."""
    return sorted((planes[rl][p] + s * nb, _slab(L.pids[m], p), nb) for rl in planes for p, nb in enumerate(plane_bytes[rl]) if nb
                  for s, m in enumerate(fibres[rl]))


@pytest.mark.parametrize("kind, args, tables", GATHER_CASES)
def test_gather_fibres_with_the_arena_writes_every_slot_once(dab, lib_calls, kind, args, tables):
    case = {"reducedim": _reducedim_case, "findmax": _findmax_case, "scan": _scan_case}[kind](dab, *args)
    L, R, fibres, plane_bytes, _ = case
    runs = _gather_on_both_ranks(dab, lib_calls, case, arena=True)
    writes, expected = [], []
    for rank, (rt, st, planes, calls) in enumerate(runs):
        assert st.use_arena and rt.log == ["arena_next_bank", "device_barrier"]
        assert tables is None or st.tables == tables
        assert set(planes) == {rl for rl, p in enumerate(R.pids) if rt.rank_of(p) == rank}
        assert all(c[0] == "dab_d2d" for c in calls)
        writes += [c[1:] for c in calls]
        expected += _expected_writes(L, fibres, plane_bytes, planes)
    assert sorted(writes) == sorted(expected)


@pytest.mark.parametrize("kind, args, tables", GATHER_CASES)
def test_gather_fibres_without_the_arena_pairs_sends_and_receives(dab, lib_calls, kind, args, tables):
    case = {"reducedim": _reducedim_case, "findmax": _findmax_case, "scan": _scan_case}[kind](dab, *args)
    L, R, fibres, plane_bytes, _ = case
    runs = _gather_on_both_ranks(dab, lib_calls, case, arena=False)
    for rank, (rt, st, planes, calls) in enumerate(runs):
        assert not st.use_arena and all(e[0] == "alloc_temp" for e in rt.log)
        assert tables is None or st.tables == tables
        other = 1 - rank
        sends = [c[1:3] for c in runs[other][3] if c[0] == "dab_send" and c[3] == rank]
        recvs = [c[1:3] for c in calls if c[0] == "dab_recv" and c[3] == other]
        assert [nb for _, nb in sends] == [nb for _, nb in recvs]    # NCCL pairs them in issue order
        writes = [c[1:] for c in calls if c[0] == "dab_d2d"] + [(dst, src, nb) for (src, _), (dst, nb) in zip(sends, recvs)]
        assert sorted(writes) == _expected_writes(L, fibres, plane_bytes, planes)
        assert all(c[2] for c in calls if c[0] in ("dab_send", "dab_recv"))
