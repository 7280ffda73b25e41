"""GPU tests of the onesweep radix sort on the paths its control flow takes: K11 (``dab_sort``), its pair form K21 (``dab_sort_pairs``)
and the callers that run it on whole chunks (``dab_sort_by_key``, ``sort`` / ``sortperm`` of a DVector), bit for bit against the
radix-key model of ``dab_sort_key.cuh`` (``radix_enc`` / ``radix_dec`` / ``by_radix_key`` of tests/hostmem_abi.py).

Which path the kernel takes is decided by properties that random data leaves to chance, so every input here is built to reach one:
  * which digit passes run (``sort_plan_kernel``): keys are built in radix-key space with exactly a chosen set of non-constant digit
    positions, then decoded to the dtype.  Each test asserts its premise on the NumPy histograms of the radix keys;
  * how many tiles a CTA takes: every instance keeps at most 3 CTAs on an SM (its tile takes over 69 KiB of shared memory), so a CTA
    takes a second ticket only past 3 * sm_count tiles.  The persistent size class has at least 4 tiles per resident CTA;
  * how a tile reaches shared memory: one bulk copy when its source is 16-byte aligned and its byte count a multiple of 16 (pairs: and
    its positions too), plain loads otherwise.  The remainder r of the last tile and the pointer phase pick the one or the other;
  * look-back skew: sorted, reversed, and one digit value per tile make the look-back walk runs of zero-count words.
Every output buffer and the scratch sit between guard bands of sentinel bytes inside their allocation, checked after the sort: a store
past either end is caught and cannot fault.  The input of an out-of-place sort is checked unchanged.

The keys-only order: radix-key order, so NaNs come last ordered by payload, of either sign (the header of dab_sort.cu).  The pair order:
a stable argsort of the collapsed key, every NaN one key, so NaNs keep their input order."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import hostmem_abi as hm
from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets the pair sort too
    import sortperm_hostmem
    sortperm_hostmem.install()

DTYPES = [np.float32, np.float64, np.int32, np.int64]
CODE = {np.dtype(np.float32): hm.F32, np.dtype(np.float64): hm.F64, np.dtype(np.int32): hm.I32, np.dtype(np.int64): hm.I64}
UINT = {4: np.uint32, 8: np.uint64}

# Tile shapes of the sort_passes<T, P, THREADS, KPT, MINB> instances in dab_sort.cu (THREADS * KPT keys per tile, MINB CTAs per SM);
# tests/test_cpu_sort.py checks them against the source
KEYS_TILE = {4: 256 * 32, 8: 256 * 16}
PAIRS_TILE = {4: 256 * 16, 8: 256 * 10}
CTAS_PER_SM = 3
TILES_PER_CTA = 4                                               # persistent class: at least this many tiles per resident CTA
GUARD = 512                                                     # sentinel bytes on either side of a buffer (a multiple of 16)
NOT_SERVED = 0xFFFFF000                                         # the first chunk length the sort refuses


# ---- data by digit set ---------------------------------------------------------------------------------------------------------
def digit_sets(width: int) -> dict:
    """The digit sets every dtype is tested with: none, the lowest, the top, both, an odd and an even interior subset, all."""
    top = width - 1
    odd, even = ((2,), (1, 2)) if width == 4 else ((1, 2, 5), (3, 6))
    return {"none": (), "low": (0,), "top": (top,), "low_top": (0, top), "odd": odd, "even": even, "all": tuple(range(width))}


def radix_digit_keys(width: int, n: int, digits, rng, pairs_float: bool = False) -> np.ndarray:
    """n radix keys in which exactly the positions ``digits`` vary; every other byte is one fixed random value.  ``pairs_float``: the
    top byte stays below 0xFF, so no key is a NaN or +Inf of a float dtype and the collapse of NaNs cannot merge keys."""
    U = UINT[width]
    fixed = rng.integers(0, 255 if pairs_float else 256, width)
    k = np.zeros(n, dtype=U)
    for d in range(width):
        hi = 255 if (pairs_float and d == width - 1) else 256
        byte = rng.integers(0, hi, n, dtype=np.uint16) if d in digits else np.full(n, fixed[d], dtype=np.uint16)
        k |= byte.astype(U) << U(8 * d)
    return k


def outlier_keys(width: int, n: int, digit: int, at: int, larger: bool, rng) -> np.ndarray:
    """All keys equal but the one at index ``at``, which differs in ``digit`` only (larger or smaller): that digit's largest bin holds
    n - 1 keys, and the pass must still run."""
    U = UINT[width]
    base = radix_digit_keys(width, 1, (), rng, pairs_float=True)[0]
    lo, hi = U(0x30), U(0xC0)
    mask = ~(U(0xFF) << U(8 * digit))
    base = (base & mask) | ((hi if not larger else lo) << U(8 * digit))
    k = np.full(n, base, dtype=U)
    k[at] = (base & mask) | ((hi if larger else lo) << U(8 * digit))
    return k


def tile_digit_keys(width: int, n: int, tile: int, rng, pairs_float: bool = False) -> np.ndarray:
    """Every digit varies, and digit 0 is one value per tile (tile t holds (97 t) mod 256): the first pass sends each tile to one bucket,
    so the look-back of every other digit walks runs of zero counts."""
    U = UINT[width]
    k = radix_digit_keys(width, n, range(width), rng, pairs_float)
    t = (np.arange(n, dtype=np.int64) // tile * 97 % 256).astype(U)
    return (k & ~U(0xFF)) | t


def decode(keys: np.ndarray, T, nan_share: float = 0.0, rng=None) -> np.ndarray:
    """Radix keys -> keys of dtype T (bit patterns).  ``nan_share`` > 0 (floats): that share of the keys becomes NaNs of random payload
    and sign; their collapsed key is the top one."""
    T = np.dtype(T)
    raw = hm.radix_dec(keys, CODE[T])
    if nan_share and T.kind == "f":
        U = UINT[T.itemsize]
        pick = rng.random(raw.size) < nan_share
        payload = rng.integers(1, 1 << (22 if T.itemsize == 4 else 51), int(pick.sum()), dtype=np.int64).astype(U)
        exp = U(0x7F800000) if T.itemsize == 4 else U(0x7FF0000000000000)
        sign = rng.integers(0, 2, payload.size).astype(U) << U(8 * T.itemsize - 1)
        raw[pick] = sign | exp | payload
    return raw.view(T)


def active_digits(radix: np.ndarray) -> tuple:
    """The digit positions whose 256-bin histogram is not one full bin: the passes sort_plan_kernel runs."""
    width = radix.dtype.itemsize
    out = []
    for d in range(width):
        h = np.bincount(((radix >> radix.dtype.type(8 * d)) & radix.dtype.type(0xFF)).astype(np.intp), minlength=256)
        if h.max() < radix.size:
            out.append(d)
    return tuple(out)


def largest_bin(radix: np.ndarray, d: int) -> int:
    return int(np.bincount(((radix >> radix.dtype.type(8 * d)) & radix.dtype.type(0xFF)).astype(np.intp), minlength=256).max())


def keys_radix(a: np.ndarray) -> np.ndarray:
    return hm.radix_enc(a.view(UINT[a.itemsize]), CODE[a.dtype])


def pairs_radix(a: np.ndarray) -> np.ndarray:
    return hm.by_radix_key(a.view(UINT[a.itemsize]), CODE[a.dtype])


# ---- the model --------------------------------------------------------------------------------------------------------------------
def model_sort(a: np.ndarray) -> np.ndarray:
    """Keys only: dec(sort(enc(raw))), as bit patterns."""
    return hm.radix_dec(np.sort(keys_radix(a)), CODE[a.dtype])


def model_pairs(a: np.ndarray):
    """Pairs: (perm, sorted collapsed keys): a stable argsort of the collapsed radix key."""
    e = pairs_radix(a)
    perm = np.argsort(e, kind="stable")
    return perm, e[perm]


def check_pairs(a, perm, ekeys, vals, base, got_k, got_v):
    """vals_out exactly; keys_out bit for bit, up to the collapse of NaNs (every NaN key comes out as a NaN)."""
    want_v = vals[perm] if vals is not None else np.int64(base) + perm.astype(np.int64)
    assert got_v.dtype == np.int64 and np.array_equal(got_v, want_v)
    U = UINT[a.itemsize]
    want_k = hm.radix_dec(ekeys, CODE[a.dtype])
    nan = (ekeys == ~U(0)) if a.dtype.kind == "f" else np.zeros(a.size, dtype=bool)
    gk = got_k.view(U)
    assert np.array_equal(gk[~nan], want_k[~nan])
    assert np.all(np.isnan(got_k[nan]))


# ---- device buffers between guard bands -------------------------------------------------------------------------------------------
class Guarded:
    """n elements of ``dtype`` starting ``phase`` elements past a 16-byte boundary, with GUARD sentinel bytes before and after, all in
    one allocation."""

    def __init__(self, dab, rt, dtype, n, phase=0, data=None, seed=0):
        from darray_b200 import _lib
        self.lib, self.rt, self.dt, self.n = _lib, rt, np.dtype(dtype), int(n)
        self.nbytes = self.n * self.dt.itemsize
        self.lo = GUARD + phase * self.dt.itemsize
        self.buf = dab.B200Array.empty(rt, (self.lo + self.nbytes + GUARD,), np.uint8)
        self.ptr = self.buf.ptr + self.lo
        g = np.random.default_rng(seed + 7919 * self.n + phase)
        self.head = g.integers(0, 256, self.lo, dtype=np.uint8)
        self.tail = g.integers(0, 256, GUARD, dtype=np.uint8)
        self._put(self.buf.ptr, self.head)
        self._put(self.ptr + self.nbytes, self.tail)
        if data is not None:
            assert data.dtype == self.dt and data.size == self.n
            self._put(self.ptr, np.ascontiguousarray(data))
        rt.sync()

    def _put(self, dst, host):
        if host.nbytes:
            self.lib.call("dab_h2d", self.rt.ctx, C.c_void_p(dst), C.c_void_p(host.ctypes.data), host.nbytes)

    def _get(self, src, nbytes):
        out = np.empty(nbytes, dtype=np.uint8)
        if nbytes:
            self.lib.call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(src), nbytes)
        return out

    def check_guards(self):
        head, tail = self._get(self.buf.ptr, self.lo), self._get(self.ptr + self.nbytes, GUARD)
        self.rt.sync()
        assert np.array_equal(head, self.head), "a store before the start of the buffer"
        assert np.array_equal(tail, self.tail), "a store past the end of the buffer"

    def read(self) -> np.ndarray:
        self.check_guards()
        got = self._get(self.ptr, self.nbytes)
        self.rt.sync()
        return got.view(self.dt)

    def free(self):
        self.buf.free()


def run_sort(dab, rt, a, inplace=False, in_phase=0, out_phase=0, tmp_phase=0):
    """dab_sort of ``a`` through guarded buffers: the keys as they come back (the input checked unchanged when out of place)."""
    from darray_b200 import _lib
    n = a.size
    src = Guarded(dab, rt, a.dtype, n, in_phase, a, seed=1)
    out = src if inplace else Guarded(dab, rt, a.dtype, n, out_phase, seed=2)
    tmp = Guarded(dab, rt, a.dtype, n, tmp_phase, seed=3)
    _lib.call("dab_sort", rt.ctx, dab.dab_dtype(a.dtype), C.c_void_p(src.ptr), C.c_void_p(out.ptr), C.c_void_p(tmp.ptr), n)
    got = out.read()
    tmp.check_guards()
    if not inplace:
        assert np.array_equal(src.read().view(np.uint8), a.view(np.uint8)), "the input of an out-of-place sort was written"
        out.free()
    src.free()
    tmp.free()
    return got


def run_pairs(dab, rt, a, vals=None, base=1, inplace=False, in_phase=0, out_phase=0):
    """dab_sort_pairs of ``a`` through guarded buffers (keys, keys_out, vals_out and the 16-byte aligned scratch): (keys_out, vals_out)."""
    from darray_b200 import _lib
    n = a.size
    code = dab.dab_dtype(a.dtype)
    keys = Guarded(dab, rt, a.dtype, n, in_phase, a, seed=11)
    kout = keys if inplace else Guarded(dab, rt, a.dtype, n, out_phase, seed=12)
    dv = Guarded(dab, rt, np.int64, n, 0, vals, seed=13) if vals is not None else None
    vout = Guarded(dab, rt, np.int64, n, 0, seed=14)
    need = C.c_size_t()
    _lib.check(_lib.lib().dab_sort_pairs_scratch_bytes(code, n, C.byref(need)))
    scratch = Guarded(dab, rt, np.uint8, need.value, 0, seed=15)
    _lib.call("dab_sort_pairs", rt.ctx, code, C.c_void_p(keys.ptr), C.c_void_p(kout.ptr), C.c_void_p(dv.ptr if dv else None), base,
              C.c_void_p(vout.ptr), C.c_void_p(scratch.ptr), need.value, n)
    got_k, got_v = kout.read(), vout.read()
    scratch.check_guards()
    if not inplace:
        assert np.array_equal(keys.read().view(np.uint8), a.view(np.uint8)), "the input keys of an out-of-place sort were written"
        kout.free()
    if dv is not None:
        assert np.array_equal(dv.read(), vals), "the input values were written"
        dv.free()
    for b in (keys, vout, scratch):
        b.free()
    return got_k, got_v


# ---- cases ------------------------------------------------------------------------------------------------------------------------
def make_case(T, name, n, tile, rng, pairs=False):
    """(keys of dtype T, expected active digits, outlier digit or None) for a named case."""
    T = np.dtype(T)
    w = T.itemsize
    pf = pairs and T.kind == "f"
    sets = digit_sets(w)
    if name in sets:
        k = radix_digit_keys(w, n, sets[name], rng, pf)
        return decode(k, T), sets[name], None
    if name == "all_nan":                                       # every digit varies, and a share of NaNs (pairs: one collapsed key)
        k = radix_digit_keys(w, n, range(w), rng, pf)
        return decode(k, T, 0.05 if T.kind == "f" else 0.0, rng), tuple(range(w)), None
    if name.startswith("outlier"):
        where = name.split("_")[1]
        at, digit, larger = {"first": (0, w - 1, True), "last": (n - 1, 0, False), "tile": (min(tile, n - 1), 1, True)}[where]
        return decode(outlier_keys(w, n, digit, at, larger, rng), T), (digit,), digit
    if name == "tile_digit":                                    # one tile: digit 0 is constant
        return decode(tile_digit_keys(w, n, tile, rng, pf), T), tuple(range(w) if n > tile else range(1, w)), None
    raise ValueError(name)


def check_premise(a, want_active, outlier, pairs=False):
    r = pairs_radix(a) if pairs else keys_radix(a)
    assert active_digits(r) == tuple(want_active), (active_digits(r), want_active)
    if outlier is not None:
        assert largest_bin(r, outlier) == a.size - 1


SMALL_NAMES = ["none", "low", "top", "low_top", "odd", "even", "all", "all_nan", "outlier_first", "outlier_last", "outlier_tile", "tile_digit"]
PHASES = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)]          # (source, out, tmp) pointer phase in elements


def small_sizes(tile):
    """One ragged tile (n > 1024, so not the rank sort) and a few tiles, with last-tile remainders that are bulk-copied (a multiple of
    16 bytes; pairs: of 4 keys) and plain-loaded."""
    one = [1025, 1028, tile // 2 + 2, tile - 1]
    few = [5 * tile + r for r in (0, 1, 2, 3, 4, tile - 1)]
    return one + few


@pytest.mark.parametrize("T", DTYPES, ids=lambda t: np.dtype(t).name)
def test_sort_digit_sets_small(dab, rt1, T):
    """K11 on one ragged tile and on a few tiles: every digit set, out of place and in place, rotating the pointer phases."""
    rng = np.random.default_rng(1100 + np.dtype(T).itemsize + (np.dtype(T).kind == "f"))
    tile = KEYS_TILE[np.dtype(T).itemsize]
    k = 0
    for n in small_sizes(tile):
        for name in SMALL_NAMES:
            a, act, outl = make_case(T, name, n, tile, rng)
            check_premise(a, act, outl)
            want = model_sort(a)
            for inplace in (False, True):
                ip, op, tp = PHASES[k % len(PHASES)]
                k += 1
                got = run_sort(dab, rt1, a, inplace, ip, op, tp)
                assert np.array_equal(got.view(want.dtype), want), (name, n, inplace, ip, op, tp)


@pytest.mark.parametrize("T", DTYPES, ids=lambda t: np.dtype(t).name)
def test_sort_pairs_digit_sets_small(dab, rt1, T):
    """K21 on one ragged tile and on a few tiles: every digit set (collapsed keys), generated and given values, in place, misaligned keys."""
    rng = np.random.default_rng(1200 + np.dtype(T).itemsize + (np.dtype(T).kind == "f"))
    tile = PAIRS_TILE[np.dtype(T).itemsize]
    k = 0
    for n in small_sizes(tile):
        for name in SMALL_NAMES:
            a, act, outl = make_case(T, name, n, tile, rng, pairs=True)
            check_premise(a, act, outl, pairs=True)
            perm, ek = model_pairs(a)
            vals = rng.permutation(n).astype(np.int64) * 5 - (1 << 40)
            variants = [dict(base=(1 << 33) + 7, in_phase=k % 2), dict(vals=vals, out_phase=(k + 1) % 2), dict(base=1, inplace=True)]
            k += 1
            for v in variants:
                got_k, got_v = run_pairs(dab, rt1, a, **v)
                check_pairs(a, perm, ek, v.get("vals"), v.get("base", 0), got_k, got_v)


# ---- the persistent size class: at least TILES_PER_CTA tiles for every resident CTA -------------------------------------------
def _persistent_n(rt, tile, r):
    """TILES_PER_CTA full tiles for every CTA the device holds at once, then a last tile of r keys."""
    sm = rt.device_info()["sm_count"]
    full = TILES_PER_CTA * CTAS_PER_SM * sm
    n = full * tile + r
    ntiles = -(-n // tile)
    assert ntiles > CTAS_PER_SM * sm and ntiles >= full
    return n


def _skip_gpu_sized():
    if HOSTMEM:
        pytest.skip("a GPU-sized case: over a thousand tiles")


# name, last-tile remainder (as a function of the tile), variants as (inplace, source, out, tmp phase)
KEYS_PERSISTENT = [
    ("all_nan", lambda t: t - 1, [(False, 1, 0, 0), (True, 0, 0, 0)]),       # every pass; in place with an even pass count
    ("odd", lambda t: 1, [(True, 0, 0, 1), (False, 0, 1, 0)]),             # first pass not digit 0, last not the top: in place stages in tmp
    ("even", lambda t: 0, [(True, 1, 0, 0), (False, 0, 0, 1)]),
    ("none", lambda t: 3, [(True, 0, 0, 0), (False, 0, 1, 0)]),            # no pass: the copy kernel, or nothing at all in place
    ("outlier_tile", lambda t: 2, [(False, 0, 0, 1), (True, 0, 0, 0)]),   # one key off in digit 1, at the first index of tile 1
    ("tile_digit", lambda t: 4, [(False, 1, 0, 0)]),
]


@pytest.mark.parametrize("T", DTYPES, ids=lambda t: np.dtype(t).name)
def test_sort_persistent(dab, rt1, T):
    """K11 with at least 4 tiles for every resident CTA: every CTA runs its tile loop past the first ticket (the bulk prefetch of the next
    tile during the look-back, the mbarrier phase flip, the reuse of the counters), on every digit set class, every pointer phase, in
    place (odd, even and no passes) and out of place, and on sorted, reversed and one-digit-per-tile input."""
    _skip_gpu_sized()
    T = np.dtype(T)
    tile = KEYS_TILE[T.itemsize]
    rng = np.random.default_rng(1300 + T.itemsize + (T.kind == "f"))
    for name, rem, variants in KEYS_PERSISTENT:
        n = _persistent_n(rt1, tile, rem(tile))
        a, act, outl = make_case(T, name, n, tile, rng)
        check_premise(a, act, outl)
        want = model_sort(a)
        for inplace, ip, op, tp in variants:
            got = run_sort(dab, rt1, a, inplace, ip, op, tp)
            assert np.array_equal(got.view(want.dtype), want), (name, n, inplace, ip, op, tp)
        if name == "all_nan":                                   # skewed look-back: the sorted keys, then reversed
            srt = want.view(T)
            assert np.array_equal(run_sort(dab, rt1, srt).view(want.dtype), want)
            rev = srt[::-1].copy()
            assert np.array_equal(run_sort(dab, rt1, rev, False, 0, 1, 0).view(want.dtype), want)
        del a, want


PAIRS_PERSISTENT = [
    ("all_nan", lambda t: t - 1, [dict(base=(1 << 33) + 3, in_phase=1), dict(vals=True), dict(base=5, inplace=True)]),
    ("odd", lambda t: 2, [dict(base=(1 << 34) + 1, inplace=True), dict(vals=True, out_phase=1)]),
    ("none", lambda t: 4, [dict(base=(1 << 33) + 9, inplace=True), dict(vals=True, in_phase=1)]),
    ("tile_digit", lambda t: 0, [dict(base=(1 << 35) - 1)]),
]


@pytest.mark.parametrize("T", DTYPES, ids=lambda t: np.dtype(t).name)
def test_sort_pairs_persistent(dab, rt1, T):
    """K21 with at least 4 tiles for every resident CTA: generated values above 2^33 and given values, in place (odd, even, no passes),
    misaligned keys in and out, and sorted / reversed input."""
    _skip_gpu_sized()
    T = np.dtype(T)
    tile = PAIRS_TILE[T.itemsize]
    rng = np.random.default_rng(1400 + T.itemsize + (T.kind == "f"))
    for name, rem, variants in PAIRS_PERSISTENT:
        n = _persistent_n(rt1, tile, rem(tile))
        a, act, outl = make_case(T, name, n, tile, rng, pairs=True)
        check_premise(a, act, outl, pairs=True)
        perm, ek = model_pairs(a)
        vals = rng.permutation(n).astype(np.int64) * 3 - (1 << 45)
        for v in variants:
            v = dict(v, vals=vals if v.get("vals") else None)
            got_k, got_v = run_pairs(dab, rt1, a, **v)
            check_pairs(a, perm, ek, v["vals"], v.get("base", 0), got_k, got_v)
        if name == "all_nan":                                   # skewed look-back: sorted input (the identity), then reversed
            srt = a[perm]
            got_k, got_v = run_pairs(dab, rt1, srt, base=(1 << 33))
            check_pairs(srt, np.arange(n), ek, None, 1 << 33, got_k, got_v)
            rev = srt[::-1].copy()
            rperm, rek = model_pairs(rev)
            got_k, got_v = run_pairs(dab, rt1, rev, vals=vals, in_phase=1)
            check_pairs(rev, rperm, rek, vals, 0, got_k, got_v)


def test_sort_by_key_persistent_f64(dab, rt1):
    """dab_sort_by_key with Float64 keys (two K11 rounds on Int64 words) at the persistent size, many ties and NaNs of several payloads."""
    _skip_gpu_sized()
    from darray_b200 import _lib
    rng = np.random.default_rng(1500)
    n = _persistent_n(rt1, KEYS_TILE[8], 5)
    keys = np.round(rng.standard_normal(n) * 100.0, 1)
    keys[rng.integers(0, n, n // 20)] = np.nan
    keys[rng.integers(0, n, n // 50)] = -np.nan
    raw = keys.view(np.uint64)
    pick = rng.integers(0, n, n // 50)
    raw[pick] = np.uint64(0x7FF0000000000000) | rng.integers(1, 1 << 51, pick.size, dtype=np.int64).astype(np.uint64)
    keys[rng.integers(0, n, n // 50)] = -0.0
    vals = rng.permutation(n).astype(np.int64)
    want = vals[orc.jl_sortperm_stable(keys)]
    dk, dv = Guarded(dab, rt1, np.float64, n, 0, keys, 21), Guarded(dab, rt1, np.int64, n, 0, vals, 22)
    out = Guarded(dab, rt1, np.int64, n, 0, None, 23)
    need = C.c_size_t()
    _lib.check(_lib.lib().dab_sort_by_key_scratch_bytes(dab.dab_dtype(np.float64), n, C.byref(need)))
    scratch = Guarded(dab, rt1, np.uint8, need.value, 0, None, 24)
    _lib.call("dab_sort_by_key", rt1.ctx, dab.dab_dtype(np.float64), C.c_void_p(dk.ptr), 8, C.c_void_p(dv.ptr), C.c_void_p(out.ptr),
              C.c_void_p(scratch.ptr), need.value, n)
    assert np.array_equal(out.read(), want)
    scratch.check_guards()
    assert np.array_equal(dk.read().view(np.uint64), keys.view(np.uint64)) and np.array_equal(dv.read(), vals)
    for b in (dk, dv, out, scratch):
        b.free()


def test_public_sort_and_sortperm_persistent(dab, rt1):
    """sort(d) and sortperm(d) of a one-chunk Float32 DVector at the persistent size of K11 (and twice that of K21): exact."""
    _skip_gpu_sized()
    rng = np.random.default_rng(1600)
    n = _persistent_n(rt1, KEYS_TILE[4], 7)
    a = (rng.standard_normal(n) * 10.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    a[rng.integers(0, n, n // 100)] = np.round(a[rng.integers(0, n, n // 100)], 0)   # ties
    a[rng.integers(0, n, 64)] = [np.inf, -np.inf, 0.0, -0.0] * 16
    d = dab.distribute(a)
    assert len(d.layout.pids) == 1
    s = dab.sort(d)
    assert np.array_equal(dab.to_array(s).view(np.uint32), model_sort(a))
    s.close()
    p = dab.sortperm(d)
    perm, _ = model_pairs(a)
    assert np.array_equal(dab.to_array(p), perm.astype(np.int64) + 1)
    p.close()
    d.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------------
def test_sort_refusals_launch_nothing(dab, rt1):
    """Arguments the sort refuses at the ABI, each before any launch, with every buffer left as it was: chunks of 0xFFFFF000 or more
    keys (no buffer of that size exists: the length is refused first), tmp aliasing in or out, no tmp, and the in-place rank sort
    without tmp."""
    from darray_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(1700)
    n = 4096
    a = rng.standard_normal(n)
    bufs = [Guarded(dab, rt1, np.float64, n, 0, a, 30 + j) for j in range(4)]
    x, y, z, w = (C.c_void_p(b.ptr) for b in bufs)
    f64 = dab.dab_dtype(np.float64)
    cases = [                                                   # the scratch length passed is the buffer's: the chunk length is refused first
        (_lib.ERR_UNSUPPORTED, lambda: L.dab_sort(rt1.ctx, f64, x, y, z, NOT_SERVED)),
        (_lib.ERR_UNSUPPORTED, lambda: L.dab_sort(rt1.ctx, f64, x, x, z, NOT_SERVED)),
        (_lib.ERR_UNSUPPORTED, lambda: L.dab_sort_pairs(rt1.ctx, f64, x, y, None, 0, z, w, 8 * n, NOT_SERVED)),
        (_lib.ERR_UNSUPPORTED, lambda: L.dab_sort_by_key(rt1.ctx, f64, x, 8, y, z, w, 8 * n, NOT_SERVED)),
        (_lib.ERR_ARG, lambda: L.dab_sort(rt1.ctx, f64, x, y, x, n)),      # tmp == in
        (_lib.ERR_ARG, lambda: L.dab_sort(rt1.ctx, f64, x, y, y, n)),      # tmp == out
        (_lib.ERR_ARG, lambda: L.dab_sort(rt1.ctx, f64, x, x, x, n)),      # in place, tmp == in == out
        (_lib.ERR_ARG, lambda: L.dab_sort(rt1.ctx, f64, x, y, None, n)),   # no tmp
        (_lib.ERR_ARG, lambda: L.dab_sort(rt1.ctx, f64, x, x, None, 1000)),   # in-place rank sort without tmp
    ]
    for k, (status, f) in enumerate(cases):
        l0 = rt1.launches()
        assert f() == status, k
        assert rt1.launches() == l0, k
    for b in bufs:
        assert np.array_equal(b.read(), a)
        b.free()


# ---- past 2^31 keys ---------------------------------------------------------------------------------------------------------------
def test_sort_past_2_31_in_place_int32(dab, rt1):
    """K11 in place on n = 2^31 + 4099 Int32 keys (the last tile plain-loaded: 4099 keys are not a multiple of 16 bytes): the 32-bit
    bucket bases, look-back counts and output offsets past 2^31.  The keys (a i mod n) - 2^30, a coprime to n, are a permutation of
    (0:n-1) - 2^30, so the sorted result is known without a host sort."""
    if HOSTMEM:
        pytest.skip("a GPU-sized case: 2^31 keys")
    from darray_b200 import _lib
    n = (1 << 31) + 4099
    if rt1.device_info()["free_bytes"] < 20 * 2 ** 30:
        pytest.skip("needs 20 GiB of free device memory")
    a = 2654435761
    assert math.gcd(a, n) == 1 and n % KEYS_TILE[4] == 4099 and (4099 * 4) % 16 != 0
    keys = dab.B200Array.empty(rt1, (n,), np.int32)
    tmp = dab.B200Array.empty(rt1, (n,), np.int32)
    step = 1 << 26
    for lo in range(0, n, step):
        i = np.arange(lo, min(n, lo + step), dtype=np.int64)
        h = ((a * i) % n - (1 << 30)).astype(np.int32)
        _lib.call("dab_h2d", rt1.ctx, C.c_void_p(keys.ptr + 4 * lo), C.c_void_p(h.ctypes.data), h.nbytes)
        rt1.sync()
    del i, h
    _lib.call("dab_sort", rt1.ctx, dab.dab_dtype(np.int32), C.c_void_p(keys.ptr), C.c_void_p(keys.ptr), C.c_void_p(tmp.ptr), n)
    tmp.free()
    got = np.empty(step, dtype=np.int32)
    for lo in range(0, n, step):
        c = min(step, n - lo)
        _lib.call("dab_d2h", rt1.ctx, C.c_void_p(got.ctypes.data), C.c_void_p(keys.ptr + 4 * lo), 4 * c)
        rt1.sync()
        want = np.arange(lo - (1 << 30), lo + c - (1 << 30), dtype=np.int32)
        assert np.array_equal(got[:c], want), lo
    keys.free()
