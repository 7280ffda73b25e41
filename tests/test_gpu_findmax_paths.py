"""GPU tests of findmax / findmin (K20, ``dab_findminmax.cu``) on every launch path of its kernels, bit for bit against the model of
Julia's loops (tests/findmax_oracle.py), through the C entries ``dab_findminmax_dim`` and ``dab_findminmax``.

Which kernel runs is decided on the host (``launch_fmdim``, ``dim_nsplit``, ``flat_grid``), so every case is built to reach one path of
``fo.fmdim_plan`` / ``fo.flat_grid`` and asserts that premise first: the whole-chunk kernel, the lead kernel with 4 or 32 lanes per run,
the strided kernel and its 16-byte form, each with and without a split of the reduced extent (then the finish fold), each lead and
strided kernel with an index input (a later pass, and the fold on the owner), an empty split, and persistent grids that loop.

Correctness rests on one comparison, "larger key, then smaller index", applied alike in the walks, the shuffle tree, the CTA tree and
the finish fold.  Random data with many ties hides a "<" turned "<=" most of the time, so each fibre gets a designed winner: at the first
or last position of a split, with an equal-key twin later (in the next split, in the same unrolled group, in another lane of the same
group); NaNs of both signs and distinct payloads beside +-Inf; -0.0 against +0.0 in both orders; a fibre of nothing but the lowest key,
which must still beat the empty accumulator.  The model's winner is asserted to be the designed one before the kernel runs.

Operands sit 0 .. VPT-1 elements past a 256-byte boundary, with sentinel bytes before and after in the same allocation; after every
call the sentinels of the outputs are checked and the inputs must be unchanged."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import findmax_oracle as fo

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets the K20 entry points too
    fo.install()

DTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_]
IDS = lambda t: np.dtype(t).name
MAP_ID, MAP_ABS, MAP_ABS2 = 0, 1, 2
MAPF = {MAP_ID: None, MAP_ABS: np.abs, MAP_ABS2: lambda x: x * x}
GUARD = 256                                                     # sentinel bytes on either side of a buffer


def _lib():
    from darray_b200 import _lib
    return _lib


def _vpt(dt) -> int:
    return 16 // np.dtype(dt).itemsize


# ---- device buffers between guard bands -------------------------------------------------------------------------------------------
class Buf:
    """``data`` (or n uninitialised elements of ``dtype``) placed ``phase`` elements past a 256-byte boundary, GUARD random bytes
    before and after it, in one allocation."""

    def __init__(self, dab, rt, data=None, phase=0, dtype=None, n=0, seed=0):
        self.rt = rt
        self.dt = np.dtype(data.dtype if data is not None else dtype)
        self.n = int(data.size if data is not None else n)
        self.lo = GUARD + phase * self.dt.itemsize
        self.nbytes = self.n * self.dt.itemsize
        g = np.random.default_rng(seed + 7919 * self.n + phase)
        self.image = g.integers(0, 256, self.lo + self.nbytes + GUARD, dtype=np.uint8)
        if data is not None:
            self.image[self.lo:self.lo + self.nbytes] = np.ascontiguousarray(data).view(np.uint8).ravel()
        self.buf = dab.B200Array.empty(rt, (self.image.size,), np.uint8)
        assert self.buf.ptr % 256 == 0
        self.ptr = self.buf.ptr + self.lo
        _lib().call("dab_h2d", rt.ctx, C.c_void_p(self.buf.ptr), C.c_void_p(self.image.ctypes.data), self.image.size)
        rt.sync()

    def _all(self) -> np.ndarray:
        out = np.empty(self.image.size, dtype=np.uint8)
        _lib().call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.buf.ptr), out.size)
        self.rt.sync()
        return out

    def unchanged(self) -> bool:
        return np.array_equal(self._all(), self.image)

    def read(self) -> np.ndarray:
        """The data, after checking that nothing outside it was written."""
        got = self._all()
        assert np.array_equal(got[:self.lo], self.image[:self.lo]), "a store before the output"
        assert np.array_equal(got[self.lo + self.nbytes:], self.image[self.lo + self.nbytes:]), "a store past the end of the output"
        return got[self.lo:self.lo + self.nbytes].view(self.dt).copy()

    def free(self):
        self.buf.free()


def _i64s(v):
    return (C.c_int64 * max(len(v), 1))(*[int(a) for a in v])


def run_dims(dab, rt, x3, which, mapc, phase=0, ii3=None, geom=((), (), ())):
    """dab_findminmax_dim over axis 1 of the (inner, red, outer) array x3 through guarded buffers: (values, indices, launches)."""
    inner, red, outer = x3.shape
    nout = inner * outer
    cd, off, gd = geom
    xb = Buf(dab, rt, x3.ravel(order="F"), phase, seed=1)
    ib = Buf(dab, rt, ii3.ravel(order="F"), 0, seed=2) if ii3 is not None else None
    ov, oi = Buf(dab, rt, None, 0, x3.dtype, nout, seed=3), Buf(dab, rt, None, 0, np.int64, nout, seed=4)
    l0 = rt.launches()
    st = _lib().lib().dab_findminmax_dim(rt.ctx, dab.dab_dtype(x3.dtype), which, mapc, C.c_void_p(xb.ptr), C.c_void_p(ib.ptr) if ib else None,
                                         inner, red, outer, len(cd), _i64s(cd), _i64s(off), _i64s(gd), C.c_void_p(ov.ptr), C.c_void_p(oi.ptr))
    _lib().check(st, rt.ctx)
    launches = rt.launches() - l0
    vals, idx = ov.read(), oi.read()
    assert xb.unchanged(), "x was written"
    assert ib is None or ib.unchanged(), "idx_in was written"
    for b in (xb, ib, ov, oi):
        if b is not None:
            b.free()
    return vals.reshape((inner, outer), order="F"), idx.reshape((inner, outer), order="F"), launches


def same(got, want, mapc) -> bool:
    """Bit for bit; after abs2 (x * x on the GPU's FP units) a NaN is only required to be a NaN."""
    got, want = np.asarray(got), np.asarray(want)
    if mapc != MAP_ABS2 or want.dtype.kind != "f":
        return fo.same_bits(got, want)
    nan = np.isnan(want)
    return got.dtype == want.dtype and np.array_equal(np.isnan(got), nan) and fo.same_bits(got[~nan], want[~nan])


def check_launches(plan, launches, what):
    if not HOSTMEM:                                             # the emulation counts one launch per entry
        assert launches == plan["launches"], (what, launches, plan["launches"])


# ---- values -----------------------------------------------------------------------------------------------------------------------
def nan_bits(dt, payload, neg=False):
    dt, payload = np.dtype(dt), int(payload)
    if dt == np.float32:
        return np.array([(0xFF800000 if neg else 0x7F800000) | payload], dtype=np.uint32).view(np.float32)[0]
    return np.array([(0xFFF0000000000000 if neg else 0x7FF0000000000000) | payload], dtype=np.uint64).view(np.float64)[0]


def lows(rng, dt, shape):
    """Background values: magnitudes 10 .. 50 of either sign, in quarter steps for floats, many ties."""
    dt = np.dtype(dt)
    if dt == np.bool_:
        raise TypeError
    m = rng.integers(40, 201, shape)
    s = np.where(rng.random(shape) < 0.5, -1, 1)
    return ((m * s) / 4).astype(dt) if dt.kind == "f" else (m // 4 * s).astype(dt)


def top_pair(dt, which, mapc):
    """(winner, twin): an equal order key after the map, above every background value."""
    if np.dtype(dt) == np.bool_:
        return (True, True) if which == fo.FINDMAX else (False, False)
    if which == fo.FINDMAX:
        return (100, 100) if mapc == MAP_ID else (-100, 100)
    return (-100, -100) if mapc == MAP_ID else (3, -3)


def worst(dt, which):
    dt = np.dtype(dt)
    if dt == np.bool_:
        return which == fo.FINDMIN
    if dt.kind == "f":
        return -np.inf if which == fo.FINDMAX else np.inf
    return np.iinfo(dt).min if which == fo.FINDMAX else np.iinfo(dt).max


def wrap_pool(dt):
    """Int32 / Int64 values where abs and abs2 wrap: abs(typemin) == typemin, squares past typemax."""
    info = np.iinfo(dt)
    big = [46341, 65536, 3] if np.dtype(dt) == np.int32 else [3037000500, 1 << 32, 3]
    return np.array([info.min, info.min + 1, info.max, 0] + big + [-b for b in big], dtype=dt)


def scenarios(dt, which, mapc, has_idx):
    dt = np.dtype(dt)
    if has_idx:
        out = ["order", "minus1", "one_valid", "split_none", "lowest"]
        return out + (["dup"] if dt.kind == "f" else [])
    out = ["plain", "lowest"]
    if dt.kind == "f":
        out += ["nan"] + (["zero"] if mapc == MAP_ID else [])
    if dt.kind == "i" and mapc != MAP_ID:
        out.append("wrap")
    return out


def deciding_positions(plan, red):
    """The bounds (lo and hi - 1) of every non-empty split, or of the first two, the middle and the last two of more than 64, and the ends
    of the run."""
    live = [(lo, hi) for lo, hi in plan["bounds"] if hi > lo]
    pick = set(range(len(live))) if len(live) <= 64 else {0, 1, len(live) // 2, len(live) - 1, len(live) - 2}
    pos = {0, red - 1}
    for s in pick:
        if 0 <= s < len(live):
            pos |= {live[s][0], live[s][1] - 1}
    if plan["kernel"] == "whole":
        t = plan["flat"]["tile"]
        pos |= {p for p in (t - 1, t, 2 * t - 1, 2 * t, 3 * t, red - 2) if 0 <= p < red}
    return sorted(pos)


def twin_deltas(plan, red, p, dup=False):
    """Offsets of an equal-key twin after position p: in the next split, in the same unrolled group, in another lane of the same group
    (lead), the neighbouring element of a 16-byte vector (whole).  ``dup``: only offsets that stay in p's lane or leave its split, where
    the walk order is the position order."""
    nxt = [lo for lo, hi in plan["bounds"] if hi > lo and lo > p]
    k = plan["kernel"]
    if k == "lead":
        G = plan["G"]
        d = [G, 4 * G] if dup else [G, 1, 4 * G - 1]
    elif k == "whole":
        d = [1, plan["flat"]["vpt"], plan["flat"]["tile"]]
    else:
        d = [1, 7, 8]
    d = d + ([nxt[0] - p] if nxt else [])
    return [v for v in d if 0 < p + v < red]


def split_of(plan, p):
    for lo, hi in plan["bounds"]:
        if lo <= p < hi:
            return lo, hi
    raise ValueError(p)


def design(rng, dt, which, mapc, plan, inner, red, outer, has_idx, t0):
    """(x3, ii3 or None, designed winner position per fibre, -1 where the model alone decides).  Fibre f takes combination t0 + f of
    (deciding position, twin offset, scenario)."""
    dt = np.dtype(dt)
    nf = inner * outer
    P = deciding_positions(plan, red)
    scen = scenarios(dt, which, mapc, has_idx)
    M = np.full((nf, red), which == fo.FINDMIN) if dt == np.bool_ else lows(rng, dt, (nf, red))   # every background element loses
    ii = None
    if has_idx:
        base = (1 << 62) - nf * red - 7 if (t0 // nf) % 2 else 1
        ii = base + rng.permutation(nf * red).reshape(nf, red).astype(np.int64)    # distinct, in no positional order
    W, W2 = top_pair(dt, which, mapc)
    want = np.full(nf, -1, dtype=np.int64)
    fibres = np.arange(nf)
    if nf > 3072:                                                # the first, some middle and the last fibres; the model decides the rest
        fibres = np.unique(np.concatenate([fibres[:1024], rng.choice(nf, 1024, replace=False), fibres[-1024:]]))
    pair = plan["kernel"] in ("strided", "vec")                  # fibres 2k and 2k + 1 alike: equal keys at one r in neighbouring lanes
    for f in fibres.tolist():
        t = t0 + f
        u = t0 + f // 2 if pair else t
        p = P[u % len(P)]
        sc = scen[(u // len(P) + u) % len(scen)]
        ds = twin_deltas(plan, red, p, dup=sc == "dup")
        q = p + ds[(u // 3) % len(ds)] if ds else None
        row = M[f]
        if sc == "lowest":
            row[:] = worst(dt, which)
            want[f] = int(np.argmin(ii[f])) if has_idx else 0
            continue
        if sc == "wrap":
            row[:] = rng.choice(wrap_pool(dt), red)
            continue
        if sc == "plain" or sc == "order" or sc == "minus1" or sc == "split_none":
            row[p] = W
            if q is not None:
                row[q] = W2
            want[f] = p
        if sc == "nan":
            neg = bool(t % 2)
            for j in (p - 1, p + 1):
                if 0 <= j < red:
                    row[j] = np.inf if (j < p) != neg else -np.inf
            row[p] = nan_bits(dt, 5 + t % 7, neg)
            if q is not None:
                row[q] = nan_bits(dt, 17 + t % 5, not neg)
            want[f] = p
        if sc == "zero":
            pos_zero = which == fo.FINDMAX
            row[:] = np.abs(row) * (-1 if pos_zero else 1)       # every background value below +0.0 (findmax) / above -0.0 (findmin)
            row[p] = 0.0 if pos_zero else -0.0
            for j in (p - 1, q):                                 # the other zero before and after the winner
                if j is not None and 0 <= j < red:
                    row[j] = -0.0 if pos_zero else 0.0
            want[f] = p
        if not has_idx:
            continue
        if sc == "order" and q is not None:                      # an equal key later with a smaller carried index wins
            lo_, hi_ = sorted((ii[f, p], ii[f, q]))
            ii[f, p], ii[f, q] = hi_, lo_
            want[f] = q
        elif sc == "minus1":                                     # the would-be winner carries -1: the twin, or the model, decides
            ii[f, p] = -1
            want[f] = q if q is not None else -1
        elif sc == "one_valid":                                  # everything but one entry is "no element"
            ii[f, :] = -1
            ii[f, p] = (1 << 62) + t
            want[f] = p
        elif sc == "split_none":                                 # the winner's whole split (or a run of 8) is "no element"
            lo_, hi_ = split_of(plan, p) if plan["nsplit"] > 1 else (p, min(p + 8, red))
            ii[f, lo_:hi_] = -1
            r2 = q if q is not None and not lo_ <= q < hi_ else hi_ if hi_ < red else lo_ - 1 if lo_ > 0 else None
            if r2 is not None:
                row[r2] = W2
            want[f] = -1 if r2 is None else r2
        elif sc == "dup" and q is not None:                      # NaNs of two payloads carrying one index: the earlier one is kept
            row[p] = nan_bits(dt, 9, bool(t % 2))
            row[q] = nan_bits(dt, 10, not t % 2)
            ii[f, q] = ii[f, p]
            want[f] = p
    x3 = M.reshape((outer, inner, red)).transpose(1, 2, 0)
    x3 = np.asfortranarray(x3)
    ii3 = np.asfortranarray(ii.reshape((outer, inner, red)).transpose(1, 2, 0)) if has_idx else None
    return x3, ii3, want.reshape((outer, inner)).T


def model(which, mapc, x3, ii3, geom=((), (), ())):
    """(values, 1-based global or carried indices, winning position along red) of every fibre, each (inner, outer)."""
    inner, red, outer = x3.shape
    if ii3 is not None:
        v, i = fo.find_carried(which, x3, ii3)
        return v, i, None
    v, i = fo.find_dims(which, x3, 2, MAPF[mapc])
    pos0 = i.reshape((inner, outer), order="F") - 1
    return v.reshape((inner, outer), order="F"), fo.global_index(pos0, *geom), (pos0 // inner) % red


def check_case(dab, rt, rng, dt, which, mapc, plan, inner, red, outer, phase, has_idx, t0, what, geom=((), (), ())):
    x3, ii3, want = design(rng, dt, which, mapc, plan, inner, red, outer, has_idx, t0)
    wv, wi, wpos = model(which, mapc, x3, ii3, geom)
    d = want >= 0
    if ii3 is not None:                                          # the premise: the designed winner is the model's
        I, O = np.nonzero(d)
        assert np.array_equal(wi[d], ii3[I, want[d], O]), what
    else:
        assert np.array_equal(wpos[d], want[d]), what
    gv, gi, launches = run_dims(dab, rt, x3, which, mapc, phase, ii3, geom)
    assert same(gv, wv, mapc), (what, np.nonzero(gv.view(np.uint8) != wv.view(np.uint8)))
    bad = np.nonzero(gi != wi)
    assert not bad[0].size, (what, bad[0][:5], bad[1][:5], gi[bad][:5], wi[bad][:5])
    check_launches(plan, launches, what)


def _sm(rt):
    return rt.device_info()["sm_count"]


def _table(rt):
    """The case table at this device's SM count; a device (or partition) of fewer than fo.MIN_SM_COUNT SMs cannot split a pass into
    enough splits to leave one empty, so the table's tests skip there."""
    sm = _sm(rt)
    if sm < fo.MIN_SM_COUNT:
        pytest.skip(f"the case table needs {fo.MIN_SM_COUNT} or more SMs, the device has {sm}")
    return fo.case_table(sm)


def _case_premise(case, dt, sm):
    name, want, shape, idx = case
    labels = fo.case_labels(case, dt, sm)
    if np.dtype(dt) == np.bool_ and want in ("vec", "vec_split"):
        want = "bool_vec_shape"                                 # Bool never takes the 16-byte kernel
    assert want in labels, (name, IDS(dt), labels)
    if want == "bool_vec_shape":
        assert not any(l.startswith("vec") for l in labels)
    return labels


# ---- the case table ---------------------------------------------------------------------------------------------------------------
def test_case_table_reaches_every_path(rt1):
    """Every label of the launch model is reached by the case table at this device's SM count, each case on its premise."""
    table = _table(rt1)
    sm = _sm(rt1)
    seen = set()
    for case in table:
        for dt in DTYPES:
            seen |= _case_premise(case, dt, sm)
    assert fo.ALL_LABELS <= seen, fo.ALL_LABELS - seen


def _combos(dt, has_idx):
    maps = [MAP_ID] if has_idx else [MAP_ID, MAP_ABS, MAP_ABS2]
    return [(w, m) for w in (fo.FINDMAX, fo.FINDMIN) for m in maps]


def _run_case(dab, rt, case, dt):
    sm = _sm(rt)
    _case_premise(case, dt, sm)
    name, _, shape, has_idx = case
    inner, red, outer, phase = shape(dt)
    plan = fo.fmdim_plan(dt, inner, red, outer, (phase * np.dtype(dt).itemsize) % 16, has_idx, sm)
    nf = inner * outer
    P = len(deciding_positions(plan, red))
    combos = _combos(dt, has_idx)
    rounds = min(40, -(-2 * P // (len(combos) * nf)))            # every deciding position at least once per dtype
    rng = np.random.default_rng(zlib.crc32(f"{name}/{IDS(dt)}".encode()))
    for c, (which, mapc) in enumerate(combos):
        for r in range(rounds):
            check_case(dab, rt, rng, dt, which, mapc, plan, inner, red, outer, phase, has_idx, (c * rounds + r) * nf,
                       (name, IDS(dt), which, mapc, r))


SMALL = [c for c in fo.case_table(132) if c[0] in ("lead4_red63", "lead32_red64", "lead32_split", "lead32_split_red65535", "whole_red65536",
                                                    "whole_misaligned", "strided", "strided_split", "vec_nout4096", "strided_nout4095",
                                                    "strided_inner_mod_vpt", "strided_base_misaligned")]
IDX = [c for c in fo.case_table(132) if c[3]]


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", [c[0] for c in SMALL])
def test_dims_paths(dab, rt1, name, dt):
    """Each launch path without an index input: every map, findmax and findmin, designed winners and twins on the split bounds."""
    case = next(c for c in _table(rt1) if c[0] == name)
    _run_case(dab, rt1, case, dt)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", [c[0] for c in IDX])
def test_dims_paths_with_index_input(dab, rt1, name, dt):
    """Each lead and strided path with carried indices: -1 entries (the would-be winner, all but one, a whole split), carried indices out
    of positional order and near 2^62, a full tie of two NaNs carrying one index, an empty split."""
    case = next(c for c in _table(rt1) if c[0] == name)
    _run_case(dab, rt1, case, dt)


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", ["strided_empty_split", "lead4_loop", "lead32_loop", "strided_loop", "vec_split", "strided_split_nout4095",
                                  "vec_loop"])
def test_dims_large_paths(dab, rt1, name, dt):
    """The paths that need more work: 1024 splits of which the last are empty, persistent grids that loop, the 16-byte kernel with a
    split, and the strided split at nout / VPT = 4095."""
    case = next(c for c in _table(rt1) if c[0] == name)
    _run_case(dab, rt1, case, dt)


# ---- the position -> global index map ---------------------------------------------------------------------------------------------
def _factor_dims(rng, n, nd):
    """nd chunk dims whose product is n: n's prime factors spread at random, 1 where none falls."""
    if nd == 0:
        return []
    dims = [1] * nd
    p, m = 2, n
    while m > 1:
        while m % p == 0:
            dims[int(rng.integers(0, nd))] *= p
            m //= p
        p += 1 if p == 2 else 2
        if p * p > m and m > 1:
            dims[int(rng.integers(0, nd))] *= m
            m = 1
    return dims


def test_global_index_map_over_0_to_8_dims(dab, rt1):
    """FmGlobal with nd = 0 .. 8 chunk dims at random offsets inside larger global dims, on the paths that apply it (the direct store,
    the finish fold, the whole-chunk slot), and one case whose global indices pass 2^40."""
    sm = _sm(rt1)
    rng = np.random.default_rng(40)
    shapes = [(1, 64, 37), (1, 2048 * 6 + 5, 3), (5, 256 * 8 + 3, 7), (3, 300, 5), (1, 65536, 1), (24, 3, 512)]
    for nd in range(9):
        for k, dt in enumerate(DTYPES):
            inner, red, outer = shapes[(nd + k) % len(shapes)]
            cd = _factor_dims(rng, inner * red * outer, nd)
            off = [int(v) for v in rng.integers(0, 50, nd)]
            gd = [c + o + int(e) for c, o, e in zip(cd, off, rng.integers(0, 9, nd))]
            plan = fo.fmdim_plan(dt, inner, red, outer, 0, False, sm)
            for which in (fo.FINDMAX, fo.FINDMIN):
                check_case(dab, rt1, rng, dt, which, MAP_ID, plan, inner, red, outer, 0, False, nd * 7 + which, ("nd", nd, IDS(dt)),
                           (cd, off, gd))
    for inner, red, outer in ((6, 50, 7), (1, 2048 * 6 + 5, 3), (1, 65536, 1)):            # indices past 2^40
        n = inner * red * outer
        cd, off = [6, n // 6 // 7, 7] if n % 42 == 0 else [1, n, 1], [5, 3, (1 << 21) + 5]
        gd = [1 << 10, max(1 << 10, cd[1] + 3), 1 << 22]
        assert fo.global_index(np.array([n - 1]), cd, off, gd)[0] > 1 << 40
        plan = fo.fmdim_plan(np.float64, inner, red, outer, 0, False, sm)
        for which in (fo.FINDMAX, fo.FINDMIN):
            check_case(dab, rt1, rng, np.float64, which, MAP_ABS, plan, inner, red, outer, 0, False, which, ("2^40", inner, red, outer),
                       (cd, off, gd))


# ---- the whole-array entry ------------------------------------------------------------------------------------------------------
def run_whole(dab, rt, x, which, mapc, phase):
    """dab_findminmax on x placed ``phase`` elements past a 256-byte boundary: (16-byte slot, launches)."""
    xb = Buf(dab, rt, x, phase, seed=5)
    slot = Buf(dab, rt, None, 0, np.uint8, 16, seed=6)
    l0 = rt.launches()
    _lib().call("dab_findminmax", rt.ctx, dab.dab_dtype(x.dtype), which, mapc, None, C.c_void_p(xb.ptr), x.size, C.c_void_p(slot.ptr))
    launches = rt.launches() - l0
    s = slot.read()
    assert xb.unchanged(), "x was written"
    xb.free()
    slot.free()
    return s, launches


def whole_positions(fg, n):
    """(winner, twin) pairs: head vs body, the two tiles of one CTA, two CTAs, one 16-byte vector, a thread's unrolled loads, the
    remainder vectors and the tail."""
    h, T, v = fg["head"], fg["tile"], fg["vpt"]
    body = h + fg["tiles"] * T
    pairs = []
    if h:
        pairs += [(0, h), (h - 1, h + T - 1), (h - 1, n - 1)]
    pairs += [(h, h + 1), (h + v - 2, h + v - 1), (h + 3, h + 3 + 256 * v), (h + 7 * v + 1, h + T + 7 * v)]
    if fg["tiles"] >= 2:
        pairs += [(h + T - 1, h + T), (h + 2 * T - 1, body)]
    if fg["tiles"] >= 3:
        pairs += [(h + 2 * T - 1, h + 2 * T), (h + T + 5, h + 2 * T + 5)]
    if fg["rem_vecs"]:
        pairs += [(body, body + v), (body - 1, body)]
    if fg["tail"]:
        pairs += [(n - fg["tail"], n - 1), (body + fg["rem_vecs"] * v - 1, n - 1)]
    return [(p, q) for p, q in pairs if 0 <= p < q < n]


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_whole_array_every_head_length(dab, rt1, dt):
    """dab_findminmax at 1, 2 and 3 tiles (one CTA with one and two tiles, two CTAs) plus remainder vectors and a tail, at every head
    length: the winner and an equal-key twin across head and body, the tiles of one CTA, two CTAs, one 16-byte vector, a thread's
    unrolled loads; NaNs, signed zeros and the lowest key, which must beat the empty accumulator."""
    dt = np.dtype(dt)
    v = _vpt(dt)
    rng = np.random.default_rng(60 + v)
    T = v * fo.RD_THREADS * fo.RD_UNROLL
    for phase in range(v):
        for tiles in (1, 2, 3):
            head, tail = (v - phase) % v, 1 + phase % max(v - 1, 1)
            n = head + tiles * T + 3 * v + tail
            fg = fo.flat_grid(dt, phase * dt.itemsize, n)
            assert fg["head"] == head and fg["tiles"] == tiles and fg["rem_vecs"] == 3 and fg["tail"] == tail
            assert fg["grid"] == (1 if tiles <= 2 else 2) and fg["tiles_per_cta"] == 2
            pairs = whole_positions(fg, n)
            for c, (p, q) in enumerate(pairs):
                which, mapc = (fo.FINDMAX, fo.FINDMIN)[c % 2], (MAP_ID, MAP_ABS, MAP_ABS2)[(c // 2 + phase) % 3]
                sc = scenarios(dt, which, mapc, False)[(c + tiles) % len(scenarios(dt, which, mapc, False))]
                if dt == np.bool_:
                    x = np.full(n, which == fo.FINDMIN)
                else:
                    x = lows(rng, dt, n)
                W, W2 = top_pair(dt, which, mapc)
                want = p
                if sc == "lowest":
                    x[:] = worst(dt, which)
                    want = 0
                elif sc == "wrap":
                    x = rng.choice(wrap_pool(dt), n)
                    want = None
                elif sc == "nan":
                    x[p], x[q] = nan_bits(dt, 3 + c, c % 2 == 0), nan_bits(dt, 40 + c, c % 2 == 1)
                    x[max(p - 1, 0)] = np.inf if p else x[0]
                    if q + 1 < n:
                        x[q + 1] = -np.inf
                elif sc == "zero":
                    pos_zero = which == fo.FINDMAX
                    x = np.abs(x) * (-1 if pos_zero else 1)
                    x[p], x[q] = (0.0, -0.0) if pos_zero else (-0.0, 0.0)
                    if p:
                        x[p - 1] = -0.0 if pos_zero else 0.0
                else:
                    x[p], x[q] = W, W2
                x = x.astype(dt)
                wv, wi = fo.find(which, x, MAPF[mapc] if dt != np.bool_ else None)
                if want is not None:
                    assert wi == want, (p, q, sc)
                s, launches = run_whole(dab, rt1, x, which, mapc, phase)
                what = (IDS(dt), phase, tiles, p, q, sc, which, mapc)
                assert same(s[:dt.itemsize].view(dt), np.asarray([wv], dtype=dt), mapc), (what, s, wv)
                assert not s[dt.itemsize:8].any() and int(s[8:16].view(np.int64)[0]) == wi, (what, s, wi)
                if not HOSTMEM:
                    assert launches == 1, what


# ---- refusals ------------------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing(dab, rt1):
    """An index input with a map other than the identity, red == 0, x off its element alignment, nd outside 0 .. 8 and a chunk dim that
    does not fit its global extent are refused; inner * outer == 0 succeeds; none of them launches or writes an output."""
    L, lib = _lib().lib(), _lib()
    x = np.arange(64, dtype=np.float32)
    ii = np.arange(1, 65, dtype=np.int64)
    xb, ib = Buf(dab, rt1, x, 0, seed=7), Buf(dab, rt1, ii, 0, seed=8)
    ov, oi = Buf(dab, rt1, None, 0, np.float32, 8, seed=9), Buf(dab, rt1, None, 0, np.int64, 8, seed=10)
    slot = Buf(dab, rt1, None, 0, np.uint8, 16, seed=11)
    X, I, V, O = C.c_void_p(xb.ptr), C.c_void_p(ib.ptr), C.c_void_p(ov.ptr), C.c_void_p(oi.ptr)
    f32 = lib.F32
    no = (0, None, None, None)

    def dim(mapc=0, xp=X, ip=None, inner=8, red=8, outer=1, gl=no):
        return lambda: L.dab_findminmax_dim(rt1.ctx, f32, fo.FINDMAX, mapc, xp, ip, inner, red, outer, *gl, V, O)

    g = lambda cd, off, gd: (len(cd), _i64s(cd), _i64s(off), _i64s(gd))
    cases = [
        (lib.ERR_ARG, dim(mapc=MAP_ABS, ip=I)),                                    # an index input with abs
        (lib.ERR_ARG, dim(mapc=MAP_ABS2, ip=I)),
        (lib.OK, dim(inner=0)),                                                    # no output: nothing to do
        (lib.OK, dim(outer=0, red=0)),
        (lib.ERR_EMPTY, dim(red=0)),
        (lib.ERR_ARG, dim(xp=C.c_void_p(xb.ptr + 2))),                             # x off its 4-byte alignment
        (lib.ERR_ARG, dim(gl=(9,) + g([1] * 9, [0] * 9, [1] * 9)[1:])),          # nd > 8
        (lib.ERR_ARG, dim(gl=(-1, None, None, None))),
        (lib.ERR_ARG, dim(gl=(2, None, None, None))),                              # nd > 0 without its arrays
        (lib.ERR_ARG, dim(gl=g([8, 8], [0, 3], [8, 10]))),                         # 3 + 8 > 10
        (lib.ERR_ARG, dim(gl=g([8, 0], [0, 0], [8, 8]))),                          # a zero chunk dim
        (lib.ERR_ARG, dim(gl=g([8, 8], [-1, 0], [9, 8]))),                         # a negative offset
        (lib.ERR_EMPTY, lambda: L.dab_findminmax(rt1.ctx, f32, 0, 0, None, X, 0, C.c_void_p(slot.ptr))),
        (lib.ERR_ARG, lambda: L.dab_findminmax(rt1.ctx, f32, 0, 0, None, C.c_void_p(xb.ptr + 1), 8, C.c_void_p(slot.ptr))),
        (lib.ERR_ARG, lambda: L.dab_findminmax(rt1.ctx, lib.F64, 1, 0, None, C.c_void_p(xb.ptr + 4), 8, C.c_void_p(slot.ptr))),
    ]
    for k, (status, f) in enumerate(cases):
        l0 = rt1.launches()
        assert f() == status, k
        rt1.sync()
        assert rt1.launches() == l0, k
        assert ov.unchanged() and oi.unchanged() and slot.unchanged(), k
    assert xb.unchanged() and ib.unchanged()
    for b in (xb, ib, ov, oi, slot):
        b.free()


# ---- positions past 2^31 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inner,red,outer,label", [(1, (1 << 30) + 3, 2, "lead32_split"), (2, (1 << 30) + 3, 1, "strided_split")])
def test_positions_past_2_31_in_a_bool_chunk(dab, rt1, inner, red, outer, label):
    """A Bool chunk of 2^31 + 6 bytes, shape (2^30 + 3, 2) reduced over dims=1 (lead kernel, split) and (2, 2^30 + 3) over dims=2
    (strided kernel, split): winners and their twins at positions past 2^31, global indices through two chunk dims."""
    if HOSTMEM:
        pytest.skip("a 2 GiB chunk is a device-memory case")
    if rt1.device_info()["free_bytes"] < 6 * 2 ** 30:
        pytest.skip("needs 6 GiB of free device memory")
    sm = _sm(rt1)
    plan = fo.fmdim_plan(np.bool_, inner, red, outer, 0, False, sm)
    assert label in fo.plan_labels(plan, np.bool_, inner, outer, 0, False)
    lib = _lib()
    n = inner * red * outer
    x = dab.B200Array.empty(rt1, (n,), np.bool_)
    ov, oi = Buf(dab, rt1, None, 0, np.bool_, 2, seed=12), Buf(dab, rt1, None, 0, np.int64, 2, seed=13)
    pos = lambda i, r, o: i + inner * (r + red * o)
    # fibre A: one deciding element at the end of its run; fibre B: two past 2^31 in the last split (lead: in two lanes, strided: in one
    # thread's walk), where the earlier must win
    A, B = ((0, 0), (0, 1)) if inner == 1 else ((0, 0), (1, 0))
    r_a = red - 2
    lo_last = plan["bounds"][-1][0]
    r_b = (red - 5, red - 1) if inner == 1 else (red - 3, red - 1)
    assert pos(B[0], r_b[0], B[1]) > 1 << 31 and r_b[0] >= lo_last
    chunk = 1 << 26
    for fill, which in ((0, fo.FINDMAX), (1, fo.FINDMIN)):
        v = np.full(1, fill, dtype=np.uint8)
        lib.call("dab_fill", rt1.ctx, lib.U8, C.c_void_p(x.ptr), n, C.c_void_p(v.ctypes.data))
        mark = np.full(1, 1 - fill, dtype=np.uint8)
        for p in (pos(A[0], r_a, A[1]), pos(B[0], r_b[0], B[1]), pos(B[0], r_b[1], B[1])):
            lib.call("dab_h2d", rt1.ctx, C.c_void_p(x.ptr + p), C.c_void_p(mark.ctypes.data), 1)
        rt1.sync()
        cd, off, gd = [inner * red, outer] if inner == 1 else [inner, red], [0, 0], [inner * red, outer] if inner == 1 else [inner, red]
        l0 = rt1.launches()
        st = lib.lib().dab_findminmax_dim(rt1.ctx, lib.U8, which, 0, C.c_void_p(x.ptr), None, inner, red, outer, 2, _i64s(cd), _i64s(off),
                                          _i64s(gd), C.c_void_p(ov.ptr), C.c_void_p(oi.ptr))
        lib.check(st, rt1.ctx)
        assert rt1.launches() - l0 == plan["launches"]
        gv, gi = ov.read().reshape((inner, outer), order="F"), oi.read().reshape((inner, outer), order="F")
        want_i = np.zeros((inner, outer), dtype=np.int64)
        want_i[A] = pos(A[0], r_a, A[1]) + 1
        want_i[B] = pos(B[0], r_b[0], B[1]) + 1
        assert np.array_equal(gv, np.full((inner, outer), bool(1 - fill))), gv
        assert np.array_equal(gi, want_i), (gi, want_i)
    x.free()
    ov.free()
    oi.free()


# ---- public API ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.int64, np.bool_], ids=IDS)
@pytest.mark.parametrize("shape,dims", [((1 << 17, 3), 1), ((3, 1 << 17), 2)])
def test_public_dims_split_shapes_int64_and_bool(dab, rt1, dt, shape, dims):
    """findmax / findmin with dims of a one-worker Int64 and Bool DArray at two shapes that split the reduced extent."""
    rng = np.random.default_rng(70)
    n = int(np.prod(shape))
    A = (rng.random(n) < 0.001) if np.dtype(dt) == np.bool_ else rng.integers(-1000, 1000, n)
    A = A.astype(dt).reshape(shape, order="F")
    if np.dtype(dt) != np.bool_:
        A[(shape[0] - 1, 1)] = np.iinfo(np.int64).max
        A[(0, shape[1] - 1)] = np.iinfo(np.int64).min
    inner, red, outer = (1, shape[0], shape[1]) if dims == 1 else (shape[0], shape[1], 1)
    assert fo.fmdim_plan(dt, inner, red, outer, 0, False, _sm(rt1))["nsplit"] > 1
    d = dab.distribute(A)
    for which, fn in ((fo.FINDMAX, dab.findmax), (fo.FINDMIN, dab.findmin)):
        V, I = fn(d, dims=dims)
        wv, wi = fo.find_dims(which, A, dims)
        assert fo.same_bits(dab.to_array(V), wv) and np.array_equal(dab.to_array(I), wi), (which, shape, dims)
        V.close()
        I.close()
    d.close()
