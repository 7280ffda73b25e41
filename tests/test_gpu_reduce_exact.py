"""The reduction kernels against exact results, on every dispatch path.

``reduce_kernel`` (``dab_reduce``) and the ``rdim_*`` kernels (``dab_reducedim``) are called through ctypes and through the public
API with inputs whose results are exact, so every comparison is bit for bit (NaN payloads excepted, as in ``same_bits``):

  * integers: any values -- the map runs in the element type (``abs``/``abs2``/``-`` wrap at 32 bits for Int32, as in Julia), then
    Int32 widens to Int64 and ``+``/``*`` run mod 2^64, which is associative, so every grouping gives the same bits;
  * float sums: multiples of 2^-10 with |x| <= 8*2^-10 -- every tile of <= 32 values is exact in Float32 and the fp64 carrier is
    exact, so the result is the exact sum rounded once; with ``accumulate`` the result is op(out, S) rounded once;
  * float products: +-1 with +-2 / +-0.5 at the edge positions (the exponent stays in {-1, 0, 1}), exact in any order;
  * max / min / extrema: Julia's rules -- any NaN gives NaN, otherwise the extreme value, and a zero result is +0.0 for max when
    a +0.0 is present and -0.0 for min when a -0.0 is present.

Float16 elements are widened to Float32 by the map (abs2 rounds x*x to Float16 first), so the same inputs are exact for them, and the
references round the exact fp64 result once to Float16; their edge values add +-65504 and subnormals.  Fibres whose sum lies just past
a rounding midpoint (``ROUND_ONCE``) tell one rounding from a rounding through Float32 on every path.

Edge values (NaN with payloads and both signs, +-0, +-Inf, typemin / typemax, Int32 values near +-2^30 and +-2^31) sit where the
kernels split their work: first and last element of a run, the head peel of an unaligned run, the last partial 16-byte vector, the
scalar tail and both sides of every split boundary.  ``launch_rdim`` is modelled below so that the shape table can be shown to reach
every kernel and branch, and the launch counter is checked against the model.
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
F32, F64, I32, I64, U8 = range(5)
F16 = 8
SUM, PROD, MAX, MIN, ALL, ANY, COUNT, EXTREMA = range(8)
MAP_ID, MAP_ABS, MAP_ABS2, MAP_NEG = range(4)
NP = {F32: np.float32, F64: np.float64, I32: np.int32, I64: np.int64, U8: np.uint8, F16: np.float16}
OPS = (SUM, PROD, MAX, MIN)
MAPS = (MAP_ID, MAP_ABS, MAP_ABS2, MAP_NEG)
RD_THREADS, RD_UNROLL = 256, 4
DTS, DT_IDS = [F32, F64, I32, I64, F16], ["f32", "f64", "i32", "i64", "f16"]

if HOSTMEM:                                                     # the Float16 code of the host-memory emulation
    import f16_hostmem
    f16_hostmem.install()


def _lib():
    from darray_b200 import _lib as L
    return L


def same_bits(got, want):
    """Bit-identical, except that NaN payloads are not compared (the GPU returns the canonical quiet NaN)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    if not np.array_equal(np.isnan(got), nan):
        return False
    u = {2: np.uint16, 4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    return np.array_equal(got.view(u)[~nan], want.view(u)[~nan])


# ---------------------------------------------------------------------------------------------------------- references
def ref_map(v, mapc):
    """The map in the element type (integers wrap like Julia's)."""
    with np.errstate(all="ignore"):
        return {MAP_ID: lambda: v, MAP_ABS: lambda: np.abs(v), MAP_ABS2: lambda: v * v, MAP_NEG: lambda: -v}[mapc]()


def result_dtype(dt, op):
    return np.dtype(np.int64) if op in (SUM, PROD) and np.dtype(dt).kind == "i" else np.dtype(dt)


def jl_extreme(m, axis, is_max):
    """Julia's maximum / minimum along ``axis``: NaN wins, then the extreme value, +0.0 > -0.0."""
    m = np.asarray(m)
    if m.dtype.kind != "f":
        return (np.max if is_max else np.min)(m, axis=axis)
    nan = np.isnan(m)
    r = (np.max if is_max else np.min)(np.where(nan, -np.inf if is_max else np.inf, m), axis=axis)
    want_neg = not is_max                                   # the zero that wins: +0.0 for max, -0.0 for min
    has = ((m == 0) & (np.signbit(m) == want_neg)).any(axis=axis)
    z = m.dtype.type(-0.0 if want_neg else 0.0)
    other = m.dtype.type(0.0 if want_neg else -0.0)
    r = np.where(r == 0, np.where(has, z, other), r)
    return np.where(nan.any(axis=axis), m.dtype.type(np.nan), r).astype(m.dtype)


def ref_reduce(m, op, axis, wide=False):
    """m: mapped values in the element type.  wide: a float sum / product as its exact fp64 value S, not rounded to the element type."""
    m = np.asarray(m)
    with np.errstate(all="ignore"):
        if op in (SUM, PROD):
            if m.dtype.kind == "f":
                w = m.astype(np.float64)               # exact: see the module docstring
                w = w.sum(axis=axis) if op == SUM else w.prod(axis=axis)
                return w if wide else w.astype(m.dtype)
            w = m.astype(np.int64)                     # NumPy's Int64 sum / prod wrap mod 2^64
            return w.sum(axis=axis, dtype=np.int64) if op == SUM else w.prod(axis=axis, dtype=np.int64)
        return jl_extreme(m, axis, op == MAX)


def ref_combine(o, r, op):
    """op(o, r) elementwise in the result type (the accumulate=1 prefill).  A float sum / product r is given as its exact fp64 value S
    (``ref_reduce(..., wide=True)``): o + S and o * S are exact in fp64 here and round once to the result type."""
    o, r = np.asarray(o), np.asarray(r)
    if op in (MAX, MIN):
        return jl_extreme(np.stack([o, r]), 0, op == MAX)
    with np.errstate(all="ignore"):
        if o.dtype.kind == "f":
            w = (o.astype(np.float64) + r.astype(np.float64)) if op == SUM else (o.astype(np.float64) * r.astype(np.float64))
            return w.astype(o.dtype)
        return (o + r) if op == SUM else (o * r)


# ---------------------------------------------------------------------------------------------------------- the dispatch model
def model_rdim(dt, inner, red, outer, base_mod16, sm_count):
    """``dab_reducedim`` -> ``launch_rdim`` (dab_reducedim.cu): which kernel, G, vector path, short 4-run path, nsplit, launches."""
    es = np.dtype(NP[dt]).itemsize
    vpt = 16 // es
    S = 8 * sm_count
    if inner * outer == 0:
        return dict(kernel="none", launches=0)
    if red == 0:
        return dict(kernel="fill", launches=None)
    if inner == 1 and outer == 1 and red >= 1 << 16:
        return dict(kernel="disguise", nsplit=1, launches=2)
    if inner == 1:
        if red < 4096 and outer >= S:
            units = red // vpt
            G = 32 if units >= 32 else 16 if units >= 16 else 8 if units >= 8 else 4 if units >= 4 else 2
            vec = red % vpt == 0 and base_mod16 == 0
            return dict(kernel="lead_group", G=G, vec=vec, short=vec and red // vpt <= G, nsplit=1, launches=1)
        max_split = max(1, red * es // 16384)
        want = 1 if outer >= S else -(-S // outer)
        nsplit = min(want, max_split, 1024)
        return dict(kernel="lead_cta", nsplit=nsplit, launches=1 + (nsplit > 1), rem=red % vpt != 0, unaligned=base_mod16 != 0)
    vec = inner % vpt == 0 and base_mod16 == 0 and inner * outer // vpt >= 4096
    base_ctas = -(-(inner * outer // vpt) // RD_THREADS) if vec else -(-(inner * outer) // RD_THREADS)
    max_split = max(1, red // 256)
    want = 1 if base_ctas >= 4 * S else -(-4 * S // base_ctas)
    nsplit = min(want, max_split, 1024)
    return dict(kernel="strided_vec" if vec else "strided", nsplit=nsplit, launches=1 + (nsplit > 1))


def branches(m):
    """The branch labels one model result reaches (both accumulate modes are run for every shape)."""
    k = m["kernel"]
    out = set()
    if k == "lead_group":
        out |= {f"group G={m['G']}", "group vec" if m["vec"] else "group scalar"} | ({"group short"} if m["short"] else set())
    elif k == "lead_cta":
        split = "nsplit=1" if m["nsplit"] == 1 else "nsplit>1"
        out |= {f"cta {split}"} | ({"cta red%VPT"} if m["rem"] else set()) | ({f"cta unaligned {split}"} if m["unaligned"] else set())
    elif k in ("strided", "strided_vec"):
        out.add(f"{k} nsplit=1" if m["nsplit"] == 1 else f"{k} nsplit>1")
    elif k == "disguise":
        out |= {"disguise acc=0", "disguise acc=1"}
    if m.get("nsplit", 1) > 1:
        out |= {"finish acc=0", "finish acc=1"}
    return out


REQUIRED = ({f"group G={g}" for g in (2, 4, 8, 16, 32)} | {"group vec", "group scalar", "group short", "cta nsplit=1", "cta nsplit>1",
            "cta red%VPT", "cta unaligned nsplit=1", "cta unaligned nsplit>1", "strided nsplit=1", "strided nsplit>1", "strided_vec nsplit=1", "strided_vec nsplit>1",
            "finish acc=0", "finish acc=1", "disguise acc=0", "disguise acc=1"})


def shape_table(dt, sm_count):
    """name -> (inner, reduce, outer, base offset in elements), sized from the element width and the SM count (S = 8 * sm_count)."""
    vpt = 16 // np.dtype(NP[dt]).itemsize
    S = 8 * sm_count
    split_red = 3 * (32768 // (16 // vpt)) + 5               # 3 splits' worth of 16 KiB plus a tail: >= 2 splits for any width
    return {
        "group_g2_short": (1, 2 * vpt, S, 0),
        "group_g4_scalar": (1, 4 * vpt + 1, S, 0),
        "group_g8_vec": (1, 12 * vpt, S + 3, 0),
        "group_g16_short": (1, 16 * vpt, S, 0),
        "group_g32_vec": (1, 4096 - vpt, S + 1, 0),
        "group_g32_unaligned": (1, 64 * vpt, S, 1),
        "group_g2_tiny": (1, 3, S + 5, 0),
        "cta_one_split": (1, 4096 + vpt + 1, S, 0),
        "cta_split": (1, split_red, 3, 0),
        "cta_split_unaligned": (1, split_red + 2, 2, vpt - 1),
        "cta_one_split_unaligned": (1, 3001, 3, 1),             # < 16 KiB per run for either width: no split
        "strided_one_split": (3, 3, 4 * S * RD_THREADS // 3 + 7, 0),
        "strided_split": (5, 3000, 7, 0),
        "strided_vec_one_split": (4 * vpt, 2, 4 * S * RD_THREADS // 4 + 1, 0),
        "strided_vec_split": (16 * vpt, 1000, 256, 0),
        "strided_unaligned_split": (16 * vpt, 700, 256, 1),
        "disguise": (1, (1 << 16) + 3, 1, 0),
        "disguise_unaligned": (1, (1 << 18) + 1, 1, 1),
    }


def test_shape_table_reaches_every_branch(dab, rt1):
    """The table below reaches every branch of launch_rdim, for a 2-, a 4- and an 8-byte element type, on this device."""
    sm = rt1.device_info()["sm_count"]
    for dt in DTS:
        got = set()
        for name, (inner, red, outer, off) in shape_table(dt, sm).items():
            es = np.dtype(NP[dt]).itemsize
            got |= branches(model_rdim(dt, inner, red, outer, (off * es) % 16, sm))
        assert REQUIRED <= got, (dt, sorted(REQUIRED - got))


# ---------------------------------------------------------------------------------------------------------- input builders
def edge_positions(red, head, vpt, nsplit, unroll_rows=8):
    """Positions along a run of length ``red`` where a kernel changes what it does."""
    split_len = -(-red // max(nsplit, 1))
    pos = {0, 1, red - 2, red - 1, head - 1, head, vpt - 1, vpt}
    nvec = (red - head) // vpt if red >= head else 0
    pos |= {head + nvec * vpt - 1, head + nvec * vpt, head + (nvec - 1) * vpt}       # last whole vector and the scalar tail
    pos |= {red - red % unroll_rows - 1, red - red % unroll_rows}                    # the strided kernels' 8-row remainder
    for s in range(1, max(nsplit, 1)):
        b = s * split_len
        pos |= {b - 1, b, b + 1}
        h = (vpt - (head + b) % vpt) % vpt if vpt > 1 else 0                         # head peel of the split that starts at b
        pos |= {b + h - 1, b + h}
    return sorted(p for p in pos if 0 <= p < red)


KINDS = 8            # float fibre kinds: 0 NaN, 1 +-Inf, 2 all <= 0 with a +0.0, 3 all >= 0 with a -0.0, 4 finite extremes, 5-7 plain
FINITE_KINDS = (2, 3, 4, 5, 6, 7)


def build(dt, op, inner, red, outer, edges, seed, kind_shift=0, kinds=None):
    """x[i, r, o] (column-major) with exact results for ``op``; every fibre gets special values at ``edges`` along r.

    Float fibre f is of kind ``kinds[(f + kind_shift) % len(kinds)]`` (default: all KINDS), so a one-fibre input takes its kind
    from ``kind_shift``; where in ``edges`` its special values land depends on the seed."""
    rng = np.random.default_rng(seed)
    kinds = np.asarray(range(KINDS) if kinds is None else kinds)
    T = NP[dt]
    shape = (inner, red, outer)
    E = np.asarray(edges, dtype=np.int64)
    fid = (np.arange(inner)[:, None] + inner * np.arange(outer)[None, :]).reshape(-1, order="F")   # fibre number, (i, o) F-order
    if np.dtype(T).kind == "f":
        if op == PROD:
            x = np.where(rng.random(shape) < 0.5, T(-1), T(1)).astype(T)
        elif op in (MAX, MIN):                                  # no zeros: a zero result comes from the kinds' placed +-0 only
            x = (rng.integers(1, 9, shape) * np.where(rng.random(shape) < 0.5, -1, 1) * 2.0 ** -10).astype(T)
        else:
            x = (rng.integers(-8, 9, shape) * 2.0 ** -10).astype(T)
        kind = kinds[(fid + kind_shift) % len(kinds)]
        xf = x
        ii, oo = fid % inner, fid // inner
        if len(E):
            r0 = int(rng.integers(len(E)))
            e1 = E[(fid + r0) % len(E)]
            e2 = E[(fid * 7 + 3 + r0) % len(E)]
            if op == PROD:                                      # +-2 and +-0.5 alternate along the edges: exponent stays in {-1, 0, 1}
                for k, p in enumerate(E):
                    xf[:, p, :] = (T(2.0) if k % 2 == 0 else T(0.5)) * np.where(rng.random((inner, outer)) < 0.5, T(-1), T(1))
            sel = kind == 2
            xf[ii[sel], :, oo[sel]] = -np.abs(xf[ii[sel], :, oo[sel]])
            sel = kind == 3
            xf[ii[sel], :, oo[sel]] = np.abs(xf[ii[sel], :, oo[sel]])
            U = {np.float16: np.uint16, np.float32: np.uint32, np.float64: np.uint64}[T]
            bits, nmant = 8 * np.dtype(T).itemsize, np.finfo(T).nmant
            sign, quiet, frac = 1 << (bits - 1), 1 << (nmant - 1), (1 << nmant) - 1
            expo = ((1 << (bits - 1)) - 1) ^ frac
            f = np.flatnonzero(kind == 0)                       # NaN: quiet and signalling payloads, both signs
            g = f // 6
            payload = (rng.integers(1, min(1 << 20, quiet), f.size).astype(np.uint64) | np.where(g % 4 < 2, quiet, 0).astype(np.uint64)) & np.uint64(frac)
            nanv = (np.uint64(expo) | payload | np.where(g % 2 == 1, np.uint64(sign), np.uint64(0))).astype(U).view(T)
            xf[ii[f], e1[f], oo[f]] = nanv
            f = np.flatnonzero(kind == 1)
            xf[ii[f], e1[f], oo[f]] = T(np.inf)
            xf[ii[f], e2[f], oo[f]] = np.where(f % 2 == 1, T(-np.inf), T(np.inf))
            f = np.flatnonzero(kind == 2)
            xf[ii[f], e1[f], oo[f]] = T(0.0)
            xf[ii[f], e2[f], oo[f]] = T(-0.0)
            f = np.flatnonzero(kind == 3)
            xf[ii[f], e1[f], oo[f]] = T(-0.0)
            if op != PROD and T != np.float16:
                f = np.flatnonzero(kind == 4)
                xf[ii[f], e1[f], oo[f]] = T(16 * 2.0 ** -10)
                xf[ii[f], e2[f], oo[f]] = T(-16 * 2.0 ** -10)
            elif op != PROD:
                # Float16 extremes.  max / min: +-65504 and the smallest and largest subnormals decide (abs2 takes 65504 to Inf).  Sums:
                # 65504 twice with one sign overflows to +-Inf (once, the result stays 65504: the rest is far below its 16-unit rounding
                # margin); subnormals 2^-24 and -3 * 2^-24 pull an exact sum 2^-23 below its grid point, which for half the sums is just
                # below a Float16 rounding midpoint: one rounding goes down, a rounding through Float32 lands on the midpoint first
                s = np.where(np.arange(len(kind)) % 2 == 0, 1.0, -1.0)              # one sign per fibre
                f = np.flatnonzero(kind == 4)
                xf[ii[f], e1[f], oo[f]] = (s[f] * 65504.0).astype(T)
                xf[ii[f], e2[f], oo[f]] = (s[f] * (65504.0 if op == SUM else -2.0 ** -24)).astype(T)
                f = np.flatnonzero(kind == 5)
                xf[ii[f], e1[f], oo[f]] = T(2.0 ** -24)
                xf[ii[f], e2[f], oo[f]] = T(-3 * 2.0 ** -24 if op == SUM else -1023 * 2.0 ** -24)
        return np.asfortranarray(xf)
    info = np.iinfo(T)
    if op == PROD:                                              # odd factors never reach 0 mod 2^64
        x = np.where(rng.random(shape) < 0.5, T(-1), T(1)).astype(T)
        big = np.asarray([info.max, info.min + 1, 46341, -65535, 65537, 3] if T == np.int32 else
                         [info.max, info.min + 1, (1 << 33) + 1, -(1 << 31) - 1, 65537, 3], dtype=T)
    else:
        if T == np.int32:
            mag = rng.integers(1 << 30, 1 << 31, shape, dtype=np.int64)
            x = np.where(rng.random(shape) < 0.5, -mag, mag - 1).astype(T)
        else:
            x = rng.integers(info.min // 2, info.max // 2, shape, dtype=np.int64).astype(T) * T(2) + T(1)
        big = np.asarray([info.max, info.min, info.max - 1, info.min + 1, 1 << 30, -(1 << 30)], dtype=T)
    xf = x
    for k, p in enumerate(E):
        xf[:, p, :] = big[(k + np.arange(inner)[:, None] + np.arange(outer)[None, :]) % len(big)]
    if op == PROD and len(E) >= 2:                              # fibre 0 only: a whole-array product stays nonzero mod 2^64
        xf[0, E[0], 0] = T(65536)
        xf[0, E[-1], 0] = T(65536)
    return np.asfortranarray(xf)


def prefill(rdt, op, n, seed):
    """accumulate=1 prefills: exact values plus NaN, -0.0 and typemax."""
    rng = np.random.default_rng(seed)
    rdt = np.dtype(rdt)
    if rdt.kind == "f":
        if op == PROD:
            o = np.where(rng.random(n) < 0.5, -1.0, 1.0) * np.where(rng.random(n) < 0.5, 2.0, 0.5)
        else:
            o = rng.integers(-64, 65, n) * 2.0 ** -10
        o = o.astype(rdt)
        specials = [np.nan, -0.0, np.inf, -np.inf, 0.0]
    else:
        o = rng.integers(-(1 << 40), 1 << 40, n).astype(rdt) * 2 + 1
        specials = [np.iinfo(rdt).max, np.iinfo(rdt).min, -1, 0, 1]
    for k, v in enumerate(specials):
        o[k::7] = v
    return o


# ---------------------------------------------------------------------------------------------------------- device helpers
class Dev:
    """One device buffer with a chosen element offset from a 256-byte aligned allocation."""

    def __init__(self, rt, host, off):
        host = np.ascontiguousarray(np.asarray(host).reshape(-1, order="F"))
        self.rt, self.dt, self.n = rt, host.dtype, host.size
        self.base = rt.alloc((self.n + 16) * host.itemsize)
        self.ptr = self.base + off * host.itemsize
        if self.n:
            _lib().call("dab_h2d", rt.ctx, C.c_void_p(self.ptr), C.c_void_p(host.ctypes.data), self.n * host.itemsize)
        rt.sync()

    def get(self, n=None, dt=None):
        dt = np.dtype(dt or self.dt)
        n = self.n if n is None else n
        out = np.empty(n, dtype=dt)
        if n:
            _lib().call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.ptr), n * dt.itemsize)
        self.rt.sync()
        return out

    def put(self, host):
        host = np.ascontiguousarray(host)
        _lib().call("dab_h2d", self.rt.ctx, C.c_void_p(self.ptr), C.c_void_p(host.ctypes.data), host.nbytes)
        self.rt.sync()

    def free(self):
        self.rt.free(self.base)


def first_bad(got, want):
    """The first three positions where got and want differ (NaN equals NaN)."""
    same = got == want
    if got.dtype.kind == "f":
        same |= np.isnan(got) & np.isnan(want)
    return np.flatnonzero(~same)[:3]


def rdim_call(rt, dt, op, mapc, x, inner, red, outer, out, acc):
    n0 = rt.launches()
    _lib().call("dab_reducedim", rt.ctx, dt, op, mapc, C.c_void_p(x.ptr if x is not None else 0), inner, red, outer, C.c_void_p(out.ptr), acc)
    rt.sync()
    return rt.launches() - n0


def _maps_for(dt, op, k):
    """Int32 (widened sums and products; -x under max / min) and Float16 (maps in Float32, abs2 rounded to Float16) take every map on
    every shape; the other types take two maps per shape, in turn."""
    if dt in (I32, F16):
        return MAPS
    return (MAPS[k % 4], MAPS[(k + 1) % 4])


# ---------------------------------------------------------------------------------------------------------- (a) dab_reducedim
@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("name", list(shape_table(F32, 132)))
def test_reducedim_exact(dab, rt1, name, dt):
    sm = rt1.device_info()["sm_count"]
    inner, red, outer, off = shape_table(dt, sm)[name]
    T = NP[dt]
    es = np.dtype(T).itemsize
    vpt = 16 // es
    k = list(shape_table(dt, sm)).index(name)
    m = model_rdim(dt, inner, red, outer, (off * es) % 16, sm)
    head = (vpt - off % vpt) % vpt if inner == 1 else 0           # head peel of the first run when runs are contiguous
    edges = edge_positions(red, head, vpt, m.get("nsplit", 1))
    # with fewer fibres than kinds, every fibre takes every kind in turn, so finite and zero results are checked on every path
    shifts = range(KINDS) if np.dtype(T).kind == "f" and inner * outer < KINDS else (0,)
    bad = []
    finite_nonzero = set()
    for op, shift in [(op, shift) for op in OPS for shift in shifts]:
        x = build(dt, op, inner, red, outer, edges, seed=1000 * k + 10 * op + dt + 100000 * shift, kind_shift=shift)
        xd = Dev(rt1, x, off)
        rdt = result_dtype(T, op)
        try:
            for mapc in _maps_for(dt, op, k + op + shift):
                mx = ref_map(x, mapc)
                want = ref_reduce(mx, op, axis=1).reshape(-1, order="F").astype(rdt)
                wide = ref_reduce(mx, op, axis=1, wide=True).reshape(-1, order="F")
                if (np.isfinite(want) & (want != 0)).any():
                    finite_nonzero.add(op)
                out = Dev(rt1, np.zeros(inner * outer, dtype=rdt), 0)
                try:
                    nl = rdim_call(rt1, dt, op, mapc, xd, inner, red, outer, out, 0)
                    got = out.get()
                    if not same_bits(got, want):
                        idx = first_bad(got, want)
                        bad.append(f"op={op} map={mapc} acc=0 first bad outputs {idx.tolist()}: got {got[idx].tolist()} want {want[idx].tolist()}")
                    if not HOSTMEM:
                        assert nl == m["launches"], (op, mapc, nl, m)
                    pre = prefill(rdt, op, inner * outer, seed=k + 7 * op)
                    out.put(pre)
                    rdim_call(rt1, dt, op, mapc, xd, inner, red, outer, out, 1)
                    got = out.get()
                    want1 = ref_combine(pre, wide, op)
                    if not same_bits(got, want1):
                        idx = first_bad(got, want1)
                        bad.append(f"op={op} map={mapc} acc=1 first bad outputs {idx.tolist()}: got {got[idx].tolist()} want {want1[idx].tolist()}")
                finally:
                    out.free()
        finally:
            xd.free()
    assert not bad, f"{name} {np.dtype(T).name} {m}: " + "; ".join(bad)
    assert finite_nonzero == set(OPS), f"{name}: no finite nonzero result checked for ops {set(OPS) - finite_nonzero}"


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_reducedim_empty_extents(dab, rt1, dt):
    """reduce == 0: SUM / PROD write the identity, MAX / MIN throw, accumulate leaves R as it is; inner*outer == 0 touches nothing."""
    L = _lib()
    T = NP[dt]
    x = Dev(rt1, np.zeros(4, dtype=T), 0)
    for op in OPS:
        rdt = result_dtype(T, op)
        out = Dev(rt1, prefill(rdt, op, 6, seed=op), 0)
        before = out.get()
        try:
            rdim_call(rt1, dt, op, MAP_ID, x, 3, 0, 2, out, 1)
            assert same_bits(out.get(), before)
            rdim_call(rt1, dt, op, MAP_ID, x, 0, 5, 2, out, 0)
            rdim_call(rt1, dt, op, MAP_ID, x, 3, 5, 0, out, 0)
            assert same_bits(out.get(), before)
            if op in (SUM, PROD):
                rdim_call(rt1, dt, op, MAP_ABS2, x, 3, 0, 2, out, 0)
                assert same_bits(out.get(), np.full(6, 0 if op == SUM else 1, dtype=rdt))
            else:
                with pytest.raises(L.DabError) as err:
                    rdim_call(rt1, dt, op, MAP_ID, x, 3, 0, 2, out, 0)
                assert err.value.status == L.ERR_EMPTY
        finally:
            out.free()
    x.free()


# ---------------------------------------------------------------------------------------------------------- (b) dab_reduce
def reduce_sizes(dt):
    vpt = 16 // np.dtype(NP[dt]).itemsize
    tile = RD_THREADS * RD_UNROLL * vpt                                  # one tile step of a CTA; a CTA streams two
    return list(range(1, vpt + 2)) + [tile - 1, tile, tile + 1, 2 * tile - 1, 2 * tile + 1, 4095, 4096, 4097, 8191, 8193, (1 << 22) + 3]


def slot_value(slot, rdt):
    return slot.view(np.uint8)[:rdt.itemsize].view(rdt)[0]


def reduce_call(rt, dt, op, mapc, x, n, slot):
    _lib().call("dab_reduce", rt.ctx, dt, op, mapc, None, C.c_void_p(x.ptr), n, C.c_void_p(slot.ptr))
    return slot.get(16, np.uint8)


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_reduce_exact(dab, rt1, dt):
    T = NP[dt]
    vpt = 16 // np.dtype(T).itemsize
    slot = Dev(rt1, np.zeros(16, dtype=np.uint8), 0)
    bad = []
    finite_nonzero = set()
    ops = OPS if dt == F16 else OPS + (EXTREMA,)          # Float16 extrema is a MIN and a MAX reduction: EXTREMA is refused
    if dt == F16:
        xd = Dev(rt1, np.ones(8, dtype=T), 0)
        with pytest.raises(_lib().DabError) as err:
            reduce_call(rt1, dt, EXTREMA, MAP_ID, xd, 8, slot)
        assert err.value.status == _lib().ERR_UNSUPPORTED
        xd.free()
    try:
        for si, n in enumerate(reduce_sizes(dt)):
            offs = range(vpt) if n < 10000 else (0, 1 % vpt)
            for off in offs:
                head = min((vpt - off % vpt) % vpt, n)
                nvec = (n - head) // vpt
                tile = RD_THREADS * RD_UNROLL * vpt
                edges = edge_positions(n, head, vpt, 1) + [p for t in (1, 2, 3, nvec * vpt // tile)
                                                           for p in (head + t * tile - 1, head + t * tile) if 0 <= p < n]
                # floats: one input with NaN, +-Inf or a signed-zero rule (kinds 0-3), one with finite values (kinds 4-7), in turn
                rot = si + off
                for op, shift in [(op, shift) for op in ops
                                  for shift in (((rot + op) % 4, 4 + (rot + op) % 4) if np.dtype(T).kind == "f" else (0,))]:
                    data_op = PROD if op == PROD else SUM if op == EXTREMA else op
                    x = build(dt, data_op, 1, n, 1, sorted(set(edges)), seed=si * 31 + off * 7 + op + 1000 * shift, kind_shift=shift).reshape(-1)
                    xd = Dev(rt1, x, off)
                    try:
                        maps = (MAP_ID,) if op == EXTREMA else (MAPS if dt == I32 else (MAPS[(si + off + op) % 4],))
                        for mapc in maps:
                            s = reduce_call(rt1, dt, op, mapc, xd, n, slot)
                            if op == EXTREMA:
                                got = s[:2 * np.dtype(T).itemsize].view(T)
                                want = np.asarray([jl_extreme(x, 0, False), jl_extreme(x, 0, True)], dtype=T)
                            else:
                                rdt = result_dtype(T, op)
                                got = np.asarray([slot_value(s, rdt)])
                                want = np.asarray([ref_reduce(ref_map(x, mapc), op, axis=0)], dtype=rdt)
                            if (np.isfinite(want) & (want != 0)).any():
                                finite_nonzero.add((op, n))
                            if not same_bits(got, want):
                                bad.append(f"n={n} off={off} kind={shift} op={op} map={mapc}: got {got.tolist()} want {want.tolist()}")
                    finally:
                        xd.free()
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:12]) + f" ({len(bad)} cases)"
    missing = {(op, n) for op in ops for n in reduce_sizes(dt)} - finite_nonzero
    assert not missing, f"no finite nonzero result checked for (op, n) in {sorted(missing)}"


@pytest.mark.parametrize("n", [1, 17, 4097, 8193, (1 << 22) + 3])
def test_reduce_bool_exact(dab, rt1, n):
    """Bool sum / count / max / min, with the odd one out at every edge position in turn."""
    slot = Dev(rt1, np.zeros(16, dtype=np.uint8), 0)
    try:
        for off in range(4):
            head = min((16 - off) % 16, n)
            for p in edge_positions(n, head, 16, 1):
                rng = np.random.default_rng(p + n)
                for op, fill in ((SUM, None), (COUNT, None), (MAX, 0), (MIN, 1)):
                    x = (rng.random(n) < 0.5).astype(np.uint8) if fill is None else np.full(n, fill, dtype=np.uint8)
                    x[p] = 1 - fill if fill is not None else x[p]
                    xd = Dev(rt1, x, off)
                    try:
                        s = reduce_call(rt1, U8, op, MAP_ID, xd, n, slot)
                    finally:
                        xd.free()
                    if op in (SUM, COUNT):
                        assert slot_value(s, np.dtype(np.int64)) == int(np.count_nonzero(x)), (n, off, p, op)
                    else:
                        assert slot_value(s, np.dtype(np.uint8)) == (x.max() if op == MAX else x.min()), (n, off, p, op)
    finally:
        slot.free()


# ---------------------------------------------------------------------------------------------------------- (b2) one rounding
# Fibres whose exact sum S lies just past a rounding midpoint of the result type, built so that every Float32 tile of every kernel is
# exact (r = 0 and r = red - 1 never share a tile on these shapes) and only the fp64 carrier holds S:
#   Float16: 32768 at r = 0, 16 in the middle, 2^-10 at r = red - 1: S = 32784 + 2^-10 rounds once to 32800 and to 32768 through
#            Float32 (where 32784 is a tie, which goes to even);
#   Float32: 1 at r = 0, 2^-27 at r = red - 1: S = 1 + 2^-27 is 1 in Float32; onto a prefill of 2^24, one rounding gives 2^24 + 2 and
#            a rounding through Float32 S gives 2^24 (a tie again).
# Signs alternate by fibre.  The prefills are chosen so that rounding op(out, S) once and rounding op(out, round(S)) differ.
ROUND_ONCE = {F16: ((32768.0, 16.0, 2.0 ** -10), (-2.0 ** -10, 0.0, 2.0 ** -10, -2.0 ** -9)),
              F32: ((1.0, 0.0, 2.0 ** -27), (2.0 ** 24, 2.0 ** 24 + 4, 0.0))}


def round_once_input(dt, inner, red, outer):
    big, mid, tiny = ROUND_ONCE[dt][0]
    sgn = np.where(np.arange(inner * outer) % 2 == 0, 1.0, -1.0).reshape((inner, outer), order="F")
    x = np.zeros((inner, red, outer))
    x[:, 0, :], x[:, red // 2, :], x[:, red - 1, :] = big * sgn, mid * sgn, tiny * sgn
    return np.asfortranarray(x.astype(NP[dt]))


def round_once_prefill(dt, S):
    """Prefills relative to the sign of S (see ROUND_ONCE), in turn."""
    o = np.asarray(ROUND_ONCE[dt][1])
    return (o[np.arange(S.size) % len(o)] * np.where(S < 0, -1.0, 1.0)).astype(NP[dt])


@pytest.mark.parametrize("dt", [F32, F16], ids=["f32", "f16"])
@pytest.mark.parametrize("name", list(shape_table(F32, 132)))
def test_reducedim_rounds_once(dab, rt1, name, dt):
    """Float SUM with accumulate = 0 and 1 on every launch_rdim branch: the result is S rounded once, and op(out, S) rounded once."""
    sm = rt1.device_info()["sm_count"]
    inner, red0, outer, off = shape_table(dt, sm)[name]
    T = NP[dt]
    es = np.dtype(T).itemsize
    red = max(red0, 3)                                            # room for the three values; the branch stays the same
    m = model_rdim(dt, inner, red, outer, (off * es) % 16, sm)
    assert m == model_rdim(dt, inner, red0, outer, (off * es) % 16, sm), (name, m)
    x = round_once_input(dt, inner, red, outer)
    xd = Dev(rt1, x, off)
    bad = []
    try:
        for mapc in (MAP_ID, MAP_ABS, MAP_NEG):
            S = ref_reduce(ref_map(x, mapc), SUM, axis=1, wide=True).reshape(-1, order="F")
            want0 = S.astype(T)
            pre = round_once_prefill(dt, S)
            want1 = (pre.astype(np.float64) + S).astype(T)
            twice = (pre.astype(np.float64) + S.astype(T).astype(np.float64)).astype(T)
            if dt == F16:
                assert not (S.astype(np.float32).astype(T) == want0).any(), "the data does not tell one rounding from two"
            assert (twice != want1).sum() >= S.size // len(ROUND_ONCE[dt][1]), "the prefills do not tell one rounding from two"
            out = Dev(rt1, np.zeros(inner * outer, dtype=T), 0)
            try:
                nl = rdim_call(rt1, dt, SUM, mapc, xd, inner, red, outer, out, 0)
                got = out.get()
                if not HOSTMEM:
                    assert nl == m["launches"], (mapc, nl, m)
                if not same_bits(got, want0):
                    idx = first_bad(got, want0)
                    bad.append(f"map={mapc} acc=0 first bad outputs {idx.tolist()}: got {got[idx].tolist()} want {want0[idx].tolist()}")
                out.put(pre)
                rdim_call(rt1, dt, SUM, mapc, xd, inner, red, outer, out, 1)
                got = out.get()
                if not same_bits(got, want1):
                    idx = first_bad(got, want1)
                    bad.append(f"map={mapc} acc=1 first bad outputs {idx.tolist()}: got {got[idx].tolist()} want {want1[idx].tolist()} "
                               f"(prefill {pre[idx].tolist()}; op(out, round(S)) = {twice[idx].tolist()})")
            finally:
                out.free()
    finally:
        xd.free()
    assert not bad, f"{name} {np.dtype(T).name} {m}: " + "; ".join(bad)


def test_reduce_f16_rounds_once(dab, rt1):
    """dab_reduce of Float16 round-once fibres at every size and head offset of test_reduce_exact: the slot holds S rounded once to
    Float16 and the exact fp64 carrier S."""
    slot = Dev(rt1, np.zeros(16, dtype=np.uint8), 0)
    bad = []
    try:
        for n in reduce_sizes(F16):
            if n < 3:
                continue
            for off in (0, 1, 7) if n < 10000 else (0, 1):
                if n == 8 and off == 0:                       # one 16-byte vector: all eight values share one Float32 tile
                    continue
                x = round_once_input(F16, 1, n, 1).reshape(-1)
                xd = Dev(rt1, x, off)
                try:
                    for mapc in (MAP_ID, MAP_ABS, MAP_NEG):
                        S = float(ref_reduce(ref_map(x, mapc), SUM, axis=0, wide=True))
                        s = reduce_call(rt1, F16, SUM, mapc, xd, n, slot)
                        got, carrier = slot_value(s, np.dtype(np.float16)), s[8:16].view(np.float64)[0]
                        if got != np.float16(S) or carrier != S:
                            bad.append(f"n={n} off={off} map={mapc}: got {got!r} carrier {carrier!r}, want {np.float16(S)!r} carrier {S!r}")
                finally:
                    xd.free()
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:12]) + f" ({len(bad)} cases)"


PRED_MAPS = range(16, 24)                # EQ NE LT LE GT GE ISNAN NONZERO


@pytest.mark.parametrize("n", [1, 9, 8193, (1 << 20) + 5])
def test_reduce_f16_predicates(dab, rt1, n):
    """COUNT / ANY / ALL of Float16 data through every predicate map, with Float16 parameters (signed zeros, a subnormal, 65504, Inf,
    NaN): compared in Float32, which is exact for Float16 operands, so NumPy's Float16 comparisons are the reference."""
    rng = np.random.default_rng(n)
    x = rng.integers(0, 1 << 16, n).astype(np.uint16).view(np.float16)             # every kind of bit pattern, NaN payloads included
    specials = np.asarray([0.0, -0.0, 2.0 ** -24, 65504.0, -np.inf, np.nan, 1.5], dtype=np.float16)
    params = [np.float16(v) for v in (0.0, -0.0, 2.0 ** -24, 65504.0, np.inf, np.nan, 1.5)]
    slot = Dev(rt1, np.zeros(16, dtype=np.uint8), 0)
    bad = []
    try:
        for off in (0, 3):
            xs = x.copy()
            for k, p in enumerate(edge_positions(n, min((8 - off) % 8, n), 8, 1)):
                xs[p] = specials[k % len(specials)]
            xd = Dev(rt1, xs, off)
            try:
                for mapc in PRED_MAPS:
                    for p in (params if mapc < 22 else params[:1]):
                        with np.errstate(invalid="ignore"):
                            m = {16: xs == p, 17: xs != p, 18: xs < p, 19: xs <= p, 20: xs > p, 21: xs >= p, 22: np.isnan(xs), 23: xs != 0}[mapc]
                        pa = np.asarray([p], dtype=np.float16)
                        for op, want in ((COUNT, int(m.sum())), (ANY, int(m.any())), (ALL, int(m.all()))):
                            _lib().call("dab_reduce", rt1.ctx, F16, op, mapc, C.c_void_p(pa.ctypes.data), C.c_void_p(xd.ptr), n, C.c_void_p(slot.ptr))
                            got = int(slot.get(16, np.uint8)[:8].view(np.int64)[0])
                            if got != want:
                                bad.append(f"off={off} map={mapc} param={p!r} op={op}: got {got} want {want}")
            finally:
                xd.free()
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:12]) + f" ({len(bad)} cases)"


# ---------------------------------------------------------------------------------------------------------- (c) the fused step
@pytest.mark.parametrize("dt", [I32, I64], ids=["i32", "i64"])
@pytest.mark.parametrize("n", [4096 * 3 + 5, (1 << 20) + 7])
def test_fused_affine_reduce_wraps(dab, rt1, dt, n):
    """y .= a.*x .+ b with a wrapping y, then sum / prod / maximum / minimum of y: the fused kernel stores the wrapped y and reduces
    it with Int64 widening; the expected value is computed from the wrapped y."""
    T = NP[dt]
    rng = np.random.default_rng(n + dt)
    a, b = (T(65537), T(2 ** 31 - 1)) if dt == I32 else (T((1 << 33) + 1), T((1 << 62) + 1))
    x = (rng.integers(np.iinfo(T).min // 4, np.iinfo(T).max // 4, n, dtype=np.int64).astype(T) * T(2))   # even x: y is odd
    with np.errstate(all="ignore"):
        y_want = (a * x + b).astype(T)
    av, bv = np.asarray(a), np.asarray(b)
    for op in OPS:
        xd = Dev(rt1, x, 1)
        yd = Dev(rt1, np.zeros(n, dtype=T), 1)
        slot = Dev(rt1, np.zeros(16, dtype=np.uint8), 0)
        try:
            n0 = rt1.launches()
            _lib().call("dab_affine", rt1.ctx, dt, C.c_void_p(yd.ptr), C.c_void_p(xd.ptr), C.c_void_p(av.ctypes.data), C.c_void_p(bv.ctypes.data), n)
            s = reduce_call(rt1, dt, op, MAP_ID, yd, n, slot)
            if not HOSTMEM:
                assert rt1.launches() - n0 == 1, "the reduce did not consume the deferred dab_affine"
            rdt = result_dtype(T, op)
            assert slot_value(s, rdt) == ref_reduce(y_want, op, axis=0), (op, slot_value(s, rdt), ref_reduce(y_want, op, axis=0))
            assert np.array_equal(yd.get(), y_want)
        finally:
            xd.free()
            yd.free()
            slot.free()


# ---------------------------------------------------------------------------------------------------------- (d) public API
def test_int32_sum_prod_widen_before_wrapping(dab, rt1):
    """Int32 sum / prod widen before they can wrap: one worker (dab_mapreduce_all) and dims=1."""
    assert dab.sum(dab.distribute(np.full(4, 2 ** 30, dtype=np.int32))) == 4294967296
    assert dab.prod(dab.distribute(np.asarray([65536, 65536, 1, 1], dtype=np.int32))) == 4294967296
    A = np.full((4, 9), 2 ** 30, dtype=np.int32, order="F")
    r = dab.to_array(dab.sum(dab.distribute(A), dims=1))
    assert r.dtype == np.int64 and np.array_equal(r, np.full((1, 9), 4294967296, dtype=np.int64))
    assert dab.sum(dab.distribute(np.full(4, 2 ** 30, dtype=np.int32)), lambda v: abs(v)) == 4294967296


@pytest.mark.parametrize("dt", [F32, F64, I32, I64], ids=["f32", "f64", "i32", "i64"])
def test_public_api_multichunk_exact(dab, rt8, dt):
    """sum / prod / maximum / minimum on 8-chunk layouts, whole-array, with dims and with init=, against the exact reference."""
    T = NP[dt]
    shape = (37, 1200)
    isf = np.dtype(T).kind == "f"
    # float inputs: finite values only, then the signed-zero rule of the op (every column <= 0 with a +0.0 for max, >= 0 with a -0.0
    # for min), then every kind (NaN and +-Inf columns included)
    cases = [(op, kinds) for op in OPS for kinds in (((4, 5, 6, 7), {MAX: (2,), MIN: (3,)}.get(op, FINITE_KINDS), None) if isf else (None,))]
    finite_nonzero = set()
    for op, kinds in cases:
        fn, sym = {SUM: (dab.sum, "+"), PROD: (dab.prod, "*"), MAX: (dab.maximum, "max"), MIN: (dab.minimum, "min")}[op]
        x = build(dt, op, 1, shape[0], shape[1], edge_positions(shape[0], 0, 16 // np.dtype(T).itemsize, 1), seed=op + 100 * dt, kinds=kinds)
        A = np.asfortranarray(x.reshape(shape, order="F"))
        if op == PROD and np.dtype(T).kind == "f":
            A = np.asfortranarray(A[:, :40])                    # keep every whole-array product inside the exponent range
        d = dab.distribute(A)
        rdt = result_dtype(T, op)
        whole = fn(d)
        want_whole = np.asarray([ref_reduce(A.reshape(-1), op, axis=0)], dtype=rdt)
        assert same_bits(np.asarray([whole], dtype=rdt), want_whole), (op, kinds, whole, want_whole)
        if np.isfinite(want_whole[0]) and want_whole[0] != 0:
            finite_nonzero.add(op)
        for dims in (1, 2, (1, 2)):
            ax = {1: (0,), 2: (1,), (1, 2): (0, 1)}[dims]
            want = A.astype(np.int64) if rdt == np.int64 else A
            want = ref_reduce(want.reshape(A.shape[0], -1) if ax == (1,) else want, op, axis=ax[0]) if len(ax) == 1 else \
                np.asarray(ref_reduce(A.reshape(-1), op, axis=0)).reshape(1, 1)
            want = np.expand_dims(want, ax[0]) if len(ax) == 1 else want
            got = dab.to_array(fn(d, dims=dims))
            assert same_bits(got, np.asarray(want, dtype=rdt)), (op, dims)
            init = {SUM: 5, PROD: -1, MAX: 3, MIN: -3}[op]
            got = dab.to_array(dab.reduce(sym, d, dims=dims, init=init))
            assert same_bits(got, ref_combine(np.full(np.shape(want), init, dtype=rdt), np.asarray(want, dtype=rdt), op)), (op, dims, "init")
    assert finite_nonzero == set(OPS), set(OPS) - finite_nonzero


def test_int32_sum_nvrtc_path_agrees(dab, rt8):
    """An Int32 sum through a closure the kernels do not know (one fused NVRTC kernel per chunk) equals the hand-written kernel
    and the reference, with and without dims."""
    rng = np.random.default_rng(3)
    mag = rng.integers(1 << 30, 1 << 31, (33, 257), dtype=np.int64)
    A = np.asfortranarray(np.where(rng.random(mag.shape) < 0.5, -mag, mag - 1).astype(np.int32))
    d = dab.distribute(A)
    want = int(A.astype(np.int64).sum())
    assert dab.mapreduce(lambda v: v + v - v, "+", d) == dab.sum(d) == want
    got = dab.to_array(dab.mapreduce(lambda v: v + v - v, "+", d, dims=1))
    assert np.array_equal(got, dab.to_array(dab.sum(d, dims=1))) and np.array_equal(got, A.astype(np.int64).sum(axis=0, keepdims=True))
    assert float(dab.mean(d)) == want / A.size
