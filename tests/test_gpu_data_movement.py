"""The data-movement kernels against a byte-exact model, on every dispatch path.

Four kernels move data between chunks: ``dab_copy_box`` (the K8 halo read, ``dab_slab.cu``), ``dab_gather_box`` (strided and
vector-indexed views, ``dab_slab.cu``), ``dab_transpose_box`` (K10, ``dab_gemv.cu``) and ``dab_adjoint_box`` (the conjugating
transpose of complex chunks, ``dab_gemv.cu``).  Every mixed-layout broadcast, ``getindex``, ``DArray(::SubDArray)``, ``copy(transpose(D))``,
the halos of ``A*x`` / ``A*B``, the sort's sample gather and the slice packing of ``mapslices`` / ``ppeval`` go through them.

They are called here through the C ABI with operands placed at chosen byte offsets from 256-byte aligned allocations.  Source and
destination allocations are filled with random bytes that include, viewed as floats, NaNs with payloads (quiet and signalling, both
signs), +-0, +-Inf and subnormals.  The expected destination is computed on the host from the bytes alone: every byte inside the box
equals its source byte, every byte outside it (gaps between rows, the bytes around the operand) is unchanged.  ``dab_adjoint_box`` is
held to Julia's ``conj``: the imaginary part's sign bit flipped, NaN payloads kept.

The host-side dispatch is mirrored below (``copy_plan``, ``transpose_labels``, ``gather_labels``), so that
``test_case_table_reaches_every_path`` can show which kernel instances and branches the case table selects; the copy tests also check
the mirror's launch count against the library's launch counter.
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
F32, F64, I32, I64, U8, I128, C64, C128 = range(8)
WIDTHS = (1, 2, 4, 8, 16)
LEAD, TRAIL = 64, 64                 # canary bytes before and after every operand (LEAD keeps the 256-byte phase mod 16)


def _lib():
    from darray_b200 import _lib as L
    return L


# ---------------------------------------------------------------------------------------------------------- random bytes
F32_SPECIALS = np.asarray([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x807FFFFF, 0x00400000, 0x7FC00000,
                           0xFFC00000, 0x7FC12345, 0xFFE54321, 0x7F800001, 0xFFA5A5A5, 0x7FFFFFFF, 0xFFFFFFFF], dtype=np.uint32)
F64_SPECIALS = np.asarray([0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001,
                           0x800FFFFFFFFFFFFF, 0x0008000000000000, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000012345678,
                           0xFFFC000087654321, 0x7FF0000000000001, 0xFFF5A5A5A5A5A5A5, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF],
                          dtype=np.uint64)


def rand_bytes(rng, n):
    """n random bytes; about one 4-byte word in 6 and one 8-byte word in 10 replaced by a float special (NaN payloads, +-0, +-Inf,
    subnormals)."""
    b = rng.integers(0, 256, n, dtype=np.uint8)
    w4 = b[:n - n % 4].view(np.uint32)
    k = rng.random(w4.size) < 1 / 6
    w4[k] = F32_SPECIALS[rng.integers(0, F32_SPECIALS.size, int(k.sum()))]
    w8 = b[:n - n % 8].view(np.uint64)
    k = rng.random(w8.size) < 1 / 10
    w8[k] = F64_SPECIALS[rng.integers(0, F64_SPECIALS.size, int(k.sum()))]
    return b


class Dev:
    """``host`` (bytes) on the device at byte offset ``LEAD + off`` from a 256-byte aligned allocation, between random canary bytes.
    ``img`` is the whole allocation as uploaded; ``at`` is where the operand starts in it."""

    def __init__(self, rt, host, off, rng):
        host = np.ascontiguousarray(host).reshape(-1).view(np.uint8)
        self.rt, self.at = rt, LEAD + off
        self.img = rand_bytes(rng, self.at + host.size + TRAIL)
        self.img[self.at:self.at + host.size] = host
        self.base = rt.alloc(self.img.size)
        self.ptr = self.base + self.at
        _lib().call("dab_h2d", rt.ctx, C.c_void_p(self.base), C.c_void_p(self.img.ctypes.data), self.img.size)
        rt.sync()

    def get(self):
        out = np.empty(self.img.size, dtype=np.uint8)
        _lib().call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.base), out.size)
        self.rt.sync()
        return out

    def free(self):
        self.rt.free(self.base)


def diff_report(got, want, at):
    bad = np.flatnonzero(got != want)
    return f"{bad.size} bytes differ, first at operand byte {(bad[:4] - at).tolist()}: got {got[bad[:4]].tolist()} want {want[bad[:4]].tolist()}"


# ---------------------------------------------------------------------------------------------------------- dispatch mirrors
def pow2_align(bits):
    """dab_slab.cu:95-99: the widest power of two <= 16 that divides ``bits``."""
    v = 16
    while v > 1 and bits & (v - 1):
        v >>= 1
    return v


def copy_rows(t, s, row_bytes, e, spp, dpp):
    """dab_slab.cu:101-124 + launch_copy_s (:82-93) + launch_copy (:68-80): one launch as (load unit, store unit, index bits)."""
    sbits, dbits = s | row_bytes, t | row_bytes
    for d in range(3):
        if e[d] > 1:
            sbits |= spp[d]
            dbits |= dpp[d]
    U, svec = pow2_align(sbits), pow2_align(dbits)
    total = row_bytes // U * e[0] * e[1] * e[2]
    return (U, min(U, svec), 32 if total < 1 << 31 else 64)


def copy_plan(es, t0, dshape, doff, s0, sshape, soff, ext):
    """dab_copy_box (dab_slab.cu:170-231) on the host, for a destination at address t0 and a source at s0: the launches as
    (load unit, store unit, index bits), the collapse depth, whether an extent-1 dimension with a larger one behind it was dropped,
    the contiguous row length after the collapse and the peel pieces."""
    if 0 in ext:
        return dict(launches=[], depth=None, dropped_unit=False, row=0, pieces=None)
    sp, dp = [es], [es]
    for d in range(1, 4):
        sp.append(sp[-1] * sshape[d - 1])
        dp.append(dp[-1] * dshape[d - 1])
    s = s0 + sum(soff[d] * sp[d] for d in range(4))
    t = t0 + sum(doff[d] * dp[d] for d in range(4))
    row = ext[0] * es                                           # the collapse loop, :195-212
    e, spp, dpp = list(ext[1:]), sp[1:], dp[1:]
    nd, depth, dropped_unit = 3, 0, False
    while nd > 0 and ((spp[0] == row and dpp[0] == row) or e[0] == 1):
        if e[0] > 1:
            row *= e[0]
        elif any(x > 1 for x in e[1:nd]) and not (spp[0] == row and dpp[0] == row):
            dropped_unit = True
        e, spp, dpp = e[1:] + [1], spp[1:] + [0], dpp[1:] + [0]
        nd -= 1
        depth += 1
    if nd == 0 and row >= 4096:                                 # the peel, :213-229
        head = (16 - (s & 15)) & 15
        head -= head % es
        body = (row - head) & ~15
        tail = row - head - body
        pieces = [(x, n, name) for x, n, name in ((0, head, "head"), (head, body, "body"), (head + body, tail, "tail")) if n]
        launches = [copy_rows(t + x, s + x, n, e, spp, dpp) for x, n, _ in pieces]
        return dict(launches=launches, depth=depth, dropped_unit=dropped_unit, row=row, pieces="+".join(p[2] for p in pieces))
    return dict(launches=[copy_rows(t, s, row, e, spp, dpp)], depth=depth, dropped_unit=dropped_unit, row=row, pieces=None)


def copy_labels(plan):
    out = {f"copy U={U} S={S} i{bits}" for U, S, bits in plan["launches"]}
    if plan["depth"] is not None:
        out.add(f"collapse depth {plan['depth']}")
    if plan["dropped_unit"]:
        out.add("collapse drops an extent-1 middle dim")
    if plan["pieces"]:
        out.add(f"peel {plan['pieces']}")
    if plan["depth"] == 3 and plan["row"] in (4095, 4096):
        out.add(f"slab {plan['row']} bytes " + ("peeled" if plan["pieces"] else "not peeled"))
    return out


VEC4_CONDITIONS = ("rows%4", "cols%4", "src_ld%4", "dst_ld%4", "src%16", "dst%16")


def transpose_labels(es, dst, dst_ld, src, src_ld, rows, cols):
    """launch_transpose (dab_gemv.cu:763-780): the vec4 kernel needs all six conditions of :769; else transpose_box_kernel<U>."""
    if rows == 0 or cols == 0:
        return set()
    if es == 4:
        fails = [c for c, ok in zip(VEC4_CONDITIONS, (rows % 4 == 0, cols % 4 == 0, src_ld % 4 == 0, dst_ld % 4 == 0, src % 16 == 0,
                                                      dst % 16 == 0)) if not ok]
        if not fails:
            return {"transpose vec4"}
        return {"transpose U=4"} | ({f"vec4 fallback on {fails[0]} alone"} if len(fails) == 1 else set())
    return {f"transpose U={es}"}


def gather_labels(es, g):
    """dab_gather_box (dab_slab.cu:233-259, the width switch at :251-258): gather_box_kernel<U> with sizeof(U) = elem_bytes, and the kinds of dimensions."""
    out = {f"gather {es}B ndim={len(g['ext'])}"}
    for k in range(len(g["ext"])):
        out.add(f"gather {es}B src {g['skind'][k]}")
        if g["dtab"][k] is not None:
            out.add(f"gather {es}B dst table")
    return out


REQUIRED = ({f"copy U={U} S={S} i32" for U in WIDTHS for S in WIDTHS if S <= U} | {"copy U=1 S=1 i64"}
            | {f"peel {p}" for p in ("head+body", "body", "head+body+tail", "body+tail")}
            | {"slab 4096 bytes peeled", "slab 4095 bytes not peeled"}
            | {f"collapse depth {k}" for k in range(4)} | {"collapse drops an extent-1 middle dim"}
            | {f"transpose U={u}" for u in WIDTHS} | {"transpose vec4"} | {f"vec4 fallback on {c} alone" for c in VEC4_CONDITIONS}
            | {"adjoint C64", "adjoint C128"}
            | {f"gather {es}B ndim={nd}" for es in WIDTHS for nd in (1, 2, 4, 8)}
            | {f"gather {es}B src {k}" for es in WIDTHS for k in ("table", "negative stride", "zero stride", "positive stride")}
            | {f"gather {es}B dst table" for es in WIDTHS})


# ---------------------------------------------------------------------------------------------------------- case tables
def copy_geoms(es):
    """name -> (src shape, src offset, dst shape, dst offset, extent), in elements, up to 4-D, column-major."""
    g = {
        "1d_ragged": ((301,), (7,), (290,), (3,), (283,)),
        "2d_box": ((67, 9), (3, 1), (71, 10), (5, 2), (33, 7)),
        "2d_ragged_rows": ((129, 5), (0, 1), (130, 6), (1, 0), (127, 4)),
        "3d_span_dim1": ((20, 6, 5), (0, 1, 1), (20, 7, 5), (0, 2, 0), (20, 4, 3)),
        "3d_spans_to_slab": ((10, 4, 6), (0, 0, 1), (10, 4, 7), (0, 0, 2), (10, 4, 5)),
        "4d_spans_then_box": ((8, 3, 4, 5), (0, 0, 0, 2), (8, 3, 5, 6), (0, 0, 1, 1), (8, 3, 4, 2)),
        "4d_unit_middle": ((30, 5, 7, 3), (2, 1, 3, 0), (31, 2, 6, 4), (0, 1, 2, 1), (17, 1, 4, 2)),
        "4d_ragged": ((13, 7, 5, 4), (1, 2, 0, 1), (12, 9, 6, 3), (0, 1, 1, 0), (11, 5, 4, 3)),
        "slab_by_collapse": ((64, 20), (0, 3), (64, 12), (0, 2), (64, 9)),
    }
    for nbytes in (4095, 4096, 5000, 6000):                    # contiguous slabs: the 4096-byte peel threshold, tails of 8 and 0 mod 16
        if nbytes % es == 0:
            n = nbytes // es
            g[f"slab_{nbytes}"] = ((n + 9,), (5,), (n + 3,), (1,), (n,))
    def to4(v, i):                                             # shapes and extents pad with 1, offsets (items 1 and 3) with 0
        return tuple(v) + (0 if i in (1, 3) else 1,) * (4 - len(v))

    return {k: tuple(to4(v, i) for i, v in enumerate(geo)) for k, geo in g.items()}


def phases(es):
    return list(range(0, 16, es))


def copy_cases(es):
    """Every geometry at every pair of (box start) phases mod 16 for source and destination."""
    return [(name, ps, pd) for name in copy_geoms(es) for ps in phases(es) for pd in phases(es)]


def box_phase_placement(es, shape, off, phase):
    """Byte offset of the operand (mod 16, a multiple of es) that puts the box start at ``phase`` mod 16."""
    pitch, start = es, 0
    for d in range(4):
        start += off[d] * pitch
        pitch *= shape[d]
    return (phase - start) % 16


TRANSPOSE_SHAPES = ((1, 1), (1, 77), (77, 1), (1, 300), (300, 1), (37, 53), (65, 129), (100, 3), (64, 64), (96, 32), (200, 130),
                    (129, 257))


def transpose_cases(es):
    """(rows, cols, src_ld, dst_ld, src phase, dst phase): every shape with tight and padded leading dimensions at two phase pairs;
    for 4-byte units the vec4 kernel and each of its six fallback reasons alone."""
    P = phases(es)
    pairs = [(a, b) for a in P for b in P]
    out = []
    for k, (r, c) in enumerate(TRANSPOSE_SHAPES):
        for j, (sld, dld) in enumerate(((r, c), (r + 3, c + 5))):
            out.append((r, c, sld, dld) + pairs[0])
            out.append((r, c, sld, dld) + pairs[(7 * k + 3 * j + 1) % len(pairs)])
    if es == 4:
        out += [(128, 68, 132, 72, 0, 0), (64, 64, 64, 64, 0, 0), (4, 4, 4, 4, 0, 0),
                (130, 68, 132, 68, 0, 0), (128, 67, 128, 68, 0, 0), (128, 68, 131, 68, 0, 0), (128, 68, 128, 69, 0, 0),
                (128, 68, 128, 68, 4, 0), (128, 68, 128, 68, 0, 8)]
    return out


def adjoint_cases(dt):
    es = 8 if dt == C64 else 16
    P = list(range(0, 16, es))
    out = []
    for k, (r, c) in enumerate(TRANSPOSE_SHAPES):
        for sld, dld in ((r, c), (r + 3, c + 5)):
            out.append((r, c, sld, dld, P[k % len(P)], P[(k + 1) % len(P)]))
    return out


def gather_geom(es, nd, seed):
    """A random gather: per dimension the destination is a padded, possibly reversed, stride or a permuted index table; the source a
    positive, negative or zero stride or an index table with repeats, out of order.  Offsets are in elements, relative to the
    operand pointers, which sit where every offset stays inside the buffer."""
    rng = np.random.default_rng(seed)
    maxe = {1: 300, 2: 40, 3: 12, 4: 7, 5: 5, 6: 4, 7: 3, 8: 3}[nd]
    ext = [int(v) for v in rng.integers(1, maxe + 1, nd)]
    ext[int(rng.integers(nd))] = max(2, ext[0])                 # at least one dimension longer than 1
    kinds = ["positive stride", "negative stride", "zero stride", "table"]
    skind = [kinds[(k + seed) % 4] for k in range(nd)]
    dstr, dtab, sstr, stab = [], [], [], []
    dr, sr = 1, 1
    for k in range(nd):
        sign = -1 if rng.random() < 0.25 else 1
        if rng.random() < 1 / 3 or (nd >= 4 and k == seed % nd):
            dtab.append((rng.permutation(ext[k]) * dr * sign).astype(np.int64))
            dstr.append(0)
        else:
            dtab.append(None)
            dstr.append(dr * sign)
        dr *= ext[k] + int(rng.integers(0, 3))
        span = ext[k] + int(rng.integers(0, 4))
        if skind[k] == "table":
            t = rng.integers(-span // 2, span - span // 2, ext[k]).astype(np.int64)
            if ext[k] >= 2:
                t[-1] = t[0]                                    # a repeat
            stab.append(t * sr)
            sstr.append(0)
        else:
            stab.append(None)
            sstr.append({"positive stride": sr, "negative stride": -sr, "zero stride": 0}[skind[k]])
        sr *= span
    return dict(ext=ext, dstr=dstr, dtab=dtab, sstr=sstr, stab=stab, skind=skind)


def gather_cases(es):
    return [(nd, 100 * nd + j) for nd in range(1, 9) for j in range(5 if nd in (1, 2, 4, 8) else 2)]


# the one copy that takes the 64-bit index: a Bool source of 65537 x 32769, a 65535 x 32769 box that does not collapse
LARGE_COPY = dict(es=1, sshape=(65537, 32769, 1, 1), soff=(1, 0, 0, 0), dshape=(65536, 32769, 1, 1), doff=(1, 0, 0, 0),
                  ext=(65535, 32769, 1, 1))


def test_case_table_reaches_every_path(capsys):
    """The case tables below reach every kernel instance and host branch of the four entry points; the list of what is reached is
    printed (``-s``) for comparison with the dispatch code."""
    got = set()
    for es in WIDTHS:
        geoms = copy_geoms(es)
        for name, ps, pd in copy_cases(es):
            sshape, soff, dshape, doff, ext = geoms[name]
            assert all(o + e <= n for o, e, n in zip(soff + doff, ext + ext, sshape + dshape)), name     # every case is a valid box
            s0 = 4096 + LEAD + box_phase_placement(es, sshape, soff, ps)
            t0 = 8192 + LEAD + box_phase_placement(es, dshape, doff, pd)
            got |= copy_labels(copy_plan(es, t0, dshape, doff, s0, sshape, soff, ext))
        for r, c, sld, dld, ps, pd in transpose_cases(es):
            got |= transpose_labels(es, 8192 + LEAD + pd, dld, 4096 + LEAD + ps, sld, r, c)
        for nd, seed in gather_cases(es):
            got |= gather_labels(es, gather_geom(es, nd, seed))
    for dt in (C64, C128):
        if adjoint_cases(dt):
            got.add("adjoint C64" if dt == C64 else "adjoint C128")
    L = LARGE_COPY
    got |= copy_labels(copy_plan(1, LEAD + 1, L["dshape"], L["doff"], LEAD, L["sshape"], L["soff"], L["ext"]))
    with capsys.disabled():
        print("\npaths reached by the case table:\n  " + "\n  ".join(sorted(got)))
    assert REQUIRED <= got, sorted(REQUIRED - got)


# ---------------------------------------------------------------------------------------------------------- dab_copy_box
def copy_model(es, dst_img, dat, dshape, doff, src_img, sat, sshape, soff, ext):
    want = dst_img.copy()
    d = want[dat:dat + es * int(np.prod(dshape))].reshape((es,) + tuple(dshape), order="F")
    s = src_img[sat:sat + es * int(np.prod(sshape))].reshape((es,) + tuple(sshape), order="F")
    d[(slice(None),) + tuple(slice(o, o + e) for o, e in zip(doff, ext))] = s[(slice(None),) + tuple(slice(o, o + e) for o, e in zip(soff, ext))]
    return want


def copy_call(rt, es, dst, dshape, doff, src, sshape, soff, ext):
    L = _lib()
    L.call("dab_copy_box", rt.ctx, es, C.c_void_p(dst.ptr), L.sz4(dshape), L.sz4(doff), C.c_void_p(src.ptr), L.sz4(sshape), L.sz4(soff),
           L.sz4(ext))
    rt.sync()


@pytest.mark.parametrize("es", WIDTHS)
def test_copy_box_bit_exact(dab, rt1, es):
    rng = np.random.default_rng(es)
    geoms = copy_geoms(es)
    bad = []
    for name, ps, pd in copy_cases(es):
        sshape, soff, dshape, doff, ext = geoms[name]
        src = Dev(rt1, rand_bytes(rng, es * int(np.prod(sshape))), box_phase_placement(es, sshape, soff, ps), rng)
        dst = Dev(rt1, rand_bytes(rng, es * int(np.prod(dshape))), box_phase_placement(es, dshape, doff, pd), rng)
        try:
            plan = copy_plan(es, dst.ptr, dshape, doff, src.ptr, sshape, soff, ext)
            n0 = rt1.launches()
            copy_call(rt1, es, dst, dshape, doff, src, sshape, soff, ext)
            nl = rt1.launches() - n0
            got, want = dst.get(), copy_model(es, dst.img, dst.at, dshape, doff, src.img, src.at, sshape, soff, ext)
            if not np.array_equal(got, want):
                bad.append(f"{name} src phase {ps} dst phase {pd} {plan['launches']} {plan['pieces']}: {diff_report(got, want, dst.at)}")
            if not np.array_equal(src.get(), src.img):
                bad.append(f"{name} src phase {ps} dst phase {pd}: the source changed")
            if not HOSTMEM and nl != len(plan["launches"]):
                bad.append(f"{name} src phase {ps} dst phase {pd}: {nl} launches, the mirror expects {plan['launches']}")
        finally:
            src.free()
            dst.free()
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:8])


def test_copy_box_index_64(dab, rt1):
    """A 1-byte box of 65535 x 32769 = 2,147,516,415 load units (> 2^31) that does not collapse: copy_box_kernel<char, char,
    unsigned long long, 8>, checked over the whole destination on the host.  Only the 1-byte pair takes the 64-bit index at a size
    that fits beside the other tests; the other 14 (load, store) instances with the 64-bit index are the same template code, and
    reaching them needs boxes of up to 64 GiB, so they are not run here."""
    L = LARGE_COPY
    sshape, soff, dshape, doff, ext = L["sshape"], L["soff"], L["dshape"], L["doff"], L["ext"]
    if rt1.device_info()["free_bytes"] < 8 * 2 ** 30:
        pytest.skip("needs 8 GiB of free device memory")
    plan = copy_plan(1, 256, dshape, doff, 0, sshape, soff, ext)
    assert plan["launches"] == [(1, 1, 64)] and plan["depth"] == 0, plan
    rng = np.random.default_rng(64)
    ns, nd = sshape[0] * sshape[1], dshape[0] * dshape[1]
    lib = _lib()
    sp, dp = rt1.alloc(ns), rt1.alloc(nd)
    try:
        src = np.frombuffer(rng.bytes(ns), dtype=np.uint8)
        lib.call("dab_h2d", rt1.ctx, C.c_void_p(sp), C.c_void_p(src.ctypes.data), ns)
        canary = np.full(nd, 0xA5, dtype=np.uint8)
        lib.call("dab_h2d", rt1.ctx, C.c_void_p(dp), C.c_void_p(canary.ctypes.data), nd)
        rt1.sync()
        del canary
        lib.call("dab_copy_box", rt1.ctx, 1, C.c_void_p(dp), lib.sz4(dshape), lib.sz4(doff), C.c_void_p(sp), lib.sz4(sshape), lib.sz4(soff),
                 lib.sz4(ext))
        rt1.sync()
        got = np.empty(nd, dtype=np.uint8)
        lib.call("dab_d2h", rt1.ctx, C.c_void_p(got.ctypes.data), C.c_void_p(dp), nd)
        rt1.sync()
    finally:
        rt1.free(sp)
        rt1.free(dp)
    s = src.reshape(sshape[:2], order="F")
    d = got.reshape(dshape[:2], order="F")
    assert (d[0] == 0xA5).all(), "the canary row of the destination was written"
    for c0 in range(0, ext[1], 4096):                           # column blocks: no full-size temporaries
        c1 = min(c0 + 4096, ext[1])
        blk_ok = np.array_equal(d[1:, c0:c1], s[1:1 + ext[0], c0:c1])
        assert blk_ok, f"columns {c0}..{c1 - 1} differ"


# ---------------------------------------------------------------------------------------------------------- dab_transpose_box / dab_adjoint_box
def transpose_model(es, dst_img, dat, dst_ld, src_img, sat, src_ld, rows, cols, conj=False):
    want = dst_img.copy()
    s = src_img[sat:sat + es * src_ld * cols].reshape((es, src_ld, cols), order="F")[:, :rows, :]
    d = want[dat:dat + es * dst_ld * rows].reshape((es, dst_ld, rows), order="F")
    d[:, :cols, :] = s.transpose(0, 2, 1)
    if conj:
        d[es - 1, :cols, :] ^= 0x80                             # little endian: the imaginary part's sign bit is the element's top bit
    return want


def run_transpose(rt, entry, code, es, case, rng, src_bytes=None):
    r, c, sld, dld, ps, pd = case
    src = Dev(rt, rand_bytes(rng, es * sld * c) if src_bytes is None else src_bytes, ps, rng)
    dst = Dev(rt, rand_bytes(rng, es * dld * r), pd, rng)
    try:
        _lib().call(entry, rt.ctx, code, C.c_void_p(dst.ptr), dld, C.c_void_p(src.ptr), sld, r, c)
        rt.sync()
        got = dst.get()
        want = transpose_model(es, dst.img, dst.at, dld, src.img, src.at, sld, r, c, conj=entry == "dab_adjoint_box")
        msg = None if np.array_equal(got, want) else f"{r}x{c} src_ld {sld} dst_ld {dld} phases {ps}/{pd}: {diff_report(got, want, dst.at)}"
        if msg is None and not np.array_equal(src.get(), src.img):
            msg = f"{r}x{c}: the source changed"
        return msg
    finally:
        src.free()
        dst.free()


@pytest.mark.parametrize("es", WIDTHS)
def test_transpose_box_bit_exact(dab, rt1, es):
    rng = np.random.default_rng(100 + es)
    bad = [m for case in transpose_cases(es) if (m := run_transpose(rt1, "dab_transpose_box", es, es, case, rng))]
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:8])


def complex_source(rng, dt, n):
    """n complex values of random bytes whose imaginary parts run through the specials (+-0, +-Inf, subnormals, NaNs of both signs with
    quiet and signalling payloads) at every third element."""
    u = np.uint32 if dt == C64 else np.uint64
    sp = F32_SPECIALS if dt == C64 else F64_SPECIALS
    w = rand_bytes(rng, n * 2 * np.dtype(u).itemsize).view(u).reshape(n, 2)
    k = np.arange(0, n, 3)
    w[k, 1] = sp[np.arange(k.size) % sp.size]
    w[k[1::2], 0] = sp[(np.arange(k[1::2].size) * 7 + 3) % sp.size]
    return w.reshape(-1).view(np.uint8)


@pytest.mark.parametrize("dt", [C64, C128], ids=["c64", "c128"])
def test_adjoint_box_bit_exact(dab, rt1, dt):
    """conj(transpose(A)) bit for bit: the real part unchanged, the imaginary part's sign bit flipped (Julia's conj keeps NaN payloads)."""
    es = 8 if dt == C64 else 16
    rng = np.random.default_rng(200 + dt)
    bad = [m for case in adjoint_cases(dt)
           if (m := run_transpose(rt1, "dab_adjoint_box", dt, es, case, rng, src_bytes=complex_source(rng, dt, case[2] * case[1])))]
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:8])


# ---------------------------------------------------------------------------------------------------------- dab_gather_box
def gather_offsets(ext, strides, tables):
    tot = np.zeros((), dtype=np.int64)
    for k in range(len(ext)):
        o = tables[k] if tables[k] is not None else np.arange(ext[k], dtype=np.int64) * strides[k]
        tot = tot[..., None] + o
    return tot.reshape(-1)


@pytest.mark.parametrize("es", WIDTHS)
def test_gather_box_bit_exact(dab, rt1, es):
    rng = np.random.default_rng(300 + es)
    L = _lib()
    bad = []
    for nd, seed in gather_cases(es):
        g = gather_geom(es, nd, seed)
        do, so = gather_offsets(g["ext"], g["dstr"], g["dtab"]), gather_offsets(g["ext"], g["sstr"], g["stab"])
        assert np.unique(do).size == do.size
        dlo, slo = int(do.min()), int(so.min())
        nd_el, ns_el = int(do.max()) - dlo + 1, int(so.max()) - slo + 1
        pd, ps = phases(es)[seed % len(phases(es))], phases(es)[(seed // 3) % len(phases(es))]
        src = Dev(rt1, rand_bytes(rng, es * ns_el), ps, rng)
        dst = Dev(rt1, rand_bytes(rng, es * nd_el), pd, rng)
        tabs = [t for t in g["dtab"] + g["stab"] if t is not None]
        tdev = Dev(rt1, np.concatenate(tabs) if tabs else np.zeros(1, dtype=np.int64), 0, rng)
        try:
            ptrs, pos = [], 0
            for t in g["dtab"] + g["stab"]:
                ptrs.append(None if t is None else tdev.ptr + 8 * pos)
                pos += 0 if t is None else t.size
            VP, LL = C.c_void_p * nd, C.c_longlong * nd
            di = VP(*ptrs[:nd]) if any(p is not None for p in ptrs[:nd]) else None
            si = VP(*ptrs[nd:]) if any(p is not None for p in ptrs[nd:]) else None
            L.call("dab_gather_box", rt1.ctx, es, nd, C.c_void_p(dst.ptr - dlo * es), LL(*g["dstr"]), di, C.c_void_p(src.ptr - slo * es),
                   LL(*g["sstr"]), si, (C.c_size_t * nd)(*g["ext"]))
            rt1.sync()
            got = dst.get()
            want = dst.img.copy()
            d_el = want[dst.at:dst.at + es * nd_el].reshape(nd_el, es)
            s_el = src.img[src.at:src.at + es * ns_el].reshape(ns_el, es)
            d_el[do - dlo] = s_el[so - slo]
            if not np.array_equal(got, want):
                bad.append(f"ndim {nd} seed {seed} ext {g['ext']} src {g['skind']}: {diff_report(got, want, dst.at)}")
        finally:
            src.free()
            dst.free()
            tdev.free()
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:8])


# ---------------------------------------------------------------------------------------------------------- refusals
def test_refusals_write_nothing(dab, rt1):
    """Zero extents are a no-op; a box past either array, a leading dimension below the box, an invalid element width or dimension
    count and a real dtype for the adjoint are refused before any launch.  The destination is checked byte for byte after each."""
    L = _lib()
    rng = np.random.default_rng(7)
    src = Dev(rt1, rand_bytes(rng, 4096), 0, rng)
    dst = Dev(rt1, rand_bytes(rng, 4096), 0, rng)
    sshape, dshape = (8, 4, 4, 2), (8, 4, 4, 2)                 # 8 B elements: 2 KiB of 4 KiB
    try:
        def untouched(what, fn, exc=None):
            n0 = rt1.launches()
            if exc is None:
                fn()
            else:
                with pytest.raises(exc):
                    fn()
            rt1.sync()
            assert np.array_equal(dst.get(), dst.img), f"{what}: the destination changed"
            if not HOSTMEM:
                assert rt1.launches() == n0, f"{what}: launched a kernel"

        def copy(es, ext, soff=(0, 0, 0, 0), doff=(0, 0, 0, 0)):
            return lambda: L.call("dab_copy_box", rt1.ctx, es, C.c_void_p(dst.ptr), L.sz4(dshape), L.sz4(doff), C.c_void_p(src.ptr), L.sz4(sshape),
                                  L.sz4(soff), L.sz4(ext))

        for d in range(4):
            ext = [8, 4, 4, 2]
            ext[d] = 0
            untouched(f"copy extent {ext}", copy(8, ext))
            ext = [8, 4, 4, 2]
            off = [0, 0, 0, 0]
            off[d] = 1
            untouched(f"copy src offset {off}", copy(8, ext, soff=off), L.DimensionMismatch)
            untouched(f"copy dst offset {off}", copy(8, ext, doff=off), L.DimensionMismatch)
            ext[d] += 1
            untouched(f"copy extent {ext}", copy(8, ext), L.DimensionMismatch)
        for es in (0, 3, 32, -8):
            untouched(f"copy elem_bytes {es}", copy(es, (2, 2, 1, 1)), L.ArgumentError)
            untouched(f"transpose elem_bytes {es}", lambda: L.call("dab_transpose_box", rt1.ctx, es, C.c_void_p(dst.ptr), 4, C.c_void_p(src.ptr),
                                                                   4, 4, 4), L.ArgumentError)

        def gather(es, nd, ext):
            LL, VP = C.c_longlong * 9, C.c_void_p * 9
            return lambda: L.call("dab_gather_box", rt1.ctx, es, nd, C.c_void_p(dst.ptr), LL(*[1] * 9), VP(), C.c_void_p(src.ptr), LL(*[1] * 9),
                                  VP(), (C.c_size_t * 9)(*ext))

        untouched("gather ndim 0", gather(4, 0, [1] * 9), L.UnsupportedError)
        untouched("gather ndim 9", gather(4, 9, [1] * 9), L.UnsupportedError)
        untouched("gather zero extent", gather(4, 3, [5, 0, 2] + [1] * 6))
        for es in (0, 3, 32):
            untouched(f"gather elem_bytes {es}", gather(es, 2, [3, 2] + [1] * 7), L.ArgumentError)
        for entry, code in (("dab_transpose_box", 8), ("dab_adjoint_box", C128)):
            def tr(rows, cols, sld, dld, entry=entry, code=code):
                return lambda: L.call(entry, rt1.ctx, code, C.c_void_p(dst.ptr), dld, C.c_void_p(src.ptr), sld, rows, cols)
            untouched(f"{entry} rows 0", tr(0, 5, 4, 5))
            untouched(f"{entry} cols 0", tr(5, 0, 5, 4))
            untouched(f"{entry} src_ld < rows", tr(6, 5, 5, 5), L.DimensionMismatch)
            untouched(f"{entry} dst_ld < cols", tr(6, 5, 6, 4), L.DimensionMismatch)
        for code in (F32, F64, I32, I64, U8):
            untouched(f"adjoint dtype {code}", lambda: L.call("dab_adjoint_box", rt1.ctx, code, C.c_void_p(dst.ptr), 4, C.c_void_p(src.ptr), 4, 4, 4),
                      L.UnsupportedError)
        assert np.array_equal(src.get(), src.img)
    finally:
        src.free()
        dst.free()
