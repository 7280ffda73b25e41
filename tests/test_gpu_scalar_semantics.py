"""Every elementwise kernel path against the model of Julia's scalar methods (tests/julia_scalar.py), bit for bit.

Three pieces of code decide what one element of ``f.(args...)`` becomes: the tracer (``_broadcast.py``: promotion, result type, Julia's
method), the hand-written kernels (``dab_unary`` / ``dab_binary`` / ``dab_binary_scalar``, element code in ``dab_scalar_ops.cuh``) and the
NVRTC kernels (``dab_bc_linear`` / ``dab_bc_rows`` / ``dab_bc_general``, ``dab_mr_partial``; element code in ``dab_jit.cu``'s prelude).
The two kernel families restate Julia's semantics separately; here both are held to the model on value grids full of the values where
elementwise code goes wrong (±0, subnormals, ties, 2^p neighbours, ±Inf, NaN of both signs with a payload, typemin / typemax), at every
16-byte phase and at the sizes where the kernels split their work, and to each other.  NaNs are compared by NaN-ness only (the device
returns the canonical quiet NaN); every other bit is compared, the sign of a zero that ``copysign`` takes from a NaN included.  Guard
bands around every output check that nothing outside ``[0, n)`` is written.
"""
import ctypes as C
import os

import numpy as np
import pytest

import julia_scalar as jl

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
F32, F64, I32, I64, U8 = range(5)
F16 = 8
CODE = {"f32": F32, "f64": F64, "i32": I32, "i64": I64, "bool": U8, "f16": F16}
MAP_ID, MAP_ABS, MAP_ABS2, MAP_NEG, MAP_SQRT, MAP_INV, MAP_FLOOR, MAP_CEIL, MAP_SIGN = range(9)
ADD, SUB, MUL, DIV, REM, BMAX, BMIN, MOD, IDIV, AND, OR, XOR = range(12)
UNARY = {MAP_ID: None, MAP_ABS: "abs", MAP_ABS2: "abs2", MAP_NEG: "neg", MAP_SQRT: "sqrt", MAP_INV: "inv", MAP_FLOOR: "floor",
         MAP_CEIL: "ceil", MAP_SIGN: "sign"}
BINARY = {ADD: "add", SUB: "sub", MUL: "mul", DIV: "div", REM: "rem", BMAX: "max", BMIN: "min", MOD: "mod", IDIV: "idiv", AND: "and",
          OR: "or", XOR: "xor"}
FLOAT_OPS = (ADD, SUB, MUL, DIV, REM, BMAX, BMIN, MOD)
INT_OPS = (ADD, SUB, MUL, REM, BMAX, BMIN, MOD, IDIV, AND, OR, XOR)
GUARD = 64                                                   # elements of sentinel before and after every output
SENTINEL = 0xA5
TAGS = ("f32", "f64", "i32", "i64")

if HOSTMEM:                                                     # the Float16 code of the host-memory emulation
    import f16_hostmem
    f16_hostmem.install()


def _lib():
    from darray_b200 import _lib as L
    return L


def _bc():
    from darray_b200 import _broadcast as bc
    return bc


def same_bits(got, want):
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


def first_bad(got, want, k=3):
    got, want = np.asarray(got), np.asarray(want)
    ok = got == want
    if got.dtype.kind == "f":
        ok = (np.isnan(got) & np.isnan(want)) | (ok & (np.signbit(got) == np.signbit(want)))
    i = np.flatnonzero(~ok)[:k]
    return [(int(j), got[j], want[j]) for j in i]


class Buf:
    """``n`` elements at element offset ``off`` past a guard band of ``GUARD`` elements, inside one allocation filled with a sentinel."""

    def __init__(self, rt, dt, n, off=0, host=None):
        self.rt, self.dt, self.n, self.off = rt, np.dtype(dt), int(n), int(off)
        self.total = self.n + 2 * GUARD + 16
        self.base = rt.alloc(self.total * self.dt.itemsize)
        self.ptr = self.base + (GUARD + self.off) * self.dt.itemsize
        self.reset()
        if host is not None:
            self.put(host)

    def reset(self):
        s = np.full(self.total * self.dt.itemsize, SENTINEL, np.uint8)
        _lib().call("dab_h2d", self.rt.ctx, C.c_void_p(self.base), C.c_void_p(s.ctypes.data), s.nbytes)

    def put(self, host):
        host = np.ascontiguousarray(np.asarray(host, dtype=self.dt))
        if host.size:
            _lib().call("dab_h2d", self.rt.ctx, C.c_void_p(self.ptr), C.c_void_p(host.ctypes.data), host.nbytes)

    def raw(self):
        out = np.empty(self.total * self.dt.itemsize, np.uint8)
        _lib().call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.base), out.nbytes)
        self.rt.sync()
        return out

    def get_checked(self, n=None, written=None):
        """The n elements, after checking that every byte outside them (or outside the ``written`` byte mask) is still the sentinel."""
        raw = self.raw()
        n = self.n if n is None else n
        lo = (GUARD + self.off) * self.dt.itemsize
        mask = np.zeros(raw.size, bool)
        if written is None:
            mask[lo:lo + n * self.dt.itemsize] = True
        else:
            mask[lo:lo + written.size] = written
        assert np.all(raw[~mask] == SENTINEL), f"write outside the output: bytes {np.flatnonzero((raw != SENTINEL) & ~mask)[:8]} (offset {lo})"
        return raw[lo:lo + n * self.dt.itemsize].view(self.dt).copy()

    def free(self):
        self.rt.free(self.base)


def sizes_for(t):
    """0, 1, VPT-1, VPT+1, one flat-grid tile (512 vectors) ± one vector ± one element, three tiles plus a tail, about 10^6."""
    vpt = 16 // np.dtype(jl.NPT[t]).itemsize
    tile = 512 * vpt
    return [0, 1, vpt - 1, vpt + 1, tile - vpt, tile - 1, tile, tile + 1, tile + vpt, 3 * tile + vpt + 3, 1_000_003]


def phases(t, nptr):
    """Equal 16-byte phases for every pointer (the vector kernels with a head peel), then each pointer alone at every other phase
    (the scalar kernels)."""
    vpt = 16 // np.dtype(jl.NPT[t]).itemsize
    out = [(k,) * nptr for k in range(vpt)]
    for j in range(nptr):
        for k in range(1, vpt):
            out.append(tuple(k if i == j else 0 for i in range(nptr)))
    return out


def tiled(m, n, rot):
    """Indices 0..m-1 tiled over n positions, rotated by rot."""
    return (np.arange(n, dtype=np.int64) + rot) % m


def _launch_layouts(t, nptr):
    """(size, phases) to run: every size at every layout, except that the sizes past three tiles run at two layouts only."""
    ph = phases(t, nptr)
    big = sizes_for(t)[-2:]
    for si, n in enumerate(sizes_for(t)):
        for lay in (ph if n not in big else (ph[0], ph[-1])):
            yield si, n, lay


# ------------------------------------------------------------------------------------------------- hand-written kernels
@pytest.mark.parametrize("t", TAGS)
def test_dab_unary_every_map(dab, rt1, t):
    g = jl.grid(t)
    T = jl.NPT[t]
    codes = [c for c in UNARY if t[0] == "f" or c not in (MAP_SQRT, MAP_INV)]
    want = {c: (g if UNARY[c] is None else jl.table1(UNARY[c], g)) for c in codes}
    for si, n, (px, py) in _launch_layouts(t, 2):
        idx = tiled(g.size, n, 7 * si)
        x = Buf(rt1, T, n, px, g[idx])
        y = Buf(rt1, T, n, py)
        for c in codes:
            y.reset()
            _lib().call("dab_unary", rt1.ctx, CODE[t], c, C.c_void_p(y.ptr), C.c_void_p(x.ptr), n)
            got = y.get_checked()
            w = want[c][idx].astype(T)
            assert same_bits(got, w), (t, UNARY[c], n, (px, py), first_bad(got, w))
        x.free()
        y.free()


@pytest.mark.parametrize("t", TAGS)
def test_dab_binary_every_op(dab, rt1, t):
    g = jl.grid(t)
    T = jl.NPT[t]
    gx, gy = jl.pairs(g, g)
    ops = FLOAT_OPS if t[0] == "f" else INT_OPS
    want = {op: jl.table2(BINARY[op], gx, gy) for op in ops}
    for si, n, (px, py, pz) in _launch_layouts(t, 3):
        idx = tiled(gx.size, n, 11 * si)
        x = Buf(rt1, T, n, px, gx[idx])
        y = Buf(rt1, T, n, py, gy[idx])
        z = Buf(rt1, T, n, pz)
        for op in ops:
            z.reset()
            _lib().call("dab_binary", rt1.ctx, CODE[t], op, C.c_void_p(z.ptr), C.c_void_p(x.ptr), C.c_void_p(y.ptr), n)
            got = z.get_checked()
            w = want[op][idx]
            assert same_bits(got, w), (t, BINARY[op], n, (px, py, pz), first_bad(got, w))
        for b in (x, y, z):
            b.free()


@pytest.mark.parametrize("t", TAGS)
def test_dab_binary_scalar_both_sides(dab, rt1, t):
    """Every grid value as the scalar, on the left and on the right, over the whole grid; then the size / phase sweep with three scalars."""
    g = jl.grid(t)
    T = jl.NPT[t]
    ops = FLOAT_OPS if t[0] == "f" else INT_OPS
    vpt = 16 // np.dtype(T).itemsize
    n0 = 3 * g.size + vpt + 1
    runs = [(n0, lay, list(range(g.size))) for lay in ((0, 0), (1, 1), (0, 1))]
    runs += [(n, lay, [si % g.size, (si * 5 + 3) % g.size, g.size - 1 - si % g.size]) for si, n, lay in _launch_layouts(t, 2)]
    for ri, (n, (px, pz), scalars) in enumerate(runs):
        idx = tiled(g.size, n, 3 * ri)
        x = Buf(rt1, T, n, px, g[idx])
        z = Buf(rt1, T, n, pz)
        for si in scalars:
            s = np.asarray(g[si], dtype=T)
            for left in (0, 1):
                sx = np.full(n, g[si], T)
                for op in ops:
                    z.reset()
                    _lib().call("dab_binary_scalar", rt1.ctx, CODE[t], op, C.c_void_p(z.ptr), C.c_void_p(x.ptr), C.c_void_p(s.ctypes.data),
                                left, n)
                    got = z.get_checked()
                    w = jl.vbin(BINARY[op], sx, g[idx]) if left else jl.vbin(BINARY[op], g[idx], sx)
                    w = np.asarray(w).astype(T)
                    # vbin is the vectorised model; spot-check it against the scalar methods on this run's first elements
                    if n:
                        m = min(n, 4)
                        sc = jl.table2(BINARY[op], sx[:m], g[idx][:m]) if left else jl.table2(BINARY[op], g[idx][:m], sx[:m])
                        assert same_bits(w[:m], sc.astype(T))
                    assert same_bits(got, w), (t, BINARY[op], "left" if left else "right", g[si], n, (px, pz), first_bad(got, w))
        x.free()
        z.free()


# ------------------------------------------------------------------------------------------------- NVRTC kernels
def bc_variant(shape, out_strides, out_ptr, out_size, args):
    """The host predicate of ``dab_broadcast_expr`` (dab_jit.cu): which of linear / rows / general runs.  args: (ptr, strides, elem size)
    per array argument.  The linear kernel steps ``lw`` elements per thread (``lin_width``): 8 when the output or an argument is Float16
    (the only 2-byte element type), else 4, and needs every pointer aligned to lw elements; the rows kernel always steps 4."""
    dense, acc = [], 1
    for d in range(4):
        dense.append(acc)
        acc *= shape[d]
    lw = 8 if 2 in [out_size] + [es for _, _, es in args] else 4
    linear = all(not (shape[d] > 1 and out_strides[d] != dense[d]) for d in range(4)) and out_ptr % (lw * out_size) == 0
    for ptr, st, es in args:
        if any(shape[d] > 1 and st[d] != dense[d] for d in range(4)) or ptr % (lw * es):
            linear = False
    if linear:
        return "linear"
    rows = shape[0] % 4 == 0 and out_strides[0] == 1 and out_ptr % (4 * out_size) == 0
    rows = rows and all(not (shape[d] > 1 and out_strides[d] % 4) for d in range(1, 4))
    for ptr, st, es in args:
        if not rows or st[0] == 0:
            continue
        if st[0] != 1 or ptr % (4 * es):
            rows = False
        rows = rows and all(not (shape[d] > 1 and st[d] % 4) for d in range(1, 4))
    return "rows" if rows else "general"


def run_bc(rt, src, out_tag, n0, n1, out_ld, out_off, args):
    """Run one NVRTC kernel on an (n0, n1) box.  args: list of (logical 2-D values of shape (n0, n1) or (1, n1), element offset, leading
    dimension).  Returns (values in the box, variant)."""
    L = _lib()
    odt = np.dtype(np.float16 if out_tag == "f16" else jl.NPT[out_tag])
    out = Buf(rt, odt, out_ld * (n1 - 1) + n0, out_off)
    bufs, ptrs, strides, dts, scal, spec = [], [], [], [], [], []
    for v, off, ld in args:
        v = np.asarray(v)
        a0 = v.shape[0]
        host = np.empty(ld * (n1 - 1) + a0, v.dtype)
        for j in range(n1):
            host[j * ld:j * ld + a0] = v[:, j]
        b = Buf(rt, v.dtype, host.size, off, host)
        bufs.append(b)
        st = [1 if a0 == n0 else 0, ld if n1 > 1 else 0, 0, 0]
        if a0 == n0 == 1:
            st[0] = 1
        ptrs.append(b.ptr)
        strides += st
        dts.append(CODE["f16" if v.dtype == np.float16 else jl.tag(v.ravel()[0])])
        scal.append(0)
        spec.append((b.ptr, st, v.dtype.itemsize))
    shape = [n0, n1, 1, 1]
    ostr = [1, out_ld, out_ld * n1, out_ld * n1]
    variant = bc_variant(shape, ostr, out.ptr, odt.itemsize, spec)
    k = len(args)
    L.call("dab_broadcast_expr", rt.ctx, src.encode(), CODE[out_tag], C.c_void_p(out.ptr), L.sz4(shape), L.sz4(ostr), k,
           (C.c_int32 * k)(*dts), (C.c_void_p * k)(*ptrs), (C.c_size_t * (4 * k))(*strides), (C.c_uint64 * k)(*scal))
    written = np.zeros(out.n * odt.itemsize, bool)
    for j in range(n1):
        written[j * out_ld * odt.itemsize:(j * out_ld + n0) * odt.itemsize] = True
    flat = out.get_checked(written=written)
    got = np.stack([flat[j * out_ld:j * out_ld + n0] for j in range(n1)], axis=1)
    for b in bufs + [out]:
        b.free()
    return got, variant


def bc_layouts():
    """(label, n0, n1, out_ld, out_off, [(off, ld, extruded)] per argument) -- each variant reached on purpose; the linear sizes straddle
    the 2048-element tile and its scalar tail."""
    out = []
    for n in (1, 3, 2047, 2048, 2049, 3 * 2048 + 5, 8 * 2048 + 4):
        out.append(("linear", n, 1, n, 0, [(0, n, False), (0, n, False)]))
    out.append(("rows", 64, 9, 68, 0, [(0, 68, False), (4, 72, False)]))                # 4-aligned padded strides
    out.append(("rows", 128, 5, 128, 0, [(0, 128, False), (0, 1, True)]))               # second argument extruded along dim 0
    out.append(("general", 2049, 1, 2049, 0, [(1, 2049, False), (0, 2049, False)]))     # a pointer one element off
    out.append(("general", 3 * 2048 + 5, 1, 3 * 2048 + 5, 1, [(1, 6149, False), (1, 6149, False)]))
    out.append(("general", 63, 7, 63, 0, [(0, 63, False), (0, 1, True)]))              # shape[0] % 4 != 0 with an extruded argument
    return out


def _bc_case(rt, src, out_tag, gx, gy, table, lay, rot):
    """One layout: arguments built from grid indices so the expected values come from the model table."""
    label, n0, n1, out_ld, out_off, specs = lay
    nx = gx.size
    ix = tiled(nx * gy.size, n0 * n1, rot).reshape((n0, n1), order="F")
    xi, yi = ix // gy.size, ix % gy.size
    if specs[1][2]:                                            # extruded second argument: one value per column
        yi = (np.arange(n1)[None, :] * 5 + rot) % gy.size
    args = [(gx[xi], specs[0][0], specs[0][1]), (gy[yi], specs[1][0], specs[1][1])]
    got, variant = run_bc(rt, src, out_tag, n0, n1, out_ld, out_off, args)
    assert variant == label, (label, variant)
    want = table[(xi * gy.size + np.broadcast_to(yi, xi.shape)).ravel(order="F")].reshape((n0, n1), order="F")
    return got, want


@pytest.mark.parametrize("t", TAGS)
def test_nvrtc_binary_matches_model_and_handwritten(dab, rt1, t):
    """For every op both paths serve: the NVRTC kernel (each variant) equals the model, and equals the hand-written kernel on the same
    elements bit for bit."""
    bc = _bc()
    g = jl.grid(t)
    T = jl.NPT[t]
    gx, gy = jl.pairs(g, g)
    ops = FLOAT_OPS if t[0] == "f" else INT_OPS
    fns = {ADD: lambda a, b: a + b, SUB: lambda a, b: a - b, MUL: lambda a, b: a * b, DIV: lambda a, b: a / b, REM: lambda a, b: a % b,
           BMAX: dab.jl_max, BMIN: dab.jl_min, MOD: dab.mod, IDIV: lambda a, b: a // b, AND: lambda a, b: a & b, OR: lambda a, b: a | b,
           XOR: lambda a, b: a ^ b}
    for op in ops:
        table = jl.table2(BINARY[op], gx, gy)
        src = bc.codegen(bc.convert(bc.trace(fns[op], [t, t]), t))
        for k, lay in enumerate(bc_layouts()):
            got, want = _bc_case(rt1, src, t, g, g, table, lay, 13 * k + op)
            assert same_bits(got, want.astype(T)), (t, BINARY[op], lay[0], lay[1:3], first_bad(got.ravel("F"), want.ravel("F")))
        # the hand-written kernel on the same pairs
        n = gx.size
        x, y, z = Buf(rt1, T, n, 0, gx), Buf(rt1, T, n, 0, gy), Buf(rt1, T, n)
        _lib().call("dab_binary", rt1.ctx, CODE[t], op, C.c_void_p(z.ptr), C.c_void_p(x.ptr), C.c_void_p(y.ptr), n)
        hand = z.get_checked()
        got, _ = run_bc(rt1, src, t, n, 1, n, 0, [(gx[:, None], 0, n), (gy[:, None], 0, n)])
        assert same_bits(got[:, 0], hand), (t, BINARY[op], first_bad(got[:, 0], hand))
        for b in (x, y, z):
            b.free()


@pytest.mark.parametrize("t", TAGS)
def test_nvrtc_unary_matches_handwritten(dab, rt1, t):
    bc = _bc()
    g = jl.grid(t)
    T = jl.NPT[t]
    fns = {MAP_ABS: abs, MAP_ABS2: dab.abs2, MAP_NEG: lambda a: -a, MAP_SIGN: dab.sign, MAP_FLOOR: dab.floor, MAP_CEIL: dab.ceil,
           MAP_SQRT: dab.sqrt, MAP_INV: dab.inv}
    n = 3 * 2048 + 5
    idx = tiled(g.size, n, 1)
    for c, f in fns.items():
        if t[0] == "i" and c in (MAP_SQRT, MAP_INV):
            continue
        src = bc.codegen(bc.convert(bc.trace(f, [t]), t))
        x, y = Buf(rt1, T, n, 0, g[idx]), Buf(rt1, T, n)
        _lib().call("dab_unary", rt1.ctx, CODE[t], c, C.c_void_p(y.ptr), C.c_void_p(x.ptr), n)
        hand = y.get_checked()
        for off, label in ((0, "linear"), (1, "general")):
            got, variant = run_bc(rt1, src, t, n, 1, n, off, [(g[idx][:, None], off, n)])
            assert variant == label
            assert same_bits(got[:, 0], hand), (t, UNARY[c], off, first_bad(got[:, 0], hand))
            assert same_bits(got[:, 0], jl.table1(UNARY[c], g)[idx].astype(T)), (t, UNARY[c])
        x.free()
        y.free()


def bc16_layouts():
    """(label, n0, n1, out_ld, out_off, [(off, ld, extruded)] per argument) for Float16 kernels, whose linear kernel steps 8 elements.  The
    element offsets 2 / 4 / 8 of the second argument give the same variant for a 2- and an 8-byte element: 4 or 16 bytes (general), 8 or
    32 bytes (rows: 4-aligned, but not 8-aligned as the linear kernel needs) and 16 or 64 bytes (linear)."""
    out = []
    for n in (1, 7, 8, 9, 4095, 4096, 4097, 2 * 4096 - 3, 3 * 4096 + 5, 8 * 4096 + 4):      # n % 8 != 0, both sides of 4096 k
        out.append(("linear", n, 1, n, 0, [(0, n, False), (8, n, False)]))
    out.append(("rows", 4100, 1, 4100, 0, [(0, 4100, False), (4, 4100, False)]))     # second argument 4 elements in: not 8-aligned
    out.append(("rows", 4100, 1, 4100, 4, [(0, 4100, False), (8, 4100, False)]))     # the output 4 elements in
    out.append(("rows", 64, 9, 72, 0, [(0, 72, False), (8, 80, False)]))             # padded leading dimensions
    out.append(("general", 4100, 1, 4100, 0, [(0, 4100, False), (2, 4100, False)]))  # second argument 2 elements in
    out.append(("general", 4097, 1, 4097, 1, [(1, 4097, False), (1, 4097, False)]))
    out.append(("general", 63, 7, 63, 0, [(0, 63, False), (0, 1, True)]))            # shape[0] % 4 != 0, second argument extruded
    return out


F16_BC = [  # (argument tags, output tag, traced closure, NumPy model on (Float16 x, y))
    (["f16", "f16"], "f16", lambda a, b: a * b + a, lambda a, b: a * b + a),                          # every operation rounded to Float16
    (["f16", "f64"], "f16", lambda a, y: a * y, lambda a, y: (a.astype(np.float64) * y).astype(np.float16)),   # Float64, rounded once
    (["f16", "f16"], "f32", lambda a, b: a - b, lambda a, b: (a - b).astype(np.float32)),              # Float16, widened exactly
]


@pytest.mark.parametrize("case", range(len(F16_BC)), ids=["f16-f16", "f16-f64-to-f16", "f16-to-f32"])
def test_nvrtc_float16_every_variant(dab, rt1, case):
    """The linear, rows and general broadcast kernels with Float16 operands against NumPy's Float16 arithmetic, bit for bit, on random bit
    patterns (NaN, Inf, subnormals, signed zeros).  The guard bands of every output check that the 16-byte stores of the 8-element step
    stop at n."""
    bc = _bc()
    tags, out_tag, f, model = F16_BC[case]
    src = bc.codegen(bc.convert(bc.trace(f, tags), out_tag))
    rng = np.random.default_rng(case)
    reached = set()
    for k, (label, n0, n1, out_ld, out_off, specs) in enumerate(bc16_layouts()):
        x = rng.integers(0, 1 << 16, (n0, n1)).astype(np.uint16).view(np.float16)
        if tags[1] == "f16":
            y = rng.integers(0, 1 << 16, (1 if specs[1][2] else n0, n1)).astype(np.uint16).view(np.float16)
        else:
            y = rng.standard_normal((1 if specs[1][2] else n0, n1)) * np.exp2(rng.integers(-30, 20, (1 if specs[1][2] else n0, n1)))
        got, variant = run_bc(rt1, src, out_tag, n0, n1, out_ld, out_off, [(x, specs[0][0], specs[0][1]), (y, specs[1][0], specs[1][1])])
        assert variant == label, (k, label, variant)
        reached.add(variant)
        with np.errstate(all="ignore"):
            want = np.asarray(model(x, np.broadcast_to(y, x.shape)))
        assert same_bits(got, want), (tags, out_tag, label, (n0, n1), first_bad(got.ravel("F"), want.ravel("F")))
    assert reached == {"linear", "rows", "general"}


MIXED = [(a, b) for a in ("bool", "i32", "i64", "f32", "f64") for b in ("bool", "i32", "i64", "f32", "f64")]
MIXED_OPS = {"add": lambda a, b: a + b, "mul": lambda a, b: a * b, "div": lambda a, b: a / b, "max": None, "lt": lambda a, b: a < b,
             "eq": lambda a, b: a == b, "ge": lambda a, b: a >= b}


def _ok_mixed(op, ta, tb):
    if op == "max" and "bool" in (ta, tb) and ta != tb:
        return False
    return True


@pytest.mark.parametrize("ta,tb", MIXED, ids=[f"{a}-{b}" for a, b in MIXED])
def test_nvrtc_mixed_types_every_variant(dab, rt1, ta, tb):
    """Mixed-type trees (Julia's methods, not promotion, for Bool * float, Bool + float, Int64 vs float comparisons): every variant,
    Bool / integer / float outputs."""
    bc = _bc()
    ga, gb = jl.grid(ta), jl.grid(tb)
    gx, gy = jl.pairs(ga, gb)
    for op, f in MIXED_OPS.items():
        f = f or dab.jl_max
        if not _ok_mixed(op, ta, tb):
            continue
        table = jl.table2(op, gx, gy)
        e = bc.trace(f, [ta, tb])
        assert jl.NPT[e.jt] == table.dtype.type, (op, ta, tb, e.jt, table.dtype)
        src = bc.codegen(bc.convert(e, e.jt))
        for k, lay in enumerate(bc_layouts()[2::3]):
            got, want = _bc_case(rt1, src, e.jt, ga, gb, table, lay, 7 * k)
            assert same_bits(got, want), (op, ta, tb, lay[0], lay[1:3], first_bad(got.ravel("F"), want.ravel("F")))


def test_float32_integer_powers(dab, rt1):
    """Float32 ^ Integer (an Int64 and an Int32 array of exponents, and literal exponents) against power_by_squaring in Float64."""
    bc = _bc()
    g = jl.grid("f32")
    ns = np.asarray(list(range(-40, 41)) + [64, 127, 128, 149, 150, -126, -127, -149, -150, 2 ** 31 - 1, -2 ** 31, 2 ** 62 + 1,
                                            np.iinfo(np.int64).max, np.iinfo(np.int64).min], np.int64)
    gx, gn = jl.pairs(g, ns)
    want = np.asarray([jl.pow_f32_int(x, int(n)) for x, n in zip(gx, gn)], np.float32)
    for nt in ("i64", "i32"):
        m = np.ones(gn.size, bool) if nt == "i64" else (gn >= -2 ** 31) & (gn < 2 ** 31)
        src = bc.codegen(bc.trace(lambda x, n: x ** n, ["f32", nt]))
        n = int(m.sum())
        got, _ = run_bc(rt1, src, "f32", n, 1, n, 0, [(gx[m][:, None], 0, n), (gn[m].astype(jl.NPT[nt])[:, None], 0, n)])
        bad = first_bad(got[:, 0], want[m], k=1000)
        assert not bad, (nt, f"{len(bad)} of {n} Float32 powers differ", bad[:5])
    for p in (-9, -3, -2, -1, 0, 1, 2, 3, 5, 24):
        src = bc.codegen(bc.trace(lambda x: x ** p, ["f32"]))
        n = g.size
        if src.startswith("__int_as_float"):                    # x^0 is the constant one(x)
            assert p == 0 and src == "__int_as_float((int)0x3f800000)"
            continue
        got, _ = run_bc(rt1, src, "f32", n, 1, n, 0, [(g[:, None], 0, n)])
        w = np.asarray([jl.literal_pow(x, p) for x in g], np.float32)
        assert same_bits(got[:, 0], w), (p, first_bad(got[:, 0], w))
    for p in (-2, -1, 0, 2, 3):
        src = bc.codegen(bc.trace(lambda x: x ** p, ["f64"]))
        if p == 0:
            continue
        g64 = jl.grid("f64")
        got, _ = run_bc(rt1, src, "f64", g64.size, 1, g64.size, 0, [(g64[:, None], 0, g64.size)])
        w = np.asarray([jl.literal_pow(x, p) for x in g64], np.float64)
        assert same_bits(got[:, 0], w), (p, first_bad(got[:, 0], w))


# ------------------------------------------------------------------------------------------------- the public API, 8-chunk layouts
def _dist(dab, v, shape=(37, 29)):
    n = int(np.prod(shape))
    return np.asfortranarray(v[tiled(v.size, n, 5)].reshape(shape, order="F"))


@pytest.mark.parametrize("ta,tb", [("bool", "f64"), ("f32", "bool"), ("bool", "bool"), ("i64", "f64"), ("f32", "i64"), ("i32", "f32"),
                                   ("i64", "i32"), ("bool", "i64")])
def test_public_broadcast_mixed_types(dab, rt8, ta, tb):
    """broadcast / map_ / broadcast_into on mixed-type arguments: the result's element type is the model's and so are the values."""
    ga, gb = jl.grid(ta), jl.grid(tb)
    gx, gy = jl.pairs(ga, gb)
    A, Bm = _dist(dab, gx), _dist(dab, gy)
    da, db = dab.distribute(A), dab.distribute(Bm)
    for op, f in MIXED_OPS.items():
        f = f or dab.jl_max
        if not _ok_mixed(op, ta, tb):
            continue
        want = jl.table2(op, A.ravel("F"), Bm.ravel("F")).reshape(A.shape, order="F")
        r = dab.broadcast(f, da, db)
        assert r.dtype == want.dtype, (op, ta, tb, r.dtype, want.dtype)
        got = dab.to_array(r)
        assert same_bits(got, want), (op, ta, tb, first_bad(got.ravel("F"), want.ravel("F")))
        dest = dab.distribute(np.zeros(A.shape, want.dtype))
        dab.broadcast_into(dest, f, da, db)
        assert same_bits(dab.to_array(dest), want), (op, ta, tb, "broadcast_into")
    for fn in ("abs", "abs2", "sign", "round", "trunc"):
        f = {"abs": abs, "abs2": dab.abs2, "sign": dab.sign, "round": dab.round_, "trunc": dab.trunc}[fn]
        if ta == "bool" or ta[0] == "f":
            want = jl.table1(fn, A.ravel("F")).reshape(A.shape, order="F")
            r = dab.map_(f, da)
            assert r.dtype == want.dtype and same_bits(dab.to_array(r), want), (fn, ta)


def test_public_fused_mapreduce(dab, rt8):
    """sum(x -> (x > 0) * x, d) with ±Inf and NaN entries (Julia: finite, exact for multiples of 2^-10), count of an Int64-vs-float
    comparison near 2^53, isequal of an Int64 DArray and a Float64 DArray."""
    rng = np.random.default_rng(11)
    for T in (np.float32, np.float64):
        v = (rng.integers(-64, 64, 40000) * 2.0 ** -10).astype(T)
        v[::97] = -np.inf
        v[5::101] = jl._nan("f32" if T == np.float32 else "f64", False)
        v[7::89] = jl._nan("f32" if T == np.float32 else "f64", True)
        d = dab.distribute(v)
        want = float(np.where(v > 0, v, 0).astype(np.float64).sum())
        got = dab.sum(d, lambda x: (x > 0) * x)
        assert float(got) == want, (T, got, want)
        assert float(dab.mapreduce(lambda x: x * (x > 0), "+", d)) == want
    base = 2 ** 53
    iv = np.asarray([base - 2, base - 1, base, base + 1, base + 2, base + 3, -base - 1, -base] * 300, np.int64)
    di = dab.distribute(iv)
    for c in (9007199254740992.0, 9007199254740994.0, -9007199254740992.0):
        want = sum(1 for x in iv.tolist() if x > c)
        assert dab.count(di, lambda x: x > c) == want, c
        want = sum(1 for x in iv.tolist() if x == c)
        assert dab.count(di, lambda x: x == c) == want, c
    fv = iv.astype(np.float64)                                  # rounds 2^53 + 1 to 2^53: equal in Float64, not in Julia
    assert not dab.isequal(di, dab.distribute(fv))
    exact = np.asarray([base - 2, base, base + 2, -base, 7] * 10, np.int64)
    assert dab.isequal(dab.distribute(exact), dab.distribute(exact.astype(np.float64)))
    assert not dab.to_array(dab.broadcast(lambda a, b: a == b, di, dab.distribute(fv))).all()


def test_public_narrowing_stores_in_range(dab, rt8):
    """An in-range Int64 value stored into an Int32 or Bool destination is exact."""
    v = np.asarray([0, 1, -1, 2 ** 31 - 1, -2 ** 31, 12345, -7] * 50, np.int64)
    d = dab.distribute(v)
    dest = dab.distribute(np.zeros(v.size, np.int32))
    dab.broadcast_into(dest, lambda x: x, d)
    assert np.array_equal(dab.to_array(dest), v.astype(np.int32))
    b = np.asarray([0, 1, 1, 0, 0, 1] * 50, np.int64)
    destb = dab.distribute(np.zeros(b.size, np.bool_))
    dab.broadcast_into(destb, lambda x: x, dab.distribute(b))
    assert np.array_equal(dab.to_array(destb), b.astype(bool))
