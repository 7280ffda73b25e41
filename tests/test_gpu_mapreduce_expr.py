"""The fused map-reduce kernel that NVRTC generates for a traced closure (``dab_mapreduce_expr``, dab_jit.cu), against exact results.

Every whole-array reduction that the fixed map codes do not cover runs through this kernel: ``mapreduce`` with a general closure or
with several arguments, ``dot``, ``isequal``, ``norm(x, p)``, ``count`` / ``any`` / ``all`` with a general predicate and Int128 values.
The kernel's source is built from the real tracer (``trace`` + ``codegen``) and called through the C ABI on every launch path that
``model_mr`` below tells apart, then the public calls are checked against the project's contract.  Inputs are chosen so that every
result is exact, and comparisons are bit for bit on the whole 16-byte result slot (NaN payloads excepted):

  * float sums: the mapped values lie on the 2^-10 grid and stay small, so every 8-value tile is exact in the value type and the
    fp64 carrier is exact: the result is the exact sum rounded once;
  * float products: +-1 with +-2 / +-0.5 at the edge positions, exact in any order (NaN, Inf and signed zeros too);
  * integers: any values.  The map wraps in its own type (Int32 wraps before it widens), then ``+`` / ``*`` wrap mod 2^64, and
    Int128 values wrap mod 2^128 in the map and in the reduction;
  * complex values: components on the grid (sums), +-1 / +-i / +-2 / +-0.5 (products; the sign of a zero component depends on the
    order of a complex product, in Julia as here, so zero components compare by value);
  * max / min: Julia's rules -- any NaN gives NaN, a zero result is +0.0 for max when a +0.0 is present and -0.0 for min when a
    -0.0 is present.  The reference functions are this module's own.

The deciding values sit where the kernel splits its work: element 0 and n-1, both sides of every tile boundary and of the half-tile
inside a tile, the lanes of one vector, both sides of CTA boundaries (the ones ``dab_mr_final`` reads in its 4-load loop included)
and the first element of the scalar tail.  A Float16 argument makes every thread step 8 elements wide (16-byte loads), so tiles are
4096 elements instead of 2048; the model and the edges take the width, and every launch case is run at both widths, with Float16,
Float32 and Float64 values of Float16 arguments (Float16 values: a Float32 tile, the fp64 carrier, one rounding to Float16).
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
OK, ERR_ARG, ERR_EMPTY, ERR_UNSUPPORTED = 0, 2, 3, 6
F32, F64, I32, I64, U8, I128, C64, C128, F16 = range(9)
SUM, PROD, MAX, MIN, ALL, ANY, COUNT, EXTREMA = range(8)
NP = {F32: np.dtype(np.float32), F64: np.dtype(np.float64), I32: np.dtype(np.int32), I64: np.dtype(np.int64), U8: np.dtype(np.bool_),
      C64: np.dtype(np.complex64), C128: np.dtype(np.complex128), F16: np.dtype(np.float16)}
TILE, MAX_PARTS = 2048, 16384           # 2 x 256 threads x 4 elements; dab_mr_final folds at most this many partials
TILE16 = 4096                           # with a Float16 argument a thread step takes 8 elements (16-byte loads): 2 x 256 x 8
G = 2.0 ** -10
M64, M128 = (1 << 64) - 1, (1 << 128) - 1
SERVED = ([(v, op) for v in (F32, F64, I32, I64, I128) for op in (SUM, PROD, MAX, MIN)] + [(U8, op) for op in (SUM, COUNT, ALL, ANY)] +
          [(v, op) for v in (C64, C128) for op in (SUM, PROD)])
# Float16 arguments: Float16, Float32 and Float64 values, each with + * max min (the kernel takes 8 elements per thread step)
SERVED16 = [(v, op) for v in (F16, F32, F64) for op in (SUM, PROD, MAX, MIN)]

if HOSTMEM:                                                     # the Float16 code of the host-memory emulation
    import f16_hostmem
    f16_hostmem.install()


def _lib():
    from darray_b200 import _lib as L
    return L


def _bc():
    from darray_b200 import _broadcast as bc
    return bc


# ---------------------------------------------------------------------------------------------------------- the launch model
def model_mr(n, tile=TILE):
    """``dab_mapreduce_expr``'s launch plan for n elements: tiles, tiles per CTA, grid, the last CTA's tiles, tail, final-fold case.
    ``tile`` is 512 thread steps of the lane width: TILE, or TILE16 with a Float16 argument."""
    ntiles = n // tile
    k = 2
    if -(-ntiles // k) > MAX_PARTS:
        k = -(-ntiles // MAX_PARTS)
    grid = max(1, -(-ntiles // k))
    last = ntiles - (grid - 1) * k if ntiles else 0
    final = "parts<=768" if grid <= 768 else "768<parts<=1024" if grid <= 1024 else "parts=16384" if grid == MAX_PARTS else "parts>1024"
    return dict(ntiles=ntiles, k=k, grid=grid, last_tiles=last, tail=(ntiles * tile, n), final=final)


def branches(n, tile=TILE):
    m = model_mr(n, tile)
    out = {m["final"], "k=2" if m["k"] == 2 else "k>2"}
    if m["ntiles"] == 0:
        out.add("tail only")
    elif m["tail"][0] == n:
        out.add("tiles, no tail")
    else:
        out.add("tiles and tail")
    if m["ntiles"] and m["last_tiles"] < m["k"]:
        out.add("short last CTA")
    if n % (tile // 512):
        out.add("partial vector")
    return out


REQUIRED = {"tail only", "tiles, no tail", "tiles and tail", "short last CTA", "partial vector", "k=2", "k>2", "parts<=768",
            "768<parts<=1024", "parts>1024", "parts=16384"}
SIZES = [1, 3, 4, 5, 2047, 2048, 2049, 2 * TILE, 3 * TILE + 5, 5 * TILE + 2047,
         767 * 2 * TILE + 2047,                 # 767 partials
         768 * 2 * TILE,                        # 768: the 4-load loop of dab_mr_final runs for no thread
         768 * 2 * TILE + TILE + 1,             # 769, the last CTA with one tile
         1024 * 2 * TILE,                       # 1024: every thread runs one 4-load step
         1024 * 2 * TILE + 2 * TILE + 3]        # 1025: thread 0 runs a 4-load step and a single load
I128_SIZES = [s for s in SIZES if s < 3 * TILE + 6] if HOSTMEM else SIZES   # the emulation folds Int128 values one Python integer at a time
PARTS_16384_N = 32767 * TILE + 5                # 16384 partials, the last CTA with one tile, a tail
K_GT_2_N = 32771 * TILE + 7                     # 3 tiles per CTA (the first size past 16384 partials of 2), short last CTA, a tail
BOOL_2_31_N = (1 << 31) + 2 * TILE + 3
# the same cases with 8-element thread steps
SIZES16 = [1, 3, 7, 8, 9, TILE16 - 1, TILE16, TILE16 + 1, 2 * TILE16, 3 * TILE16 + 5, 5 * TILE16 + 4095,
           767 * 2 * TILE16 + 4093, 768 * 2 * TILE16, 768 * 2 * TILE16 + TILE16 + 1, 1024 * 2 * TILE16, 1024 * 2 * TILE16 + 2 * TILE16 + 3]
PARTS_16384_N16 = 32767 * TILE16 + 5
K_GT_2_N16 = 32771 * TILE16 + 7
FULL_SIZE_RUNS16 = [(F16, SUM), (F32, MAX)]     # both sizes, in test_full_size_float16_argument


def carrier(val, op):
    """Width of the kernel's accumulator (ACC_T) in bytes."""
    if val in (I128, C64, C128):
        return 16
    return 4 if val in (F32, I32) and op in (MAX, MIN) else 8


FULL_SIZE_RUNS = {PARTS_16384_N: [(F32, SUM), (F32, MAX), (C128, SUM)], K_GT_2_N: [(F32, SUM), (F32, MAX), (I128, SUM)],
                  BOOL_2_31_N: [(U8, ALL), (U8, ANY)]}


def test_shape_table_reaches_every_branch():
    """For each carrier width (4, 8, 16 bytes), the sizes its (value type, op) pairs run on reach every case of the launch plan."""
    for width in (4, 8, 16):
        got = set()
        for val, op in SERVED:
            if carrier(val, op) == width:
                for n in (I128_SIZES if val == I128 else SIZES):
                    got |= branches(n)
        for n, runs in FULL_SIZE_RUNS.items():
            if any(carrier(v, o) == width for v, o in runs):
                got |= branches(n)
        assert REQUIRED <= got, (width, sorted(REQUIRED - got))
    assert model_mr(K_GT_2_N)["k"] == 3 and model_mr(K_GT_2_N - 7 - 3 * TILE)["k"] == 2     # the first ntiles past 2 * 16384
    assert model_mr(PARTS_16384_N)["grid"] == MAX_PARTS and model_mr(1)["grid"] == 1
    got = set()                                                  # 8-element steps: SIZES16 and the full-size Float16-argument runs
    for n in SIZES16 + [PARTS_16384_N16, K_GT_2_N16]:
        got |= branches(n, TILE16)
    assert REQUIRED <= got, ("width 8", sorted(REQUIRED - got))
    assert model_mr(K_GT_2_N16, TILE16)["k"] == 3 and model_mr(PARTS_16384_N16, TILE16)["grid"] == MAX_PARTS


def edge_positions(n, tile=TILE):
    """Where the kernel changes what it does, for n elements and a tile of ``tile`` elements (lane width tile // 512)."""
    m = model_mr(n, tile)
    k, grid, nt = m["k"], m["grid"], m["ntiles"]
    w, half = tile // 512, tile // 2
    pos = {0, 1, 2, 3, w - 1, w, n - 2, n - 1}
    for t in {0, 1, nt // 2, nt - 2, nt - 1}:
        if 0 <= t < nt:
            b = t * tile
            pos |= {b, b + 1, b + half - 1, b + half, b + half + 1, b + tile - 1}
    lane = w * 37                                    # the lanes of thread 37's vectors, in both halves of the first and last tile
    for t in {0, max(nt - 1, 0)}:
        pos |= {t * tile + h + lane + j for h in (0, half) for j in range(w)}
    for c in {1, 2, grid // 2, grid - 1, 256, 511, 512, 767, 768, 769, 1023, 1024}:
        if 0 < c < grid:
            pos |= {c * k * tile - 1, c * k * tile}
    tail = nt * tile
    pos |= {tail - 1, tail, tail + 1}
    return np.asarray(sorted(p for p in pos if 0 <= p < n), dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------- references
def wrap128(v):
    v &= M128
    return v - (1 << 128) if v >> 127 else v


def jl_extreme(m, is_max):
    """Julia's maximum / minimum of a float array: NaN wins, then the extreme value, +0.0 > -0.0."""
    m = np.asarray(m)
    if np.isnan(m).any():
        return m.dtype.type(np.nan)
    r = m.max() if is_max else m.min()
    if r == 0:
        want_neg = not is_max
        has = ((m == 0) & (np.signbit(m) == want_neg)).any()
        r = m.dtype.type(-0.0 if want_neg == has else 0.0)
    return r


def spec16(val, op):
    """(Float16, traced closure, its NumPy twin) with a Float16 argument: Float16 values (every operation rounds to Float16, as NumPy's
    float16 does), Float32 values (a Float32 constant promotes) and Float64 values (a Python float is a Float64 literal)."""
    if val in (F16, F32):
        T = NP[val].type
        f = {SUM: lambda x: x * T(2) - T(2.0 ** -7), PROD: lambda x: (x + x) * T(0.5)}.get(op, lambda x: -(x * T(2)))
        return NP[F16], f, f
    f, twin = {SUM: (lambda x: x * 2.0 - 2.0 ** -7, lambda x: x.astype(np.float64) * 2.0 - 2.0 ** -7),
               PROD: (lambda x: (x + x) * 0.5, lambda x: (x + x).astype(np.float64) * 0.5)}.get(
        op, (lambda x: -(x * 2.0), lambda x: -(x.astype(np.float64) * 2.0)))
    return NP[F16], f, twin


def spec(val, op, arg16=False):
    """(input element type, traced closure, its NumPy twin).  None of the closures is one of the fixed map codes."""
    bc = _bc()
    if arg16:
        return spec16(val, op)
    if val in (F32, F64):
        T = NP[val].type
        if op == SUM:
            f = lambda x: x * T(2) - T(2.0 ** -7)
        elif op == PROD:
            f = lambda x: (x + x) * T(0.5)
        else:
            f = lambda x: -(x + x)
        return NP[val], f, f
    if val in (I32, I64):
        T = NP[val].type
        f = lambda x: x * T(3) - T(8)                     # odd x stays odd: products never reach 0 mod 2^64
        return NP[val], f, f
    if val == U8:
        return NP[U8], lambda b: (b | False) & True, lambda b: b
    if val == I128:
        import darray_b200 as dab
        return np.dtype(np.int64), lambda x: dab.Int128(x) * dab.Int128(x) * 3 + 1, lambda x: 3 * x * x + 1
    if op == SUM:                                          # z*2 - 1 with Julia's Complex-Real methods: (2re - 1, 2im)
        def twin(z):
            R = NP[val].type(0).real.dtype.type
            out = np.empty(np.shape(z), dtype=NP[val])
            out.real, out.imag = z.real * R(2) - R(1), z.imag * R(2)
            return out
        return NP[val], lambda z: z * 2 - 1, twin
    return NP[val], lambda z: bc.conj(z), np.conj


def mapped(val, twin, x):
    """The NumPy twin on an input array; Int128 values as Python integers when they may not fit 64 bits."""
    with np.errstate(all="ignore"):
        if val == I128:
            if x.size and np.abs(x.astype(np.float64)).max() < 2 ** 20:
                return twin(x.astype(np.int64))           # small: exact in Int64
            return [wrap128(twin(int(v))) for v in x.tolist()]
        if val in (C64, C128):
            return twin(x).astype(NP[val])
        return np.asarray(twin(x)).astype(NP[val])


def acc_of(val, op, m):
    """The exact reduction of mapped values m, in a form that ``acc_join`` can combine: Python ints (mod 2^64 / 2^128), fp64 sums and
    products, complex128, the extreme in the value type, or the number of trues."""
    if val == U8:
        return int(np.count_nonzero(m))
    if val == I128:
        if isinstance(m, np.ndarray):
            if op == SUM:
                return int(m.sum(dtype=np.int64))
            if op == PROD:
                r = 1
                for v, c in zip(*np.unique(m, return_counts=True)):
                    r = r * pow(int(v), int(c), 1 << 128) & M128
                return wrap128(r)
            m = [int(v) for v in (m.max(), m.min())] if m.size else []
        r = {SUM: 0, PROD: 1}.get(op)
        for v in m:
            r = v if r is None else (wrap128(r + v) if op == SUM else wrap128(r * v) if op == PROD else max(r, v) if op == MAX else min(r, v))
        return r
    m = np.asarray(m)
    if m.size == 0:
        return None
    with np.errstate(all="ignore"):
        if val in (I32, I64):
            w = m.astype(np.int64)
            if op in (SUM, PROD):
                return int(w.sum(dtype=np.int64) if op == SUM else w.prod(dtype=np.int64)) & M64
            return m.max() if op == MAX else m.min()
        if val in (C64, C128):
            w = m.astype(np.complex128)
            if op == SUM:
                return complex(w.real.sum(), w.imag.sum())
            return complex(np.prod(w))
        if op in (SUM, PROD):
            w = m.astype(np.float64)
            return float(w.sum() if op == SUM else w.prod())
        return jl_extreme(m, op == MAX)


def acc_join(val, op, a, b):
    if a is None:
        return b
    if b is None:
        return a
    if val == U8:
        return a + b
    if val == I128:
        return acc_of(val, op, [a, b])
    if val in (I32, I64):
        if op == SUM:
            return (a + b) & M64
        if op == PROD:
            return (a * b) & M64
        return max(a, b) if op == MAX else min(a, b)
    if op == SUM:
        return a + b
    if op == PROD:
        return a * b
    return jl_extreme(np.asarray([a, b], dtype=NP[val]), op == MAX)


def want_slot(val, op, acc, n):
    """The 16-byte result slot and its float fields (offset, dtype): word 0 the result in OUT_T, word 1 the carrier; a 16-byte
    carrier fills the slot."""
    w = bytearray(16)
    fl = []
    i64 = lambda v: int(v & M64).to_bytes(8, "little")
    if val == I128:
        w[:] = (acc & M128).to_bytes(16, "little")
    elif val in (C64, C128):
        R = np.float32 if val == C64 else np.float64
        w[:2 * np.dtype(R).itemsize] = np.asarray([acc.real, acc.imag], dtype=np.float64).astype(R).tobytes()
        fl = [(0, R), (np.dtype(R).itemsize, R)]
    elif val == F16:                                       # Float32 carrier for max / min
        w[:2] = np.float16(acc).tobytes()
        w[8:16 if op in (SUM, PROD) else 12] = (np.float64 if op in (SUM, PROD) else np.float32)(acc).tobytes()
        fl = [(0, np.float16), (8, np.float64 if op in (SUM, PROD) else np.float32)]
    elif val in (F32, F64):
        T = NP[val].type
        if op in (SUM, PROD):
            w[:NP[val].itemsize] = T(acc).tobytes()
            w[8:] = np.float64(acc).tobytes()
            fl = [(0, T), (8, np.float64)]
        else:
            w[:NP[val].itemsize] = w[8:8 + NP[val].itemsize] = T(acc).tobytes()
            fl = [(0, T), (8, T)]
    elif val in (I32, I64):
        if op in (SUM, PROD):
            w[:8] = w[8:] = i64(acc)
        else:
            w[:NP[val].itemsize] = w[8:8 + NP[val].itemsize] = NP[val].type(acc).tobytes()
    else:
        res = {SUM: acc, COUNT: acc, ALL: int(acc == n), ANY: int(acc != 0)}[op]
        w[:8], w[8:] = i64(res), i64(acc)
    return bytes(w), fl


def slot_matches(got, want, fl, zero_sign_free=False):
    g, w = bytearray(got), bytearray(want)
    for off, T in fl:
        sz = np.dtype(T).itemsize
        a, b = np.frombuffer(bytes(g[off:off + sz]), T)[0], np.frombuffer(bytes(w[off:off + sz]), T)[0]
        if np.isnan(b) or (zero_sign_free and b == 0):
            if not (np.isnan(a) if np.isnan(b) else a == 0):
                return False
            g[off:off + sz] = w[off:off + sz] = bytes(sz)
    return g == w


def show(slot):
    return bytes(slot).hex(" ", 8)


# ---------------------------------------------------------------------------------------------------------- device helpers
class Dev:
    """A device copy of a host array, ``off`` elements past a 256-byte aligned allocation."""

    def __init__(self, rt, host, off=0):
        host = np.ascontiguousarray(host)
        self.rt, self.dt, self.n = rt, host.dtype, host.size
        self.base = rt.alloc((self.n + off + 4) * host.itemsize)
        self.ptr = self.base + off * host.itemsize
        self.put(0, host)

    def put(self, i, host):
        host = np.ascontiguousarray(host, dtype=self.dt)
        if host.size:
            _lib().call("dab_h2d", self.rt.ctx, C.c_void_p(self.ptr + i * self.dt.itemsize), C.c_void_p(host.ctypes.data), host.nbytes)
        self.rt.sync()

    def free(self):
        self.rt.free(self.base)


class Slot:
    FILL = bytes([0xA5]) * 16

    def __init__(self, rt):
        self.rt, self.dev = rt, Dev(rt, np.zeros(16, dtype=np.uint8))
        self.ptr = self.dev.ptr

    def clear(self):
        self.dev.put(0, np.frombuffer(self.FILL, dtype=np.uint8))

    def get(self):
        out = np.empty(16, dtype=np.uint8)
        _lib().call("dab_d2h", self.rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(self.ptr), 16)
        self.rt.sync()
        return out.tobytes()

    def free(self):
        self.dev.free()


def mr_status(rt, src, val, op, n, dts, ptrs, scal, out_ptr, nargs=None):
    """``dab_mapreduce_expr`` through the C ABI; returns the status instead of raising."""
    k = len(dts)
    m = max(k, 1)
    st = _lib().lib().dab_mapreduce_expr(rt.ctx, src, val, op, n, k if nargs is None else nargs, (C.c_int32 * m)(*dts),
                                         (C.c_void_p * m)(*ptrs), (C.c_uint64 * m)(*scal), C.c_void_p(out_ptr))
    rt.sync()
    return st


def source(f, tags):
    bc = _bc()
    e = bc.trace(f, tags)
    return bc.codegen(e).encode(), e.jt


def code_of(dt):
    return {np.dtype(v): k for k, v in NP.items()}[np.dtype(dt)]


def val_code(jt):
    return {"f32": F32, "f64": F64, "i32": I32, "i64": I64, "bool": U8, "i128": I128, "c64": C64, "c128": C128, "f16": F16}[jt]


# ---------------------------------------------------------------------------------------------------------- input builders
def nan_values(T, count):
    """NaNs of both signs, quiet and signalling, with payloads."""
    U = {2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(T).itemsize]
    bits, nmant = 8 * np.dtype(T).itemsize, np.finfo(T).nmant
    quiet = 1 << (nmant - 1)
    expo = ((1 << (bits - 1)) - 1) ^ ((1 << nmant) - 1)
    out = []
    for j in range(count):
        payload = ((0x2A5 + 7 * j) & (quiet - 1)) | (quiet if j % 4 < 2 else 0)
        out.append(np.asarray([expo | payload | ((1 << (bits - 1)) if j % 2 else 0)], dtype=U).view(T)[0])
    return out


def base_input(val, op, n, rng, arg16=False):
    """Input values whose mapped values never decide a max / min / all / any on their own and keep every sum and product exact."""
    T = spec(val, op, arg16)[0]
    if val in (F32, F64, F16):
        if op == SUM:
            return (rng.integers(-8, 9, n) * G).astype(T)
        if op == PROD:
            return np.where(rng.random(n) < 0.5, -1.0, 1.0).astype(T)
        s = 1.0 if op == MAX else -1.0                     # mapped -(2x): < 0 for max, > 0 for min
        return (s * rng.integers(1, 9, n) * G).astype(T)
    if val in (I32, I64):
        if op == PROD:
            return np.where(rng.random(n) < 0.5, -1, 1).astype(T)
        if op in (MAX, MIN):
            return rng.integers(-1000, 1000, n).astype(T)
        info = np.iinfo(T)
        return rng.integers(info.min, info.max, n, dtype=np.int64, endpoint=True).astype(T)
    if val == U8:
        if op in (SUM, COUNT):
            return rng.random(n) < 0.5
        return np.full(n, op == ALL, dtype=np.bool_)
    if val == I128:
        if op == PROD:
            return np.where(rng.random(n) < 0.5, -2, 2).astype(np.int64)    # 3x^2 + 1 = 13: odd factors stay nonzero mod 2^128
        return rng.integers(-30000, 30000, n).astype(np.int64)
    R = np.float32 if val == C64 else np.float64
    if op == SUM:
        return (rng.integers(-8, 9, n) * G + 1j * rng.integers(-8, 9, n) * G).astype(T)
    units = np.asarray([1, -1, 1j, -1j], dtype=T)
    return units[rng.integers(0, 4, n)]


def edge_cases(val, op, x_e, rng):
    """Full sets of values for the edge positions, one per launch.  Sums, products and counts take all edges at once, with finite,
    extreme and special values; max / min / all / any put the deciding value at one position per launch."""
    T = x_e.dtype.type
    k = len(x_e)
    cases = []
    if val in (F32, F64, F16):
        if op in (SUM, PROD):
            fin = np.asarray([16, -15, 14, -13, 12, -11] if op == SUM else [2, -0.5, -2, 0.5], dtype=np.float64)
            fin = (fin * (G if op == SUM else 1.0))[np.arange(k) % len(fin)].astype(T)
            cases.append(fin)
            j = int(rng.integers(k))
            for special in (nan_values(T, 4)[int(rng.integers(4))], T(np.inf)):
                c = fin.copy()
                c[j] = special
                cases.append(c)
            c = fin.copy()
            c[j], c[(j + k // 2) % k] = T(np.inf), T(-np.inf)
            cases.append(c)
            z = fin.copy()
            z[::2] = np.where(np.arange(0, k, 2) % 4 == 0, T(0.0), T(-0.0))
            cases.append(z)
            return cases
        s = 1.0 if op == MAX else -1.0
        nans = nan_values(T, 8)
        for j in run_positions(k):
            c = x_e.copy()
            c[j] = T(-s * 4 * G) if j % 2 else T(-s * np.inf)          # the mapped extreme: +-8 2^-10 or +-Inf
            cases.append(c)
            c = x_e.copy()
            c[j] = nans[j % 8]
            cases.append(c)
            c = x_e.copy()                                       # the winning zero at j, the losing one at another position
            c[j], c[(j + k // 2) % k] = (T(-0.0), T(0.0)) if op == MAX else (T(0.0), T(-0.0))
            cases.append(c)
            c = x_e.copy()                                       # the losing zero alone
            c[j] = T(0.0) if op == MAX else T(-0.0)
            cases.append(c)
        return cases
    if val in (I32, I64):
        info = np.iinfo(T)
        big = np.asarray([info.max, info.min, info.max - 1, info.min + 1, 1 << 30, -(1 << 30)] if op != PROD else
                         [info.max, info.min + 1, 46341 if T == np.int32 else (1 << 33) + 1, -65535, 65537, 3], dtype=T)
        if op in (SUM, PROD):
            return [big[np.arange(k) % len(big)], big[(np.arange(k) + 3) % len(big)]]
        with np.errstate(all="ignore"):
            win = big[np.argmax(big * T(3) - T(8)) if op == MAX else np.argmin(big * T(3) - T(8))]
        for j in run_positions(k):
            for v in (win, big[j % len(big)]):
                c = x_e.copy()
                c[j] = v
                cases.append(c)
        return cases
    if val == U8:
        if op in (SUM, COUNT):
            return [np.arange(k) % 2 == 0, np.arange(k) % 3 != 1]
        cases.append(x_e.copy())
        for j in run_positions(k):
            c = x_e.copy()
            c[j] = not c[j]
            cases.append(c)
        return cases
    if val == I128:
        big = np.asarray([np.iinfo(np.int64).max, np.iinfo(np.int64).min, (1 << 62) + 3, -(1 << 40) - 1, 1 << 63 - 1, 5], dtype=np.int64)
        if op == PROD:
            big = np.asarray([(1 << 62) - 2, -(1 << 62), 1 << 40, -4, 6, -(1 << 33)], dtype=np.int64)   # even: odd factors
        if op in (SUM, PROD):
            return [big[np.arange(k) % len(big)], big[(np.arange(k) + 2) % len(big)]]
        for j in run_positions(k):
            c = x_e.copy()
            c[j] = big[j % len(big)]
            cases.append(c)
        return cases
    R = np.float32 if val == C64 else np.float64
    if op == SUM:
        fin = ((np.arange(k) % 7 - 3) * 5 * G + 1j * (np.arange(k) % 5 - 2) * 9 * G).astype(T)
        cases.append(fin)
        j = int(rng.integers(k))
        c = fin.copy()
        c[j] = complex(R(np.nan), 1.0)
        cases.append(c)
        c = fin.copy()
        c[j], c[(j + k // 2) % k] = complex(np.inf, 2.0), complex(1.0, -np.inf)
        cases.append(c)
        return cases
    vals = np.asarray([2, 0.5j, -2j, -0.5, 1j, -1], dtype=T)
    return [vals[np.arange(k) % len(vals)], vals[(np.arange(k) + 1) % len(vals)]]


def run_positions(k):
    """The edge positions that take the deciding value, one per launch (a sample of them on the host-memory emulation)."""
    return range(k) if not HOSTMEM else range(0, k, max(1, k // 3))


def run_abi_cases(rt, slot, val, op, n, rng, arg16=False):
    """Upload one input of n elements, then run every edge case of (val, op) on it; returns a list of failures.  arg16: the input is
    Float16 (spec16), and the edges are those of 8-element thread steps."""
    T, f, twin = spec(val, op, arg16)
    src, jt = source(f, [_bc().tag_of(T)])
    assert val_code(jt) == val, (jt, val)
    x = base_input(val, op, n, rng, arg16)
    tile = TILE16 if arg16 else TILE
    E = edge_positions(n, tile)
    rest = np.ones(n, dtype=bool)
    rest[E] = False
    acc_rest = acc_of(val, op, mapped(val, twin, x[rest]))
    xd = Dev(rt, x)
    cur = x[E].copy()
    bad = []
    try:
        for case in edge_cases(val, op, cur.copy(), rng):
            case = np.asarray(case, dtype=T)
            diff = (case.view(np.uint8).reshape(len(E), -1) != cur.view(np.uint8).reshape(len(E), -1)).any(axis=1)
            for j in np.flatnonzero(diff):
                xd.put(int(E[j]), case[j:j + 1])
            cur = case
            acc = acc_join(val, op, acc_rest, acc_of(val, op, mapped(val, twin, case)))
            want, fl = want_slot(val, op, acc, n)
            slot.clear()
            n0 = rt.launches()
            st = mr_status(rt, src, val, op, n, [code_of(T)], [xd.ptr], [0], slot.ptr)
            got = slot.get()
            if st != OK:
                bad.append(f"n={n}: status {st}")
            elif not HOSTMEM and rt.launches() - n0 != 2:
                bad.append(f"n={n}: {rt.launches() - n0} launches")
            elif not slot_matches(got, want, fl, zero_sign_free=val in (C64, C128) and op == PROD):
                changed = E[np.flatnonzero(case.view(np.uint8).reshape(len(E), -1).any(axis=1))][:4]
                bad.append(f"n={n} model={model_mr(n, tile)} edges~{changed.tolist()}: got [{show(got)}] want [{show(want)}]")
    finally:
        xd.free()
    return bad


# ---------------------------------------------------------------------------------------------------------- (1) every served pair, every size
def _sid(p):
    return {F32: "f32", F64: "f64", I32: "i32", I64: "i64", U8: "bool", I128: "i128", C64: "c64", C128: "c128", F16: "f16"}[p[0]] + "-" + \
        {SUM: "sum", PROD: "prod", MAX: "max", MIN: "min", ALL: "all", ANY: "any", COUNT: "count"}[p[1]]


@pytest.mark.parametrize("pair", SERVED, ids=_sid)
def test_abi_exact_on_every_launch_path(dab, rt1, pair):
    val, op = pair
    slot = Slot(rt1)
    bad = []
    try:
        for si, n in enumerate(I128_SIZES if val == I128 else SIZES):
            bad += run_abi_cases(rt1, slot, val, op, n, np.random.default_rng(1000 * si + 10 * val + op))
    finally:
        slot.free()
    assert not bad, f"{len(bad)} failures: " + "; ".join(bad[:6])


SIZES16_RUN = SIZES16 if not HOSTMEM else [s for s in SIZES16 if s < 6 * TILE16]   # the emulation evaluates Float16 trees slowly


@pytest.mark.parametrize("pair", SERVED16, ids=lambda p: "f16arg-" + _sid(p))
def test_abi_exact_float16_argument_every_launch_path(dab, rt1, pair):
    """A Float16 argument makes every thread step 8 elements wide (tiles of 4096): every launch case at that width, for Float16,
    Float32 and Float64 values."""
    val, op = pair
    slot = Slot(rt1)
    bad = []
    try:
        for si, n in enumerate(SIZES16_RUN):
            bad += run_abi_cases(rt1, slot, val, op, n, np.random.default_rng(1000 * si + 10 * val + op), arg16=True)
    finally:
        slot.free()
    assert not bad, f"{len(bad)} failures: " + "; ".join(bad[:6])


@pytest.mark.parametrize("n", [9, TILE16 + 1, 3 * TILE16 + 5, 40 * TILE16 + 1001])
def test_argument_tables_float16_mixed_widths(dab, rt1, n):
    """Float16 arrays with Float32, Float64 and Int32 arrays and a Float16 scalar (the 8-element step reads 16, 32 and 64 bytes per
    argument), and pointers 8 or 16 elements past their allocation."""
    rng = np.random.default_rng(n)
    h = _grid(rng, n).astype(np.float16)
    f32 = _grid(rng, n).astype(np.float32)
    f64 = _grid(rng, n).astype(np.float64)
    i32 = rng.integers(-1000, 1000, n).astype(np.int32)
    f16 = np.float16
    cases = [
        (lambda a, x: a * x, [h, f32], SUM, lambda: h.astype(np.float32) * f32),                       # Float32 values
        (lambda a, x: a * x, [h, f32], MAX, lambda: h.astype(np.float32) * f32),
        (lambda a, y: a * y + a, [h, f64], SUM, lambda: h.astype(np.float64) * f64 + h),                 # Float64 values
        (lambda a, i: a * i, [h, i32], SUM, lambda: h * i32.astype(f16)),                                # Float16 * Int32: Float16, rounded
        (lambda a, i: a * i, [h, i32], MIN, lambda: h * i32.astype(f16)),
        (lambda a, s: a * s, [h, (f16(1.5), f16)], SUM, lambda: h * f16(1.5)),                            # a Float16 scalar
        (lambda a, x, y, i: (a * x + y) * i, [h, f32, f64, i32], SUM, lambda: (h.astype(np.float32) * f32 + f64) * i32),
    ]
    slot = Slot(rt1)
    bad = []
    try:
        for ci, (f, args, op, ref) in enumerate(cases):
            with np.errstate(all="ignore"):
                m = np.asarray(ref())
            for offs in ([0] * len(args), [8 * (k % 3) for k in range(len(args))]):
                st, got, want = _arg_table_case(rt1, slot, f, args, op, m, offs)
                if st != OK:
                    bad.append(f"case {ci} offs {offs}: status {st}")
                elif not slot_matches(got, *want):
                    bad.append(f"case {ci} offs {offs}: got [{show(got)}] want [{show(want[0])}]")
    finally:
        slot.free()
    assert not bad, "; ".join(bad)


def test_float16_alignment_refusals(dab, rt1):
    """With a Float16 argument every array argument must be aligned to 8 of its elements: a Float16 array 1..7 elements in, a Float32 array
    4 elements (16 bytes) in and a Float64 array 4 elements (32 bytes) in are refused without a launch; 8 elements in is served exactly."""
    rng = np.random.default_rng(17)
    n = 2 * TILE16 + 5
    h = _grid(rng, n).astype(np.float16)
    x32 = _grid(rng, n).astype(np.float32)
    x64 = _grid(rng, n).astype(np.float64)
    slot = Slot(rt1)
    bufs = {dt: Dev(rt1, np.zeros(n + 16, NP[dt])) for dt in (F16, F32, F64)}

    def place(dt, a, e):                                                   # a, e elements past a 256-byte aligned allocation
        bufs[dt].put(e, a)
        return bufs[dt].ptr + e * NP[dt].itemsize

    try:
        src1, _ = source(lambda a: a * np.float16(2), ["f16"])
        src2, _ = source(lambda a, x: a * x, ["f16", "f32"])
        src3, _ = source(lambda a, y: a * y, ["f16", "f64"])
        refusals = [(src1, F16, [F16], [place(F16, h, e)]) for e in range(1, 8)]
        refusals += [(src2, F32, [F16, F32], [place(F16, h, 0), place(F32, x32, 4)]), (src3, F64, [F16, F64], [place(F16, h, 0), place(F64, x64, 4)])]
        for src, val, dts, ptrs in refusals:
            slot.clear()
            n0 = rt1.launches()
            assert mr_status(rt1, src, val, SUM, n, dts, ptrs, [0] * len(dts), slot.ptr) == ERR_UNSUPPORTED, (val, ptrs)
            assert rt1.launches() == n0 and slot.get() == Slot.FILL, (val, ptrs)
        served = [(src1, F16, [F16], [h], h * np.float16(2)), (src2, F32, [F16, F32], [h, x32], h.astype(np.float32) * x32),
                  (src3, F64, [F16, F64], [h, x64], h.astype(np.float64) * x64)]
        for src, val, dts, arrs, m in served:
            ptrs = [place(dt, a, 8) for dt, a in zip(dts, arrs)]           # 8 elements in: aligned, served
            slot.clear()
            assert mr_status(rt1, src, val, SUM, n, dts, ptrs, [0] * len(dts), slot.ptr) == OK, val
            want, fl = want_slot(val, SUM, acc_of(val, SUM, m), n)
            got = slot.get()
            assert slot_matches(got, want, fl), (val, show(got), show(want))
    finally:
        slot.free()
        for d in bufs.values():
            d.free()


# ---------------------------------------------------------------------------------------------------------- (2) argument tables
def _upload_args(rt, arrays, offs):
    return [Dev(rt, a, o) if isinstance(a, np.ndarray) else None for a, o in zip(arrays, offs)]


def _scalar_bits(v, dt):
    return int.from_bytes(np.asarray([v], dtype=dt).tobytes().ljust(8, b"\0"), "little")


def _arg_table_case(rt, slot, f, args, op, ref, offs=None):
    """args: NumPy arrays (device arguments) or (value, dtype) scalars; ref: the exact mapped values, reduced here exactly."""
    bc = _bc()
    tags = [bc.tag_of(a.dtype) if isinstance(a, np.ndarray) else bc.tag_of(a[1]) for a in args]
    e = bc.trace(f, tags)
    larg = [bc.LocalArg(None, a[0], bc.tag_of(a[1])) if not isinstance(a, np.ndarray) else bc.LocalArg(object(), None, t)
            for a, t in zip(args, tags)]
    e2, larg2 = bc.split_c128_scalars(e, larg)
    src = bc.codegen(e2).encode()
    offs = offs or [0] * len(args)
    devs = _upload_args(rt, args, offs)
    n = next(a.size for a in args if isinstance(a, np.ndarray))
    try:
        dts = [code_of(bc._NPT[la.tag]) for la in larg2]
        ptrs = [d.ptr if d is not None else None for d in devs] + [None] * (len(larg2) - len(devs))
        scal = [0 if isinstance(a, np.ndarray) else _scalar_bits(a[0], a[1]) for a in args]
        scal += [_scalar_bits(la.scalar, np.float64) for la in larg2[len(args):]]
        for k, la in enumerate(larg2[:len(args)]):
            if la.arr is None:
                scal[k] = _scalar_bits(la.scalar, bc._NPT[la.tag])
        val = val_code(e.jt)
        slot.clear()
        st = mr_status(rt, src, val, op, n, dts, ptrs, scal, slot.ptr)
        if st != OK:
            return st, None, None
        acc = acc_of(val, op, ref)
        want, fl = want_slot(val, op, acc, n)
        got = slot.get()
        return st, got, (want, fl)
    finally:
        for d in devs:
            if d is not None:
                d.free()


def _grid(rng, n, lo=-8, hi=8):
    return rng.integers(lo, hi + 1, n) * G


@pytest.mark.parametrize("n", [5, 2049, 3 * TILE + 5, 40 * TILE + 1001])
def test_argument_tables_mixed_widths_and_scalars(dab, rt1, n):
    """2 to 8 arguments: Bool, Int32, Int64, Float32, Float64 and complex arrays, scalars first / in the middle / last, a ComplexF64 scalar
    (two Float64 slots), and array pointers 4 or 8 elements past their allocation."""
    rng = np.random.default_rng(n)
    b = rng.random(n) < 0.5
    i32 = rng.integers(-1000, 1000, n).astype(np.int32)
    i64 = rng.integers(-1000, 1000, n).astype(np.int64)
    f32 = _grid(rng, n).astype(np.float32)
    f64 = _grid(rng, n).astype(np.float64)
    z64 = (_grid(rng, n) + 1j * _grid(rng, n)).astype(np.complex64)
    u = np.asarray([1, -1, 1j, -1j], dtype=np.complex64)[rng.integers(0, 4, n)]
    ones, zi, zl = np.ones(n, dtype=np.float32), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int64)
    slot = Slot(rt1)
    cases = [
        # scalar first: Float32 * Int64 -> Float32
        (lambda s, x: x * s + 1, [(3, np.int64), f32], SUM, lambda: f32.astype(np.float64) * 3 + 1),
        # scalar in the middle, Bool array last: Int32 * Float64 + Bool -> Float64
        (lambda i, s, c: i * s + c, [i32, (0.25, np.float64), b], SUM, lambda: i32 * 0.25 + b),
        (lambda i, s, c: i * s + c, [i32, (0.25, np.float64), b], MAX, lambda: i32 * 0.25 + b),
        # three integer widths and a scalar last: Int64 values that wrap
        (lambda i, l, c, s: (i + l) * s + c, [i32, i64, b, ((1 << 60) + 1, np.int64)], SUM,
         lambda: (i32.astype(np.int64) + i64) * ((1 << 60) + 1) + b),
        (lambda x, y, c: (x > y) | c, [f32, f64, b], COUNT, lambda: (f32 > f64) | b),
        # 7 arguments and a ComplexF64 scalar last: 8 slots
        (lambda c, i, l, x, y, z, w: (z * x + y) + (i + l) * c + w,
         [b, i32, i64, f32, f64, z64, (complex(0.5, -0.25), np.complex128)], SUM,
         lambda: (z64.astype(np.complex128) * f32 + f64) + (i32.astype(np.int64) + i64) * b + complex(0.5, -0.25)),
        # a ComplexF64 scalar first, then six arrays: a product of units
        (lambda w, x, y, z, i, l, c: w * c + z * x - y + i - l, [(complex(0.0, 0.0), np.complex128), ones, ones.astype(np.float64) * 0, u, zi, zl, b],
         PROD, lambda: u.astype(np.complex128)),
    ]
    bad = []
    try:
        for ci, (f, args, op, ref) in enumerate(cases):
            with np.errstate(all="ignore"):
                m = np.asarray(ref())
            for offs in ([0] * len(args), [4 * (k % 3) for k in range(len(args))]):
                st, got, want = _arg_table_case(rt1, slot, f, args, op, m, offs)
                if st != OK:
                    bad.append(f"case {ci} offs {offs}: status {st}")
                elif not slot_matches(got, *want, zero_sign_free=op == PROD):
                    bad.append(f"case {ci} offs {offs}: got [{show(got)}] want [{show(want[0])}]")
    finally:
        slot.free()
    assert not bad, "; ".join(bad)


def test_same_source_other_types_and_kinds(dab, rt1):
    """One source string, compiled for different argument types, value types and array / scalar kinds in one process: each call gets its
    own kernel and its own correct result."""
    rng = np.random.default_rng(5)
    n = 3 * TILE + 7
    slot = Slot(rt1)
    f = lambda x, y: x * y + x
    runs = []
    for tags in (["f32", "f32"], ["i64", "i64"], ["f64", "f64"], ["i32", "i32"]):
        src, jt = source(f, tags)
        runs.append((tags, src, jt))
    assert len({r[1] for r in runs}) == 1, [r[1] for r in runs]
    try:
        for rep in range(2):
            for tags, _, jt in runs:
                T = np.dtype(_bc()._NPT[tags[0]])
                if T.kind == "f":
                    x, y = _grid(rng, n).astype(T), _grid(rng, n).astype(T)
                else:
                    x, y = rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(T), rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(T)
                for y_arg in (y, (y[0], T)):
                    yv = y if isinstance(y_arg, np.ndarray) else np.full(n, y[0], dtype=T)
                    with np.errstate(all="ignore"):
                        m = (x * yv + x).astype(T)
                    st, got, want = _arg_table_case(rt1, slot, f, [x, y_arg], SUM, m)
                    assert st == OK and slot_matches(got, *want), (rep, tags, isinstance(y_arg, np.ndarray), show(got), show(want[0]))
    finally:
        slot.free()


# ---------------------------------------------------------------------------------------------------------- (3) refusals
def test_refusals_launch_nothing(dab, rt1):
    """Every refusal returns its status, launches nothing and leaves the next valid call correct."""
    rng = np.random.default_rng(9)
    n = 2 * TILE + 5
    x = _grid(rng, n).astype(np.float32)
    xd = Dev(rt1, x, 0)
    big = Dev(rt1, np.zeros(n + 16, dtype=np.float32), 0)
    big.put(0, np.concatenate([np.zeros(8, np.float32), x]))                     # x again, 8 elements into an allocation
    slot = Slot(rt1)
    src, _ = source(lambda v: v * np.float32(2) - np.float32(1), ["f32"])
    want, fl = want_slot(F32, SUM, float((x.astype(np.float64) * 2 - 1).sum()), n)
    valid = (src, F32, SUM, n, [F32], [xd.ptr], [0])
    refusals = [
        ("n == 0", (src, F32, SUM, 0, [F32], [xd.ptr], [0]), {}, ERR_EMPTY),
        ("no arguments", (src, F32, SUM, n, [F32], [xd.ptr], [0]), {"nargs": 0}, ERR_ARG),
        ("9 arguments", (src, F32, SUM, n, [F32] * 9, [xd.ptr] * 9, [0] * 9), {}, ERR_ARG),
        ("bad value dtype", (src, 42, SUM, n, [F32], [xd.ptr], [0]), {}, ERR_ARG),
        ("bad argument dtype", (src, F32, SUM, n, [I128], [xd.ptr], [0]), {}, ERR_ARG),
        ("ComplexF64 scalar", (b"a0", C128, SUM, n, [C128], [None], [0]), {}, ERR_ARG),
        ("misaligned by 1", (src, F32, SUM, n, [F32], [big.ptr + 4], [0]), {}, ERR_UNSUPPORTED),
        ("misaligned by 2", (src, F32, SUM, n, [F32], [big.ptr + 8], [0]), {}, ERR_UNSUPPORTED),
        ("misaligned by 7", (src, F32, SUM, n, [F32], [big.ptr + 28], [0]), {}, ERR_UNSUPPORTED),
        ("misaligned second argument", (src, F32, SUM, n, [F32, F32], [xd.ptr, big.ptr + 12], [0, 0]), {}, ERR_UNSUPPORTED),
        ("null result slot", (src, F32, SUM, n, [F32], [xd.ptr], [0]), {"out": 0}, ERR_ARG),
        ("null expression", (None, F32, SUM, n, [F32], [xd.ptr], [0]), {}, ERR_ARG),
    ]
    for v, op in [(U8, PROD), (U8, MAX), (U8, MIN), (F32, ALL), (F64, ANY), (I32, COUNT), (I64, ALL), (C64, MAX), (C128, MIN), (C64, ALL),
                  (I128, COUNT), (I128, ANY), (F32, EXTREMA), (F64, 99)]:
        refusals.append((f"value {v} op {op}", (src, v, op, n, [F32], [xd.ptr], [0]), {}, ERR_UNSUPPORTED))
    try:
        for name, (s, v, op, nn, dts, ptrs, scal), kw, code in refusals:
            slot.clear()
            n0 = rt1.launches()
            st = mr_status(rt1, s, v, op, nn, dts, ptrs, scal, kw.get("out", slot.ptr), nargs=kw.get("nargs"))
            assert st == code, (name, st, code)
            assert rt1.launches() == n0, (name, "launched")
            assert slot.get() == Slot.FILL, (name, "wrote the slot")
            st = mr_status(rt1, *valid, slot.ptr)
            assert st == OK and slot_matches(slot.get(), want, fl), (name, "the next valid call")
        st = mr_status(rt1, src, F32, SUM, n, [F32], [big.ptr + 32], [0], slot.ptr)         # 8 elements in: aligned to 4, accepted
        assert st == OK and slot_matches(slot.get(), want, fl)
    finally:
        xd.free()
        big.free()
        slot.free()


# ---------------------------------------------------------------------------------------------------------- (4) public calls
LAYOUTS = {1: [[70001]], 2: [[0, 9000], [4099, 2047]], 8: [[3000, 0, 2049, 5, 4103, 1, 2048, 12345]]}


def _darray(dab, x, parts):
    cuts = np.cumsum([0] + list(parts))
    return dab.darray_from_chunks([x[cuts[k]:cuts[k + 1]] for k in range(len(parts))], (len(parts),))


def contract(val, op, x_chunks, rdt):
    """Each chunk reduced exactly and rounded once to the result type, then a left fold in procs order in the result type; an empty
    chunk contributes the identity."""
    rdt = np.dtype(rdt)
    vals = []
    for m in x_chunks:
        if len(m) == 0:
            vals.append(rdt.type({PROD: 1, ALL: 1}.get(op, 0)))
            continue
        a = acc_of(val, op, m)
        if val == U8:
            a = {ALL: int(a == len(m)), ANY: int(a != 0)}.get(op, a)
        if rdt.kind in "iu" and op in (SUM, PROD, COUNT, ALL, ANY):
            a = a - (1 << 64) if a >> 63 else a
        vals.append(rdt.type(a))
    r = vals[0]
    with np.errstate(all="ignore"):
        for v in vals[1:]:
            if op in (MAX, MIN):
                r = jl_extreme(np.asarray([r, v], dtype=rdt), op == MAX) if rdt.kind == "f" else (max(r, v) if op == MAX else min(r, v))
            elif op == ALL:
                r = rdt.type(r and v)
            elif op == ANY:
                r = rdt.type(r or v)
            elif rdt.kind == "c":
                r = rdt.type(complex(r.real + v.real, r.imag + v.imag))
            else:
                r = rdt.type(r + v if op in (SUM, COUNT) else r * v)
    return r


def _same(got, want):
    """Same value and type; NaN equals NaN (payloads are not compared)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype:
        return False
    if want.dtype.kind == "c":
        got, want = np.asarray([got.real, got.imag]), np.asarray([want.real, want.imag])
    if want.dtype.kind == "f":
        nan = np.isnan(want)
        return np.array_equal(np.isnan(got), nan) and got[~nan].tobytes() == want[~nan].tobytes()
    return got.tobytes() == want.tobytes()


def _chunks(x, parts):
    cuts = np.cumsum([0] + list(parts))
    return [x[cuts[k]:cuts[k + 1]] for k in range(len(parts))]


@pytest.mark.parametrize("nw", [1, 2, 8])
def test_public_mapreduce_dot_count(dab, request, nw):
    """mapreduce with a closure, dot, count / any / all with general predicates, on layouts with an empty chunk: exact against the
    contract, with the result type and 2 launches per non-empty chunk."""
    rt = request.getfixturevalue(f"rt{nw}")
    for li, parts in enumerate(LAYOUTS[nw]):
        n = sum(parts)
        nonempty = sum(1 for p in parts if p)
        rng = np.random.default_rng(100 * nw + li)
        for val in (F32, F64, I32, I64):
            T = NP[val]
            for op in (SUM, PROD, MAX, MIN):
                _, f, twin = spec(val, op)
                x = base_input(val, op, n, rng)
                E = [p for p in np.cumsum([0] + parts)[:-1] if p < n] + [n - 1]
                if val in (F32, F64) and op in (MAX, MIN):
                    x[E[int(rng.integers(len(E)))]] = T.type(-(1 if op == MAX else -1) * 5 * G)
                if op in (MAX, MIN) and 0 in parts:
                    d = _darray(dab, x, parts)
                    with pytest.raises(dab.ArgumentError):
                        dab.mapreduce(f, {MAX: "max", MIN: "min"}[op], d)
                    d.close()
                    continue
                d = _darray(dab, x, parts)
                n0 = rt.launches()
                got = dab.mapreduce(f, {SUM: "+", PROD: "*", MAX: "max", MIN: "min"}[op], d)
                if not HOSTMEM:
                    assert rt.launches() - n0 == 2 * nonempty, (val, op, rt.launches() - n0)
                rdt = np.int64 if val in (I32, I64) and op in (SUM, PROD) else T
                want = contract(val, op, [mapped(val, twin, c) for c in _chunks(x, parts)], rdt)
                assert _same(got, want), (nw, parts, val, op, got, want)
                d.close()
        # dot: Float32, Float64, Int64 and ComplexF64 (conj of the first argument)
        for T in (np.float32, np.float64, np.int64, np.complex128):
            if T == np.complex128:
                x = (_grid(rng, n) + 1j * _grid(rng, n)).astype(T)
                y = (_grid(rng, n) + 1j * _grid(rng, n)).astype(T)
                prodv = np.conj(x) * y
                val = C128
            elif T == np.int64:
                x, y = rng.integers(-2 ** 62, 2 ** 62, n), rng.integers(-2 ** 62, 2 ** 62, n)
                with np.errstate(all="ignore"):
                    prodv = x * y
                val = I64
            else:
                x, y = _grid(rng, n).astype(T), _grid(rng, n).astype(T)
                prodv = x * y
                val = F32 if T == np.float32 else F64
            dx, dy = _darray(dab, x, parts), _darray(dab, y, parts)
            n0 = rt.launches()
            got = dab.dot(dx, dy)
            if not HOSTMEM:
                assert rt.launches() - n0 == 2 * nonempty
            want = contract(val, SUM, _chunks(prodv, parts), T)
            assert _same(got, want), ("dot", nw, T, got, want)
            dx.close()
            dy.close()
        # count / any / all with predicates that are not a comparison of the element with a constant
        x = _grid(rng, n, -40, 40).astype(np.float64)
        d = _darray(dab, x, parts)
        pred, twin = (lambda v: v * v > 0.001), (lambda v: v * v > 0.001)
        assert dab.count(d, pred) == int(np.count_nonzero(twin(x)))
        band = lambda v: (v > 0.01) & (v < 0.02)
        assert dab.any(d, band) == bool(((x > 0.01) & (x < 0.02)).any())
        d.close()
        starts = [int(c) for c in np.cumsum([0] + parts)[:-1]]
        for p in sorted({s for s, q in zip(starts, parts) if q} | {n - 1} | {v for v in (TILE, TILE + 1024, 2 * TILE) if v < n}):
            xa = np.full(n, 3.0)
            xa[p] = -3.0
            d = _darray(dab, xa, parts)
            n0 = rt.launches()
            assert dab.all(d, lambda v: v * v - 9.0 == 0.0) is True
            assert dab.all(d, lambda v: v * 2.0 > 0.0) is False, p
            assert dab.any(d, lambda v: v * 2.0 < 0.0) is True, p
            assert dab.count(d, lambda v: v * 2.0 < 0.0) == 1, p
            if not HOSTMEM:
                assert rt.launches() - n0 == 8 * nonempty
            d.close()


@pytest.mark.parametrize("nw", [1, 2, 8])
def test_public_multi_argument_isequal_norm(dab, request, nw):
    """mapreduce over a DArray of another layout (the halo path), a host array and scalars; isequal with one differing element at each
    split position, -0.0 == 0.0 and NaN != NaN; norm(x, p) for general p against a long-double reference."""
    rt = request.getfixturevalue(f"rt{nw}")
    for li, parts in enumerate(LAYOUTS[nw]):
        n = sum(parts)
        rng = np.random.default_rng(7 * nw + li)
        x, y, h = _grid(rng, n), _grid(rng, n), _grid(rng, n)
        d = _darray(dab, x, parts)
        e = dab.distribute(y)                                          # the default layout: not d's
        f = lambda a, b, c, s, t: a * b + c * s - t
        got = dab.mapreduce(f, "+", d, e, h, 0.75, np.float32(0.125))
        m = x * y + h * 0.75 - 0.125
        assert _same(got, contract(F64, SUM, _chunks(m, parts), np.float64)), (nw, parts, got)
        xi = rng.integers(-2 ** 62, 2 ** 62, n)
        yi = rng.integers(-2 ** 62, 2 ** 62, n)
        di, ei = _darray(dab, xi, parts), dab.distribute(yi)
        got = dab.mapreduce(lambda a, b, s: a * b - s, "*", di, ei, 3)
        with np.errstate(all="ignore"):
            mi = xi * yi - 3
        assert _same(got, contract(I64, PROD, _chunks(mi, parts), np.int64)), (nw, parts, got)
        di.close()
        ei.close()
        # isequal
        xs = np.where(x == 0, 1.0, x)
        d2 = _darray(dab, xs, parts)
        assert dab.isequal(d2, xs.copy()) is True
        d3 = dab.distribute(xs)
        assert dab.isequal(d2, d3) is True
        d3.close()
        zs = xs.copy()
        zs[::3] = 0.0
        dz = _darray(dab, zs, parts)
        assert dab.isequal(dz, np.where(zs == 0, -0.0, zs)) is True             # -0.0 == 0.0
        starts = np.cumsum([0] + parts)
        pos = set()
        for k, p in enumerate(parts):
            if p:
                s = int(starts[k])
                pos |= {s + q for q in (0, 1, p - 1, TILE - 1, TILE, TILE + 1023, TILE + 1024, (p // TILE) * TILE) if 0 <= q < p}
        for p in sorted(pos):
            o = xs.copy()
            o[p] = o[p] + 1.0
            assert dab.isequal(d2, o) is False, p
        nn = xs.copy()
        nn[n // 2] = np.nan
        dn = _darray(dab, nn, parts)
        assert dab.isequal(dn, nn.copy()) is False                               # NaN is not == NaN
        for t in (d, e, d2, dz, dn):
            t.close()
        # norm(x, p): powers and their sum in Float64, within a bound of a long-double reference
        for T in (np.float64, np.float32):
            xv = (rng.standard_normal(n) * 3).astype(T)
            dv = _darray(dab, xv, parts)
            for p in (3, 1.5, 0.5):
                got = dab.norm(dv, p)
                s = np.sum(np.abs(xv.astype(np.longdouble)) ** np.longdouble(p))
                ref = s ** (np.longdouble(1) / np.longdouble(p))
                assert np.asarray(got).dtype == np.dtype(T), (T, p, type(got))
                tol = (4 * n + 16) * np.finfo(np.float64).eps / min(p, 1.0) + (np.finfo(np.float32).eps if T == np.float32 else 0)
                assert abs(np.longdouble(got) - ref) <= tol * ref, (nw, T, p, got, ref)
            dv.close()


# ---------------------------------------------------------------------------------------------------------- (5) full size
def _need(rt, gib):
    if rt.device_info()["free_bytes"] < gib * 2 ** 30:
        pytest.skip(f"needs {gib} GiB of free device memory")


def test_full_size_k_gt_2_exact(dab, rt1):
    """3 tiles per CTA (n >= 32769 * 2048): Float32 sum and max (8- and 4-byte carriers) and an Int128 sum (16 bytes), exact."""
    _need(rt1, 3)
    assert model_mr(K_GT_2_N)["k"] == 3
    slot = Slot(rt1)
    bad = []
    try:
        for val, op in FULL_SIZE_RUNS[K_GT_2_N]:
            bad += run_abi_cases(rt1, slot, val, op, K_GT_2_N, np.random.default_rng(val * 10 + op))
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:6])


def test_full_size_16384_partials(dab, rt1):
    """16384 partials in dab_mr_final: Float32 sum and max, and a ComplexF64 sum (1 GiB)."""
    _need(rt1, 4)
    assert model_mr(PARTS_16384_N)["grid"] == MAX_PARTS
    slot = Slot(rt1)
    bad = []
    try:
        for val, op in FULL_SIZE_RUNS[PARTS_16384_N]:
            bad += run_abi_cases(rt1, slot, val, op, PARTS_16384_N, np.random.default_rng(val * 10 + op + 1))
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:6])


@pytest.mark.parametrize("n", [PARTS_16384_N16, K_GT_2_N16], ids=["parts16384", "k3"])
def test_full_size_float16_argument(dab, rt1, n):
    """The final-fold cases of 8-element steps: 16384 partials (the last CTA with one tile) and 3 tiles per CTA, each with a tail, for a
    Float16 argument (about 134M elements) with Float16 and Float32 values (8- and 4-byte carriers)."""
    _need(rt1, 2)
    m = model_mr(n, TILE16)
    assert (m["grid"] == MAX_PARTS) if n == PARTS_16384_N16 else (m["k"] == 3), m
    slot = Slot(rt1)
    bad = []
    try:
        for val, op in FULL_SIZE_RUNS16:
            bad += run_abi_cases(rt1, slot, val, op, n, np.random.default_rng(val * 10 + op + 2), arg16=True)
    finally:
        slot.free()
    assert not bad, "; ".join(bad[:6])


def test_full_size_bool_all_any_past_2_31(dab, rt1):
    """Bool all / any over one chunk of more than 2^31 elements, the deciding element past index 2^31 (64-bit indexing)."""
    _need(rt1, 4)
    n = BOOL_2_31_N
    src, _ = source(spec(U8, ALL)[1], ["bool"])
    base = rt1.alloc(n + 64)
    slot = Slot(rt1)
    try:
        for op, fill in ((ALL, 1), (ANY, 0)):
            v = np.asarray([fill], dtype=np.uint8)
            _lib().call("dab_fill", rt1.ctx, U8, C.c_void_p(base), n, C.c_void_p(v.ctypes.data))
            rt1.sync()
            for p in (None, (1 << 31) + 5, n - 1, model_mr(n)["tail"][0]):
                if p is not None:
                    flip = np.asarray([1 - fill], dtype=np.uint8)
                    _lib().call("dab_h2d", rt1.ctx, C.c_void_p(base + p), C.c_void_p(flip.ctypes.data), 1)
                slot.clear()
                assert mr_status(rt1, src, U8, op, n, [U8], [base], [0], slot.ptr) == OK
                count = (n if fill else 0) + (0 if p is None else (-1 if fill else 1))
                want, fl = want_slot(U8, op, count, n)
                assert slot.get() == want, (op, p, show(slot.get()), show(want))
                if p is not None:
                    back = np.asarray([fill], dtype=np.uint8)
                    _lib().call("dab_h2d", rt1.ctx, C.c_void_p(base + p), C.c_void_p(back.ctypes.data), 1)
                    rt1.sync()
    finally:
        rt1.free(base)
        slot.free()
