"""TEST INFRASTRUCTURE -- a model of Julia's scalar methods for Bool, Int32, Int64, Float32 and Float64, written from the Base definitions
(``base/bool.jl``, ``base/int.jl``, ``base/float.jl``, ``base/intfuncs.jl``, ``base/math.jl``, ``base/number.jl``).

It is the reference the elementwise kernels are checked against (``tests/test_gpu_scalar_semantics.py``), so it shares nothing with the
tracer: every method is picked here from the Julia types of the operands, the way Julia dispatches.

  * Values are NumPy scalars of the Julia type (``np.bool_``, ``np.int32``, ``np.int64``, ``np.float32``, ``np.float64``).
  * Float arithmetic runs in the operand's own NumPy type, which rounds as IEEE requires; integer arithmetic wraps.
  * Comparisons between Int64 and a float type are exact comparisons of the two values (Python's int/float comparison is exact).
  * Int64 -> Float32 rounds once (Python's int -> float would round twice).

Documented deviations of the backend are encoded as such and named in ``DEVIATIONS``: integer division, ``rem`` and ``mod`` by zero give 0
(Julia throws ``DivideError``), ``typemin ÷ -1`` wraps (Julia throws), and a Float32 power whose exponent is ``typemin`` uses the magnitude
2^63 / 2^31 (Julia throws ``DomainError`` unless x = ±1).
"""
from __future__ import annotations

import math

import numpy as np

NPT = {"bool": np.bool_, "i32": np.int32, "i64": np.int64, "f32": np.float32, "f64": np.float64}
TAG = {np.dtype(v): k for k, v in NPT.items()}
BITS = {"i32": 32, "i64": 64}
DEVIATIONS = ("integer div / rem / mod by zero give 0", "typemin ÷ -1 wraps", "Float32 ^ typemin uses the exponent's magnitude")


def tag(v) -> str:
    return TAG[np.asarray(v).dtype]


def isfloat(t: str) -> bool:
    return t[0] == "f"


def promote_type(a: str, b: str) -> str:
    """Bool < Int32 < Int64 < Float32 < Float64, except that any float wins over the integers: Int64 with Float32 is Float32."""
    if a == b:
        return a
    if isfloat(a) or isfloat(b):
        return "f64" if "f64" in (a, b) else "f32"
    order = ("bool", "i32", "i64")
    return a if order.index(a) > order.index(b) else b


def _wrap(v: int, t: str):
    b = BITS[t]
    v &= (1 << b) - 1
    return NPT[t](v - (1 << b) if v >> (b - 1) else v)


def _f32_of_int(v: int) -> np.float32:
    """Round an integer to Float32 once, ties to even."""
    a = abs(v)
    if a < 1 << 24:
        return np.float32(v)
    shift = a.bit_length() - 24
    q, r = divmod(a, 1 << shift)
    half = 1 << (shift - 1)
    if r > half or (r == half and q & 1):
        q += 1
    return np.float32(math.copysign(float(q << shift), v))   # q << shift has <= 25 significant bits: exact in Float64


def convert(v, t: str):
    """``convert(T, v)`` for the conversions the kernels perform: widening, int -> float (rounded once), Bool -> number, and the
    narrowing integer stores (in range they are exact; out of range Julia throws InexactError and the backend wraps)."""
    s = tag(v)
    if s == t:
        return v
    if isfloat(t):
        if isfloat(s):
            return NPT[t](v)
        return _f32_of_int(int(v)) if t == "f32" else np.float64(float(int(v)))   # Python int -> float rounds once
    if isfloat(s):
        raise ValueError("float -> integer conversions are not modelled")
    if t == "bool":
        return np.bool_(int(v) != 0)
    return _wrap(int(v), t)


def _ints(a, b):
    return int(a), int(b)


# ---- arithmetic ---------------------------------------------------------------------------------------------------------------
def _arith(op: str, a, b, t: str):
    """``op`` between two values of the same type ``t``."""
    if isfloat(t):
        with np.errstate(all="ignore"):
            if op == "add":
                return a + b
            if op == "sub":
                return a - b
            if op == "mul":
                return a * b
            if op == "div":
                return a / b
            if op == "rem":
                return np.fmod(a, b)                     # exact; sign of the dividend
            if op == "mod":                              # base/float.jl: mod(x::T, y::T) where T<:AbstractFloat
                r = np.fmod(a, b)
                if r == 0:
                    return np.copysign(r, b)
                return r + b if (r > 0) != (b > 0) else r
            if op in ("max", "min"):                     # NaN wins; +0.0 > -0.0
                if np.isnan(a) or np.isnan(b):
                    return NPT[t](np.nan)
                if a == b:
                    pick_a = np.signbit(b) if op == "max" else np.signbit(a)
                    return a if pick_a else b
                return (a if a > b else b) if op == "max" else (a if a < b else b)
        raise ValueError(f"{op} is not defined on {t}")
    if t == "bool":
        if op == "div":
            return _arith("div", convert(a, "f64"), convert(b, "f64"), "f64")
        x, y = bool(a), bool(b)
        r = {"and": x and y, "or": x or y, "xor": x != y, "max": x or y, "min": x and y, "mul": x and y}.get(op)
        if r is None:
            raise ValueError(f"{op} of two Bools")
        return np.bool_(r)
    x, y = _ints(a, b)
    if op == "add":
        return _wrap(x + y, t)
    if op == "sub":
        return _wrap(x - y, t)
    if op == "mul":
        return _wrap(x * y, t)
    if op == "div":                                      # /(x::Integer, y::Integer) = float(x) / float(y)
        return _arith("div", convert(a, "f64"), convert(b, "f64"), "f64")
    if op == "idiv":                                     # truncated; deviations: x ÷ 0 = 0, typemin ÷ -1 wraps
        if y == 0:
            return NPT[t](0)
        q = abs(x) // abs(y)
        return _wrap(q if (x < 0) == (y < 0) else -q, t)
    if op == "rem":                                      # sign of the dividend; deviation: rem(x, 0) = 0
        if y == 0:
            return NPT[t](0)
        r = abs(x) % abs(y)
        return _wrap(-r if x < 0 else r, t)
    if op == "mod":                                      # sign of the divisor; deviation: mod(x, 0) = 0
        if y == 0:
            return NPT[t](0)
        return _wrap(x % y, t)
    if op == "max":
        return NPT[t](max(x, y))
    if op == "min":
        return NPT[t](min(x, y))
    if op == "and":
        return _wrap(x & y, t)
    if op == "or":
        return _wrap(x | y, t)
    if op == "xor":
        return _wrap(x ^ y, t)
    raise ValueError(op)


_CMP = {"eq": lambda x, y: x == y, "ne": lambda x, y: x != y, "lt": lambda x, y: x < y, "le": lambda x, y: x <= y,
        "gt": lambda x, y: x > y, "ge": lambda x, y: x >= y}


def binop(op: str, a, b):
    """Julia's method of ``op`` for the two operands' types (``add sub mul div idiv rem mod max min and or xor`` and the comparisons
    ``eq ne lt le gt ge``)."""
    ta, tb = tag(a), tag(b)
    # base/bool.jl: the Bool methods that are not promotion
    if op == "mul" and ta == "bool" and isfloat(tb):     # *(x::Bool, y::AbstractFloat) = ifelse(x, y, copysign(zero(y), y))
        return b if a else np.copysign(NPT[tb](0), b)
    if op == "mul" and tb == "bool" and isfloat(ta):
        return binop("mul", b, a)
    if op == "add" and ta == "bool" and isfloat(tb):     # +(x::Bool, y::AbstractFloat) = ifelse(x, oneunit(y) + y, y)
        return (NPT[tb](1) + b) if a else b
    if op == "add" and tb == "bool" and isfloat(ta):
        return binop("add", b, a)
    if ta == tb == "bool" and op in ("add", "sub"):      # +(x::Bool, y::Bool) = Int(x) + Int(y)
        return _arith(op, convert(a, "i64"), convert(b, "i64"), "i64")
    if op in _CMP:
        if {ta, tb} in ({"i64", "f32"}, {"i64", "f64"}):  # base/float.jl: exact comparisons of the values
            x = int(a) if ta == "i64" else float(a)
            y = int(b) if tb == "i64" else float(b)
            return np.bool_(_CMP[op](x, y))
        t = promote_type(ta, tb)
        x, y = convert(a, t), convert(b, t)
        with np.errstate(all="ignore"):
            return np.bool_(_CMP[op](x, y))
    t = promote_type(ta, tb)
    if t == "bool" and op in ("add", "sub"):
        t = "i64"
    return _arith(op, convert(a, t), convert(b, t), t)


# ---- unary functions ------------------------------------------------------------------------------------------------------------
def unop(op: str, a):
    t = tag(a)
    if op in ("isnan", "isinf", "isfinite"):
        if not isfloat(t):
            return np.bool_(op == "isfinite")
        return np.bool_({"isnan": np.isnan, "isinf": np.isinf, "isfinite": np.isfinite}[op](a))
    if op in ("sqrt", "inv") and not isfloat(t):         # sqrt(x::Integer) / inv(x::Integer) work in Float64
        return unop(op, convert(a, "f64"))
    if t == "bool":
        if op in ("abs", "abs2", "sign", "floor", "ceil", "trunc", "round"):   # abs(x::Bool) = x, abs2 = x*x = x & x, sign(x::Bool) = x
            return a
        if op == "neg":                                  # -(x::Bool) = -Int(x)
            return _arith("sub", np.int64(0), convert(a, "i64"), "i64")
        raise ValueError(op)
    if not isfloat(t):
        x = int(a)
        if op == "abs":
            return _wrap(abs(x), t)
        if op == "abs2":
            return _wrap(x * x, t)
        if op == "neg":
            return _wrap(-x, t)
        if op == "sign":
            return NPT[t]((x > 0) - (x < 0))
        if op in ("floor", "ceil", "trunc", "round"):
            return a
        raise ValueError(op)
    T = NPT[t]
    with np.errstate(all="ignore"):
        if op == "abs":
            return np.abs(a)
        if op == "abs2":
            return a * a
        if op == "neg":
            return -a
        if op == "sign":                                 # sign(x::Real): ±1, keeps ±0 and NaN
            return a if (a == 0 or np.isnan(a)) else T(1) if a > 0 else T(-1)
        if op == "inv":
            return T(1) / a
        if op == "sqrt":
            return np.sqrt(a)
        if op == "floor":
            return np.floor(a)
        if op == "ceil":
            return np.ceil(a)
        if op == "trunc":
            return np.trunc(a)
        if op == "round":                                # RoundNearest: ties to even
            return np.rint(a)
    raise ValueError(op)


def ifelse(c, a, b):
    t = promote_type(tag(a), tag(b))
    return convert(a, t) if bool(c) else convert(b, t)


# ---- powers ---------------------------------------------------------------------------------------------------------------------
def power_by_squaring(x: np.float64, p: int) -> np.float64:
    """``Base.power_by_squaring`` replayed operation by operation in Float64 (``p >= 0``; a shift by the full width gives 0)."""
    with np.errstate(all="ignore"):
        if p == 1:
            return x
        if p == 0:
            return np.float64(1)
        if p == 2:
            return x * x
        t = (p & -p).bit_length()                        # trailing_zeros(p) + 1
        p >>= t
        t -= 1
        while t > 0:
            x = x * x
            t -= 1
        y = x
        while p > 0:
            t = (p & -p).bit_length()
            p >>= t
            t -= 1
            while t >= 0:
                x = x * x
                t -= 1
            y = y * x
        return y


def pow_f32_int(x: np.float32, n: int) -> np.float32:
    """``^(x::Float32, n::Integer)`` (base/math.jl): ``n == -2`` is ``inv(x)^2``, ``n == 3`` is ``x*x*x``, otherwise
    ``Float32(power_by_squaring(Float64(x), n))``, from ``inv(Float64(x))`` for a negative n.  A typemin exponent uses its magnitude."""
    x = np.float32(x)
    with np.errstate(all="ignore"):
        if n == -2:
            i = np.float32(1) / x
            return i * i
        if n == 3:
            return x * x * x
        if n < 0:
            return np.float32(power_by_squaring(np.float64(1) / np.float64(x), -n))
        return np.float32(power_by_squaring(np.float64(x), n))


def literal_pow(x, p: int):
    """``x^p`` with a literal integer p (``Base.literal_pow``): 0 -> one(x), 1 -> x, 2 -> x*x, 3 -> x*x*x, -1 -> inv(x),
    -2 -> (i = inv(x); i*i); any other p is ``x^p`` -- for Float32 ``pow_f32_int``; Float64 and integer bases are not modelled."""
    t = tag(x)
    if p == 0:
        return NPT[t](1)
    if p == 1:
        return x
    if p == 2:
        return binop("mul", x, x)
    if p == 3:
        return binop("mul", binop("mul", x, x), x)
    if p == -1:
        return unop("inv", x)
    if p == -2:
        i = unop("inv", x)
        return binop("mul", i, i)
    if t == "f32":
        return pow_f32_int(x, p)
    raise ValueError(f"{t} ^ {p} is not modelled (a pow call on the device)")


# ---- vectorised forms (checked against the scalar methods above by tests/test_cpu_scalar_semantics.py) ---------------------------
def vbin(op: str, a, b) -> np.ndarray:
    """``binop`` on NumPy arrays of ONE type (what the kernels see after the tracer's promotion)."""
    a, b = np.asarray(a), np.asarray(b)
    fl = a.dtype.kind == "f"
    with np.errstate(all="ignore"):
        if op in ("add", "sub", "mul", "div") and (fl or op != "div"):
            return {"add": np.add, "sub": np.subtract, "mul": np.multiply, "div": np.divide}[op](a, b)
        if op in _CMP:
            return _CMP[op](a, b)
        if op in ("and", "or", "xor"):
            return {"and": np.bitwise_and, "or": np.bitwise_or, "xor": np.bitwise_xor}[op](a, b)
        if op in ("max", "min"):
            if not fl:
                return (np.maximum if op == "max" else np.minimum)(a, b)
            r = np.where(a > b, a, b) if op == "max" else np.where(a < b, a, b)
            tie = np.where(np.signbit(b), a, b) if op == "max" else np.where(np.signbit(a), a, b)
            r = np.where(a == b, tie, r)
            return np.where(np.isnan(a) | np.isnan(b), a.dtype.type(np.nan), r).astype(a.dtype)
        if fl and op == "rem":
            return np.fmod(a, b)
        if fl and op == "mod":                            # NumPy's floored mod is Julia's (copysign of a zero, r + y otherwise)
            return np.mod(a, b)
        if op == "div":
            return a.astype(np.float64) / b.astype(np.float64)
        z = np.zeros((), a.dtype)
        bs = np.where((b == 0) | (b == -1), np.ones((), a.dtype), b)
        if op == "rem":
            return np.where((b == 0) | (b == -1), z, np.fmod(a, bs))
        if op == "mod":
            return np.where((b == 0) | (b == -1), z, np.mod(a, bs))
        if op == "idiv":
            q = a // bs
            q = q + ((a - q * bs != 0) & ((a < 0) != (bs < 0))).astype(a.dtype)     # floored -> truncated
            return np.where(b == 0, z, np.where(b == -1, np.negative(a), q)).astype(a.dtype)
    raise ValueError(op)


def vun(op: str, a) -> np.ndarray:
    """``unop`` on a NumPy array (a Bool array only takes what Julia keeps Bool)."""
    a = np.asarray(a)
    fl = a.dtype.kind == "f"
    with np.errstate(all="ignore"):
        if op == "abs":
            return np.abs(a) if a.dtype != np.bool_ else a
        if op == "abs2":
            return a * a if a.dtype != np.bool_ else a
        if op == "neg":
            return np.negative(a)
        if op == "sign":
            return np.where(a > 0, a.dtype.type(1), np.where(a < 0, a.dtype.type(-1), a)).astype(a.dtype)
        if op == "sqrt":
            return np.sqrt(a)
        if op == "inv":
            return a.dtype.type(1) / a
        if op in ("floor", "ceil", "trunc", "round"):
            return {"floor": np.floor, "ceil": np.ceil, "trunc": np.trunc, "round": np.rint}[op](a) if fl else a
    raise ValueError(op)


def vcmp_exact(op: str, a, b) -> np.ndarray:
    """``op`` between an Int64 array and a float array (either side), comparing the values exactly."""
    a, b = np.asarray(a), np.asarray(b)
    flip = a.dtype.kind == "f"
    i, f = (b, a) if flip else (a, b)
    f = f.astype(np.float64)
    with np.errstate(all="ignore"):
        t = np.trunc(np.where((f >= -(2.0 ** 63)) & (f < 2.0 ** 63), f, 0.0))          # [-2^63, 2^63): the Int64 cast is exact
        ti = t.astype(np.int64)
        c = np.where(i != ti, np.where(i < ti, -1, 1), np.where(f - t > 0, -1, np.where(f - t < 0, 1, 0)))
        c = np.where(f >= 2.0 ** 63, -1, np.where(f < -(2.0 ** 63), 1, c))
        c = np.where(np.isnan(f), 2, c)
    c = np.where(c == 2, 2, -c) if flip else c
    return {"eq": c == 0, "ne": c != 0, "lt": c == -1, "le": (c == -1) | (c == 0), "gt": c == 1, "ge": (c == 1) | (c == 0)}[op]


# ---- value grids: where elementwise kernels go wrong --------------------------------------------------------------------------------
def _nan(t: str, neg: bool) -> np.ndarray:
    """A quiet NaN with a payload, of either sign."""
    if t == "f32":
        return np.asarray([0xFFC01234 if neg else 0x7FC01234], np.uint32).view(np.float32)[0]
    return np.asarray([0xFFF8000000001234 if neg else 0x7FF8000000001234], np.uint64).view(np.float64)[0]


def grid(t: str, seed: int = 7) -> np.ndarray:
    """The special values of type ``t``, each once (floats: both signs)."""
    T = NPT[t]
    if t == "bool":
        return np.asarray([False, True])
    if not isfloat(t):
        info = np.iinfo(T)
        v = [0, 1, -1, 2, -2, 3, -3, 7, -7, int(info.min), int(info.min) + 1, int(info.max), int(info.max) - 1]
        if t == "i64":
            v += [2 ** 31, -2 ** 31, 2 ** 53 + 1, 2 ** 53 - 1, -(2 ** 53 + 1), -(2 ** 53 - 1), 2 ** 24 + 1, -(2 ** 24 + 1)]
        return np.asarray(v, dtype=T)
    info = np.finfo(T)
    mant = 23 if t == "f32" else 52
    tiny = float(info.smallest_subnormal)
    # 0, the smallest and largest subnormal, floatmin, 1 - eps/2, the ties of round, 2^(p-1) -+ 1/2 and 2^p neighbours, 2^63, floatmax, Inf
    mag = [0.0, tiny, float(info.tiny) - tiny, float(info.tiny), 1 - float(info.eps) / 2, 0.5, 1.0, 1.5, 2.5, 3.0,
           2.0 ** (mant - 1) + 0.5, 2.0 ** mant - 0.5, 2.0 ** mant + 1, 2.0 ** (mant + 1) - 1, 2.0 ** (mant + 1), 2.0 ** (mant + 1) + 2,
           2.0 ** 63, float(info.max), np.inf]
    rng = np.random.default_rng(seed)
    mag += list(np.ldexp(rng.random(3) + 1.0, rng.integers(-20, 20, 3)))
    v = [T(m) for m in mag] + [T(-m) for m in mag]
    return np.asarray(v + [_nan(t, False), _nan(t, True)], dtype=T)


def pairs(xs, ys):
    """The cartesian product as two flat arrays (x varies slowest)."""
    return np.repeat(xs, len(ys)), np.tile(ys, len(xs))


# ---- tables over value grids ------------------------------------------------------------------------------------------------------
def table2(op: str, xs, ys) -> np.ndarray:
    """``op(x, y)`` for every (x, y) in zip(xs, ys), as an array of the result type."""
    out = [binop(op, a, b) for a, b in zip(xs, ys)]
    return np.asarray(out, dtype=np.asarray(out[0]).dtype) if out else np.zeros(0)


def table1(op: str, xs) -> np.ndarray:
    out = [unop(op, a) for a in xs]
    return np.asarray(out, dtype=np.asarray(out[0]).dtype) if out else np.zeros(0)
