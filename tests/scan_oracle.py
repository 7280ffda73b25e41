"""TEST INFRASTRUCTURE for scans (``cumsum`` / ``cumprod`` / ``accumulate`` and their ``!`` forms).

  * ``jl_accumulate``: a sequential restatement of Julia's ``accumulate!`` (base/accumulate.jl) on NumPy arrays -- the result-type table,
    ``reduce_first``, the fold in the result type's arithmetic (Float32 adds in Float32, Int32 ``accumulate(+)`` wrapping at 32 bits,
    ``add_sum`` / ``mul_prod`` widening), Julia's ``max`` / ``min`` (tests/julia_scalar.py: NaN propagates, max(-0.0, 0.0) = 0.0).
    It is the reference the kernels are checked against on inputs whose results are exact in any order.
  * ``install_hostmem(fake)``: emulated ``dab_scan`` / ``dab_scan_totals`` / ``dab_scan_carrier_dtype`` on a ``hostmem_abi.HostMemABI``,
    following the kernels' carrier arithmetic (fp64 for float sums and products, Int64 for integers and Bool, the element type for max /
    min), so that the host runtime's whole scan flow runs without a GPU.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import julia_scalar as jl

F32, F64, I32, I64, U8 = range(5)
SUM, PROD, MAX, MIN = range(4)
OPS = {"+": SUM, "*": PROD, "max": MAX, "min": MIN}
_NP = {F32: np.dtype(np.float32), F64: np.dtype(np.float64), I32: np.dtype(np.int32), I64: np.dtype(np.int64), U8: np.dtype(np.bool_)}


def result_type(dtype, op: str, cum: bool) -> np.dtype:
    """The issue's table: cumsum / cumprod (``cum``: add_sum / mul_prod) and accumulate(op) (promote_op(op, T, T))."""
    dt = np.dtype(dtype)
    if dt == np.dtype(np.int32):
        return np.dtype(np.int64) if cum and op in ("+", "*") else dt
    if dt == np.dtype(np.bool_):
        return np.dtype(np.int64) if op == "+" else dt
    return dt


def _fold_rows(op: str, rows: np.ndarray, W: np.dtype, init=None) -> np.ndarray:
    """Sequential fold along axis 0 in the arithmetic of W; the first row is reduce_first (or op(init, x1))."""
    x = rows.astype(W) if W != np.dtype(np.bool_) else rows.astype(bool)
    if init is not None:
        x = np.concatenate([np.full((1,) + x.shape[1:], init, dtype=x.dtype), x])
    if op in ("+", "*") and x.dtype != np.dtype(np.bool_):
        with np.errstate(all="ignore"):
            out = (np.cumsum if op == "+" else np.cumprod)(x, axis=0, dtype=x.dtype)
    else:
        out = np.empty_like(x)
        if len(x):
            out[0] = x[0]
        for r in range(1, len(x)):
            b = {"+": "or", "*": "and"}.get(op, op) if x.dtype == np.dtype(np.bool_) else op
            out[r] = jl.vbin({"max": "max", "min": "min", "or": "or", "and": "and"}[b], out[r - 1], x[r])
    return out[1:] if init is not None else out


def jl_accumulate(op: str, A: np.ndarray, dims: int, init=None, cum: bool = False) -> np.ndarray:
    """``accumulate(op, A; dims, init)`` (``cum``: ``cumsum`` / ``cumprod``) as Julia computes it, one fibre after another."""
    A = np.asarray(A)
    R = result_type(A.dtype, op, cum)
    if dims > A.ndim:
        return A.astype(R)                                       # copyto!(B, A): init is not applied
    B = np.moveaxis(A, dims - 1, 0)
    if A.dtype == np.dtype(np.bool_) and op == "+":
        W = np.dtype(np.int64)                                   # Bool + Bool is Int
    else:
        W = R
    out = _fold_rows(op, B, W, init)
    return np.moveaxis(out.astype(R), 0, dims - 1)


# ---- host-memory emulation of the scan entry points --------------------------------------------------------------------------------


def carrier(in_code: int, op: int) -> np.dtype:
    if op in (MAX, MIN):
        return _NP[in_code]
    return np.dtype(np.float64) if in_code in (F32, F64) else np.dtype(np.int64)


def served(in_code: int, op: int, out_code: int) -> bool:
    if op not in (SUM, PROD, MAX, MIN):
        return False
    if in_code in (F32, F64, I64):
        return out_code == in_code
    if in_code == I32:
        return out_code == I32 or (op in (SUM, PROD) and out_code == I64)
    if in_code == U8:
        return out_code == (I64 if op == SUM else U8)
    return False


def _identity(A: np.dtype, op: int):
    if op == SUM:
        return A.type(-0.0) if A.kind == "f" else A.type(0)
    if op == PROD:
        return A.type(1)
    if A == np.dtype(np.bool_):
        return op == MIN
    if A.kind == "f":
        return A.type(-np.inf if op == MAX else np.inf)
    info = np.iinfo(A)
    return A.type(info.min if op == MAX else info.max)


def emulate_scan(in_code, op, out_code, x: np.ndarray, inner, ln, outer, carry):
    """The kernels' result: the inclusive scan of each fibre in the carrier, seeded by carry, each output narrowed once."""
    A = carrier(in_code, op)
    v = x.reshape((inner, ln, outer), order="F")
    rows = np.moveaxis(v, 1, 0).astype(A)                         # (len, inner, outer)
    name = {SUM: "+", PROD: "*", MAX: "max", MIN: "min"}[op]
    if carry is not None:
        rows = np.concatenate([carry.reshape((1, inner, outer), order="F"), rows])
    if op in (SUM, PROD) or A != np.dtype(np.bool_):
        out = _fold_rows(name, rows, A)
    else:
        out = _fold_rows(name, rows, np.dtype(np.bool_))
    if carry is not None:
        out = out[1:]
    return np.moveaxis(out, 0, 1)                                 # (inner, len, outer) in the carrier


def install_hostmem(fake):
    """Adds ``dab_scan`` / ``dab_scan_totals`` / ``dab_scan_carrier_dtype`` to a ``hostmem_abi.HostMemABI``."""
    import hostmem_abi as H

    def check(in_code, op, out_code):
        return 0 if served(int(in_code), int(op), int(out_code)) else 6      # DAB_ERR_UNSUPPORTED

    def dab_scan_carrier_dtype(in_code, op, out_code, out):
        st = check(in_code, op, out_code)
        if st == 0:
            A = carrier(int(in_code), int(op))
            out._obj.value = (F64 if A.kind == "f" else I64) if int(op) in (SUM, PROD) else int(in_code)
        return st

    def _args(in_code, op, out_code, x, inner, ln, outer, carry_p):
        in_code, op, out_code, inner, ln, outer = (int(v) for v in (in_code, op, out_code, inner, ln, outer))
        A = carrier(in_code, op)
        xv = H._view(x, inner * ln * outer, _NP[in_code]).copy()
        cv = H._view(carry_p, inner * outer, A).copy() if H._addr(carry_p) else None
        return in_code, op, out_code, inner, ln, outer, A, xv, cv

    def dab_scan(ctx, in_code, op, out_code, x, inner, ln, outer, carry_p, y):
        st = check(in_code, op, out_code)
        if st:
            return st
        in_code, op, out_code, inner, ln, outer, A, xv, cv = _args(in_code, op, out_code, x, inner, ln, outer, carry_p)
        if inner * ln * outer == 0:
            return 0
        r = emulate_scan(in_code, op, out_code, xv, inner, ln, outer, cv)
        with np.errstate(all="ignore"):
            H._view(y, inner * ln * outer, _NP[out_code])[:] = r.reshape(-1, order="F").astype(_NP[out_code])
        fake.launches += 1
        return 0

    def dab_scan_totals(ctx, in_code, op, out_code, x, inner, ln, outer, totals):
        st = check(in_code, op, out_code)
        if st:
            return st
        in_code, op, out_code, inner, ln, outer, A, xv, _ = _args(in_code, op, out_code, x, inner, ln, outer, None)
        if inner * outer == 0:
            return 0
        tv = H._view(totals, inner * outer, A)
        if ln == 0:
            tv[:] = _identity(A, op)
        else:
            tv[:] = emulate_scan(in_code, op, out_code, xv, inner, ln, outer, None)[:, -1, :].reshape(-1, order="F")
        fake.launches += 1
        return 0

    fake.dab_scan = dab_scan
    fake.dab_scan_totals = dab_scan_totals
    fake.dab_scan_carrier_dtype = dab_scan_carrier_dtype
    return fake
