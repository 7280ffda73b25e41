"""TEST INFRASTRUCTURE -- a NumPy model of Julia's ``findmax`` / ``findmin`` (Base ``_findmax`` / ``findminmax!``), and a host-memory
emulation of the K20 entry points (``dab_findminmax``, ``dab_findminmax_dim``, ``dab_combine_findminmax``) for tests/hostmem_abi.py.

The model of Julia's loops is written from memory of Base (Julia 1.10): ``findmax`` replaces the current best ``(v, i)`` by a later
``(x, k)`` when ``isless(v, x)``, ``findmin`` when ``isgreater(v, x)``, with ``isless`` / ``isgreater`` on floats as below.  There is no
Julia here to check it against.

* ``seq_find`` is the literal sequential loop over column-major linear order.
* ``find`` / ``find_dims`` are the vectorised model: the first position of the largest order key, the key being the isless order of the
  mapped value (every NaN on top, reversed for findmin).  tests/test_cpu_findmax.py checks them against ``seq_find``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import hostmem_abi as hm

FINDMAX, FINDMIN = 0, 1


def isless(a, b) -> bool:
    """Base.isless for Bool, Int32, Int64, Float32, Float64 scalars: NaN after everything, -0.0 before +0.0."""
    if isinstance(a, np.floating):
        an, bn = bool(np.isnan(a)), bool(np.isnan(b))
        return (not an and (bn or bool(np.signbit(a)) > bool(np.signbit(b)))) or bool(a < b)
    return bool(a < b)


def isgreater(a, b) -> bool:
    """Base.isgreater: ``isless(b, a)`` between ordered values, ``isless(a, b)`` when either is unordered (NaN)."""
    if isinstance(a, np.floating) and (np.isnan(a) or np.isnan(b)):
        return isless(a, b)
    return isless(b, a)


def seq_find(which: int, a: np.ndarray, f=None):
    """``findmax(f, a)`` / ``findmin(f, a)`` as Julia's loop: (value, 0-based column-major linear index)."""
    flat = np.asarray(a).ravel(order="F")
    m = flat if f is None else _apply(f, flat)
    better = isless if which == FINDMAX else isgreater
    v, i = m[0], 0
    for k in range(1, m.size):
        if better(v, m[k]):
            v, i = m[k], k
    return v, i


def _apply(f, x):
    with np.errstate(all="ignore"):
        return np.asarray(f(x)).astype(np.asarray(f(x[:1])).dtype)


def order_keys(which: int, m: np.ndarray) -> np.ndarray:
    """Order keys as uint64: larger is better for both functions."""
    m = np.asarray(m)
    if m.dtype == np.bool_:
        k = m.astype(np.uint64)
        return k if which == FINDMAX else ~k
    code = {np.dtype(np.float32): hm.F32, np.dtype(np.float64): hm.F64, np.dtype(np.int32): hm.I32, np.dtype(np.int64): hm.I64}[m.dtype]
    raw = m.view(np.uint32 if m.dtype.itemsize == 4 else np.uint64)
    k = hm.radix_enc(raw, code).astype(np.uint64)
    top = np.uint64(0xFFFFFFFF if m.dtype.itemsize == 4 else 0xFFFFFFFFFFFFFFFF)
    if which == FINDMIN:
        k = top - k
    if m.dtype.kind == "f":
        with np.errstate(over="ignore"):
            k = np.where(np.isnan(m), top, k - np.uint64(1) if which == FINDMIN else k)
    return k


def find(which: int, a: np.ndarray, f=None):
    flat = np.asarray(a).ravel(order="F")
    m = flat if f is None else _apply(f, flat)
    i = int(np.argmax(order_keys(which, m)))              # the first position of the largest key
    return m[i], i


def julia_index(shape, i0: int):
    if len(shape) == 1:
        return i0 + 1
    return tuple(int(c) + 1 for c in np.unravel_index(i0, shape, order="F"))


def find_dims(which: int, a: np.ndarray, dims, f=None):
    """``findmax(f, a; dims)``: (values, 1-based global linear indices), both shaped like ``reduced_indices(a, dims)``."""
    a = np.asarray(a)
    N = a.ndim
    dims = {dims} if isinstance(dims, int) else set(dims)
    red = [k for k in range(N) if k + 1 in dims]
    kept = [k for k in range(N) if k + 1 not in dims]
    rshape = tuple(1 if k + 1 in dims else s for k, s in enumerate(a.shape))
    m = a if f is None else _apply(f, a.ravel(order="F")).reshape(a.shape, order="F")
    g = np.arange(a.size, dtype=np.int64).reshape(a.shape, order="F")
    nk = int(np.prod([a.shape[k] for k in kept])) if kept else 1
    nr = int(np.prod([a.shape[k] for k in red])) if red else 1
    M = np.transpose(m, kept + red).reshape((nk, nr), order="F")
    G = np.transpose(g, kept + red).reshape((nk, nr), order="F")
    if nk == 0:
        return np.empty(rshape, dtype=m.dtype), np.empty(rshape, dtype=np.int64)
    pos = np.argmax(order_keys(which, M.ravel()).reshape(M.shape), axis=1)
    rows = np.arange(nk)
    return M[rows, pos].reshape(rshape, order="F"), (G[rows, pos] + 1).reshape(rshape, order="F")


def same_bits(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


# ---- host-memory emulation of the K20 entry points ----------------------------------------------------------------------------------
_DT = {hm.F32: np.float32, hm.F64: np.float64, hm.I32: np.int32, hm.I64: np.int64, hm.U8: np.bool_}
_MAPS = {0: None, 1: np.abs, 2: lambda x: x * x}


def _check(dtype, which, mapc):
    if int(dtype) in (6, 7) or int(dtype) not in _DT:
        return 6                                                                           # DAB_ERR_UNSUPPORTED
    if int(which) not in (FINDMAX, FINDMIN):
        return 2                                                                           # DAB_ERR_ARG
    if int(mapc) not in _MAPS:
        return 6
    return 0


def _mapf(dtype, mapc):
    return None if int(dtype) == hm.U8 else _MAPS[int(mapc)]


def dab_findminmax(self, ctx, dtype, which, mapc, param, x, n, out):
    st = _check(dtype, which, mapc)
    if st:
        return st
    n = int(n)
    if n == 0:
        return 3                                                                           # DAB_ERR_EMPTY
    v, i = find(int(which), hm._view(x, n, _DT[int(dtype)]).copy(), _mapf(dtype, mapc))
    slot = np.zeros(16, dtype=np.uint8)
    vb = np.asarray([v]).view(np.uint8)
    slot[:vb.size] = vb
    slot[8:16] = np.asarray([i], dtype=np.int64).view(np.uint8)
    C.memmove(hm._addr(out), slot.ctypes.data, 16)
    self.launches += 1
    return 0


def dab_findminmax_dim(self, ctx, dtype, which, mapc, x, idx_in, inner, red, outer, nd, cdims, offs, gdims, out_v, out_i):
    st = _check(dtype, which, mapc)
    if st:
        return st
    inner, red, outer, nd, dt = int(inner), int(red), int(outer), int(nd), _DT[int(dtype)]
    if inner * outer == 0:
        return 0
    if red == 0:
        return 3
    xs = hm._view(x, inner * red * outer, dt).copy().reshape((inner, red, outer), order="F")
    f = _mapf(dtype, mapc)
    m = xs if f is None else _apply(f, xs.ravel(order="F")).reshape(xs.shape, order="F")
    if idx_in is not None and hm._addr(idx_in):
        ii = hm._view(idx_in, inner * red * outer, np.int64).copy().reshape((inner, red, outer), order="F")
    else:
        pos = np.arange(inner * red * outer, dtype=np.int64)
        if nd:
            cd = [int(cdims[k]) for k in range(nd)]
            of = [int(offs[k]) for k in range(nd)]
            gd = [int(gdims[k]) for k in range(nd)]
            c = np.unravel_index(pos, cd, order="F")
            pos = np.ravel_multi_index(tuple(cc + o for cc, o in zip(c, of)), gd, order="F")
        ii = (pos + 1).reshape((inner, red, outer), order="F")
    keys = order_keys(int(which), m.ravel(order="F")).reshape(m.shape, order="F")
    vals = np.empty((inner, outer), dtype=m.dtype)
    idx = np.empty((inner, outer), dtype=np.int64)
    for o in range(outer):
        for i in range(inner):
            ok = ii[i, :, o] != -1
            k, g = keys[i, ok, o], ii[i, ok, o]
            best = np.lexsort((g, ~k))[0]                # largest key, then smallest index
            vals[i, o], idx[i, o] = m[i, ok, o][best], g[best]
    hm._view(out_v, inner * outer, vals.dtype)[:] = vals.ravel(order="F")
    hm._view(out_i, inner * outer, np.int64)[:] = idx.ravel(order="F")
    self.launches += 1
    return 0


def dab_combine_findminmax(self, dtype, which, records, count, out):
    return self._real().dab_combine_findminmax(int(dtype), int(which), C.c_void_p(hm._addr(records)), C.c_size_t(int(count)),
                                                  C.c_void_p(hm._addr(out)))


def install():
    """Add the K20 entry points to the emulation class (idempotent).  ``dab_combine_findminmax`` is host-only: the real library's."""
    hm.HostMemABI.dab_findminmax = dab_findminmax
    hm.HostMemABI.dab_findminmax_dim = dab_findminmax_dim
    hm.HostMemABI.dab_combine_findminmax = dab_combine_findminmax
