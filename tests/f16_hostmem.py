"""TEST INFRASTRUCTURE -- Float16 (``DAB_F16 = 8``) for the host-memory emulation of the C ABI (tests/hostmem_abi.py), so that the host flow
of Float16 DArrays (constructors, movers, broadcast routing, reductions with and without dims, refusals) runs on a CPU-only machine.

``install()`` wraps the emulation's ``dab_fill``, ``dab_rand_u01``, ``dab_reduce`` / ``dab_reduce_host`` / ``dab_mapreduce_all``,
``dab_reducedim``, ``dab_broadcast_expr`` and ``dab_mapreduce_expr``: a call that involves the Float16 code is emulated here, every other
call goes to the method it replaced, so the emulation existing tests see is unchanged.  The models follow the kernels' definitions:
``rand(Float16)`` is ``(hash32 >> 22) * 2^-10``; reductions map each value in Float32 (abs2 rounds ``x*x`` to Float16), sum / prod in an
exact fp64 carrier rounded once to Float16, max / min exact; elementwise expressions evaluate on NumPy float16 values, whose + - * / sqrt
are correctly rounded as Julia's Float16 methods are.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import hostmem_abi as hm

F16 = 8
_H = np.dtype(np.float16)


def _dt(code: int) -> np.dtype:
    return _H if int(code) == F16 else hm._ELEM[int(code)]


def _map(v: np.ndarray, mapc: int, param):
    x = v.astype(np.float32)
    with np.errstate(all="ignore"):
        if mapc >= 16:
            q = np.float32(param) if param is not None else None
            return {16: lambda: x == q, 17: lambda: x != q, 18: lambda: x < q, 19: lambda: x <= q, 20: lambda: x > q, 21: lambda: x >= q,
                    22: lambda: np.isnan(x), 23: lambda: x != 0}[mapc]()
        return {0: lambda: x, 1: lambda: np.abs(x), 2: lambda: (v * v).astype(np.float32), 3: lambda: -x}[mapc]()


def _fold(m: np.ndarray, op: int, axis=None):
    with np.errstate(all="ignore"):
        if op == 0:
            return m.astype(np.float64).sum(axis=axis).astype(_H)
        if op == 1:
            return m.astype(np.float64).prod(axis=axis).astype(_H)
        return np.asarray(hm.jl_extreme(m, 0 if axis is None else axis, op == 2)).astype(_H)


def _param(param):
    return hm._view(param, 1, _H)[0] if param is not None and hm._addr(param) else None


def install():
    """Add the Float16 code to the emulation class (idempotent)."""
    H = hm.HostMemABI
    if getattr(H, "_f16_installed", False):
        return
    H._f16_installed = True
    orig = {n: getattr(H, n) for n in ("dab_fill", "dab_rand_u01", "dab_reduce", "dab_mapreduce_all", "dab_reducedim", "dab_broadcast_expr",
                                       "dab_mapreduce_expr")}

    def dab_fill(self, ctx, dtype, x, n, value):
        if int(dtype) != F16:
            return orig["dab_fill"](self, ctx, dtype, x, n, value)
        hm._view(x, int(n), _H)[:] = hm._view(value, 1, _H)[0]
        self.launches += 1
        return 0

    def dab_rand_u01(self, ctx, dtype, x, n, seed, offset):
        if int(dtype) != F16:
            return orig["dab_rand_u01"](self, ctx, dtype, x, n, seed, offset)
        from oracle import darray_oracle as orc
        idx = np.arange(int(offset), int(offset) + int(n), dtype=np.uint64)
        k = (orc.hash_u32(int(seed), idx) >> np.uint32(22)).astype(np.float64)
        hm._view(x, int(n), _H)[:] = (k * 2.0 ** -10).astype(_H)
        self.launches += 1
        return 0

    def _reduce(self, which, ctx, dtype, op, mapc, param, x, n, out):
        if int(dtype) != F16:
            return orig[which](self, ctx, dtype, op, mapc, param, x, n, out)
        op, mapc = int(op), int(mapc)
        if op == 7:
            return 6                                                 # DAB_ERR_UNSUPPORTED: extrema is a MIN and a MAX reduction
        v = hm._view(x, int(n), _H)
        m = _map(v, mapc, _param(param))
        slot = np.zeros(16, dtype=np.uint8)
        if mapc >= 16 or op in (4, 5, 6):
            c = int(np.count_nonzero(m))
            slot.view(np.int64)[0] = {0: c, 6: c, 4: int(c == v.size), 5: int(c != 0)}[op]
        else:
            if int(n) == 0 and op in (2, 3):
                return 3
            r = _fold(m, op) if int(n) else np.asarray(1.0 if op == 1 else 0.0, _H)
            slot[:2] = np.asarray([r], dtype=_H).view(np.uint8)
            if op in (0, 1):                                         # the fp64 carrier, as the kernel leaves it in bytes [8, 16)
                with np.errstate(all="ignore"):
                    w = m.astype(np.float64)
                    slot[8:] = np.asarray([w.sum() if op == 0 else w.prod()]).view(np.uint8)
        C.memmove(hm._addr(out), slot.ctypes.data, 16)
        self.launches += 1
        return 0

    def dab_reducedim(self, ctx, dtype, op, mapc, x, inner, red, outer, out, accumulate):
        if int(dtype) != F16:
            return orig["dab_reducedim"](self, ctx, dtype, op, mapc, x, inner, red, outer, out, accumulate)
        op, mapc, inner, red, outer = int(op), int(mapc), int(inner), int(red), int(outer)
        if inner * outer == 0 or (red == 0 and int(accumulate)):
            return 0
        if red == 0 and op in (2, 3):
            return 3
        v = hm._view(x, inner * red * outer, _H).reshape((inner, red, outer), order="F")
        m = _map(v, mapc, None)
        o = hm._view(out, inner * outer, _H).reshape((inner, outer), order="F")
        if int(accumulate):
            m = np.concatenate([o.astype(np.float32)[:, None, :], m], axis=1)
        o[...] = _fold(m, op, axis=1)
        self.launches += 1
        return 0

    def _float16_call(dts, nargs, *codes):
        return any(int(c) == F16 for c in codes) or any(int(dts[k]) == F16 for k in range(int(nargs)))

    def dab_broadcast_expr(self, ctx, src, out_dtype, out, shape, out_strides, nargs, dts, ptrs, strides, scal):
        if not _float16_call(dts, nargs, out_dtype):
            return orig["dab_broadcast_expr"](self, ctx, src, out_dtype, out, shape, out_strides, nargs, dts, ptrs, strides, scal)
        from numpy.lib.stride_tricks import as_strided
        expr = self.exprs[src]
        shp = tuple(hm._sz4(shape))
        args = []
        for k in range(int(nargs)):
            dt = _dt(dts[k])
            if ptrs[k]:
                st = [int(strides[4 * k + d]) for d in range(4)]
                span = 1 + sum((shp[d] - 1) * st[d] for d in range(4))
                args.append(as_strided(hm._view(ptrs[k], span, dt), shape=shp, strides=[s * dt.itemsize for s in st]).copy())
            else:
                args.append(np.frombuffer(int(scal[k]).to_bytes(8, "little")[:dt.itemsize], dtype=dt)[0])
        odt = _dt(out_dtype)
        ost = hm._sz4(out_strides)
        ospan = 1 + sum((shp[d] - 1) * ost[d] for d in range(4))
        dest = as_strided(hm._view(out, ospan, odt), shape=shp, strides=[s * odt.itemsize for s in ost])
        with np.errstate(all="ignore"):
            dest[...] = np.broadcast_to(np.asarray(hm.eval_expr(expr, args)), shp).astype(odt)
        self.launches += 1
        return 0

    def dab_mapreduce_expr(self, ctx, src, val_dtype, op, n, nargs, dts, ptrs, scal, out):
        if not _float16_call(dts, nargs, val_dtype):
            return orig["dab_mapreduce_expr"](self, ctx, src, val_dtype, op, n, nargs, dts, ptrs, scal, out)
        op, n = int(op), int(n)
        if any(ptrs[k] and hm._addr(ptrs[k]) % (8 * _dt(dts[k]).itemsize) for k in range(int(nargs))):
            return 6                                                 # DAB_ERR_UNSUPPORTED: arrays must be aligned to 8 elements
        args = []
        for k in range(int(nargs)):
            dt = _dt(dts[k])
            args.append(hm._view(ptrs[k], n, dt).copy() if ptrs[k] else np.frombuffer(int(scal[k]).to_bytes(8, "little")[:dt.itemsize], dtype=dt)[0])
        with np.errstate(all="ignore"):
            v = np.broadcast_to(np.asarray(hm.eval_expr(self.exprs[src], args)), (n,)).astype(_dt(val_dtype))
        slot = np.zeros(16, dtype=np.uint8)
        if v.dtype == np.bool_:
            c = int(np.count_nonzero(v))
            slot.view(np.int64)[:] = [{0: c, 6: c, 4: int(c == n), 5: int(c != 0)}[op], c]
        else:                                                        # word 1: the fp64 carrier of + and *; max / min: the extreme again,
            with np.errstate(all="ignore"):                          # in Float32 for Float16 values
                acc = (v.astype(np.float64).sum() if op == 0 else v.astype(np.float64).prod()) if op in (0, 1) else hm.jl_extreme(v, 0, op == 2)
            slot[:v.itemsize] = np.asarray([acc], dtype=v.dtype).view(np.uint8)
            wide = np.float64 if op in (0, 1) else (np.float32 if v.dtype == _H else v.dtype)
            b = np.asarray([acc], dtype=wide).view(np.uint8)
            slot[8:8 + b.size] = b
        C.memmove(hm._addr(out), slot.ctypes.data, 16)
        self.launches += 2
        return 0

    H.dab_fill = dab_fill
    H.dab_rand_u01 = dab_rand_u01
    H.dab_reduce = lambda self, ctx, dtype, op, mapc, param, x, n, out: _reduce(self, "dab_reduce", ctx, dtype, op, mapc, param, x, n, out)
    H.dab_mapreduce_all = lambda self, ctx, dtype, op, mapc, param, x, n, out: _reduce(self, "dab_mapreduce_all", ctx, dtype, op, mapc, param,
                                                                                        x, n, out)
    H.dab_reduce_host = H.dab_mapreduce_all
    H.dab_reducedim = dab_reducedim
    H.dab_broadcast_expr = dab_broadcast_expr
    H.dab_mapreduce_expr = dab_mapreduce_expr
