"""TEST INFRASTRUCTURE -- an emulation of part of the C ABI (include/dab200.h) over HOST memory, so that the host runtime above the ABI can
run on a CPU-only machine.

Why: the host logic (``distributedarrays.jl_b200/*.py``: tracer and kernel routing, stride tables and ``collapse_dims``, layouts and halo
plans, the samplesort flow incl. ``by``, the Int128 fold, ``copy`` / ``copyto!`` / ``norm`` compositions) can otherwise only run on a GPU
box.  With this module installed by the ``hostmem`` fixture the real ``Runtime`` / ``DArray`` / ``broadcast`` / ``mapreduce`` / ``sort``
code runs unchanged against "device pointers" that are addresses of host buffers, and results are compared with the oracle / NumPy.  It is
never importable from the product: the package has no reference to it, and ``_lib.lib()`` keeps failing loudly when ``libdab200.so`` is
missing.  Nothing here says anything about the CUDA kernels; those are checked by the ``-m gpu`` tier only.

Emulated entry points: lifecycle and buffers (alloc / free / h2d / d2h / d2d / fill / rand_u01), the elementwise family the real
``run_local`` routes to (``dab_affine``, ``dab_unary``, ``dab_binary``, ``dab_binary_scalar``, ``dab_broadcast_expr`` as the strided 4-D
box walk of the NVRTC kernel), ``dab_copy_box`` / ``dab_gather_box`` (halo and view copies, 1- to 16-byte elements), ``dab_transpose_box`` / ``dab_adjoint_box``, ``dab_reduce`` / ``dab_mapreduce_all`` /
``dab_reducedim`` / ``dab_mapreduce_expr`` (sums in a wide carrier: an order-free stand-in for the kernels' trees, compared at tolerance),
``dab_sort`` / ``dab_sort_by_key`` / ``dab_sorted_split``.  The host-only entry points (``dab_reduce_result_dtype``,
``dab_combine_ordered``) are the real library's.

Where the ALGORITHM is the thing under test the emulation follows the kernels, not a NumPy shortcut:
  * ``dab_sort`` / ``dab_sort_by_key`` sort through the same order-preserving radix-key bijection as ``dab_sort_key.cuh``;
    ``dab_sort_by_key`` packs ``radix_key << 32 | position`` into signed 64-bit words (top bit flipped), sorts the words, runs the
    second round on the high half for 64-bit keys and gathers by the low halves -- the composition of ``dab_sortby.cu`` step by step
    (the kernels' own element code is additionally replayed in C++ by ``tools/sortby_host_check.cu``);
  * ``dab_sorted_split`` is the binary search of ``sort_bounds_kernel`` (NaN bound, -0.0 bound, all-NaN tail).
Traced closures are evaluated by a small NumPy interpreter of the expression tree (``eval_expr``; the fixture records which traced
expression each generated source string came from); Int128 sub-expressions run on Python integers wrapped to 128 bits.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import julia_scalar as jl

F32, F64, I32, I64, U8 = range(5)
_NP = {F32: np.dtype(np.float32), F64: np.dtype(np.float64), I32: np.dtype(np.int32), I64: np.dtype(np.int64), U8: np.dtype(np.uint8)}
SIGN64 = np.uint64(0x8000000000000000)
_UNIT = {1: np.dtype(np.uint8), 2: np.dtype(np.uint16), 4: np.dtype(np.uint32), 8: np.dtype(np.uint64), 16: np.dtype("V16")}   # data-movement units


# ---- dab_sort_key.cuh in NumPy ------------------------------------------------------------------------------------------------
def radix_enc(raw: np.ndarray, code: int) -> np.ndarray:
    """raw: the keys' bit patterns as uint32 / uint64."""
    with np.errstate(over="ignore"):
        if code == I32:
            return raw ^ np.uint32(0x80000000)
        if code == I64:
            return raw ^ SIGN64
        if code == F32:
            top, c = np.uint32(0x80000000), np.uint32(0x007FFFFF)
        else:
            top, c = SIGN64, np.uint64(0x000FFFFFFFFFFFFF)
        return np.where((raw & top) != 0, ~raw, raw | top) - c


def radix_dec(k: np.ndarray, code: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        if code == I32:
            return k ^ np.uint32(0x80000000)
        if code == I64:
            return k ^ SIGN64
        if code == F32:
            top, c = np.uint32(0x80000000), np.uint32(0x007FFFFF)
        else:
            top, c = SIGN64, np.uint64(0x000FFFFFFFFFFFFF)
        k = k + c
        return np.where((k & top) != 0, k ^ top, ~k)


def _utype(code: int):
    return np.uint32 if code in (I32, F32) else np.uint64


def by_radix_key(raw: np.ndarray, code: int) -> np.ndarray:
    """``by_radix_key`` of dab_sortby.cu: all NaN keys collapse to the largest key."""
    e = radix_enc(raw, code)
    if code in (F32, F64):
        u = _utype(code)
        absmask = u(0x7FFFFFFF) if code == F32 else u(0x7FFFFFFFFFFFFFFF)
        inf = u(0x7F800000) if code == F32 else u(0x7FF0000000000000)
        e = np.where((raw & absmask) > inf, ~u(0), e)
    return e


# ---- memory -----------------------------------------------------------------------------------------------------------------------
def _addr(x) -> int:
    if x is None:
        return 0
    if isinstance(x, int):
        return x
    if isinstance(x, C.c_void_p):
        return x.value or 0
    if isinstance(x, C.Array):
        return C.addressof(x)
    if hasattr(x, "_obj"):          # byref(...)
        return C.addressof(x._obj)
    raise TypeError(type(x))


def _view(ptr, n: int, dt) -> np.ndarray:
    dt = np.dtype(dt)
    if n == 0:
        return np.empty(0, dtype=dt)
    buf = (C.c_char * (n * dt.itemsize)).from_address(_addr(ptr))
    return np.frombuffer(buf, dtype=dt, count=n)


def _sz4(a):
    return [int(v) for v in a]


class HostMemABI:
    """Duck-types the ``ctypes.CDLL`` of libdab200.so for the entry points listed in the module docstring."""

    def __init__(self):
        self.blocks = {}
        self.launches = 0
        self.calls = []
        self.exprs = {}                                         # generated source -> traced Expr (filled by the fixture's codegen wrapper)

    # -- lifecycle / diagnostics
    def dab_abi_version(self):
        return 1

    def dab_device_count(self, n):
        n._obj.value = 1
        return 0

    def dab_init(self, device, ctx):
        ctx._obj.value = 0xDAB
        return 0

    def dab_shutdown(self, ctx):
        return 0

    def dab_last_error(self, ctx):
        return b"hostmem_abi"

    def dab_status_string(self, st):
        return b"hostmem_abi status"

    def dab_sync(self, ctx):
        return 0

    def dab_launch_count(self, ctx, out):
        out._obj.value = self.launches
        return 0

    # -- events (wall clock), device info, pinned host memory: what bench.py needs to run its host logic against the emulation
    def dab_event_create(self, ctx, out):
        self._events = getattr(self, "_events", {})
        h = 0xE000 + 8 * len(self._events)
        self._events[h] = 0.0
        out._obj.value = h
        return 0

    def dab_event_record(self, ctx, ev):
        import time
        self._events[_addr(ev)] = time.perf_counter()
        return 0

    def dab_event_elapsed_ms(self, ctx, e0, e1, out):
        out._obj.value = max(1e-6, (self._events[_addr(e1)] - self._events[_addr(e0)]) * 1e3)
        return 0

    def dab_event_destroy(self, ctx, ev):
        self._events.pop(_addr(ev), None)
        return 0

    def dab_device_info(self, ctx, sm, cc, free_b, total_b):
        sm._obj.value, cc._obj.value, free_b._obj.value, total_b._obj.value = 132, 90, 1 << 30, 1 << 30
        return 0

    def dab_stream(self, ctx, out):
        out._obj.value = 0
        return 0

    # -- buffers
    def _alloc(self, ctx, nbytes, out):
        buf = C.create_string_buffer(max(int(nbytes), 1) + 256)
        base = (C.addressof(buf) + 255) & ~255
        self.blocks[base] = buf
        out._obj.value = base
        return 0

    def _free(self, ctx, p):
        self.blocks.pop(_addr(p), None)
        return 0

    dab_alloc = dab_alloc_async = dab_host_alloc = _alloc
    dab_free = dab_free_async = dab_host_free = _free

    def _copy(self, ctx, dst, src, n):
        n = int(n)
        if n:
            C.memmove(_addr(dst), _addr(src), n)
        return 0

    dab_h2d = dab_d2h = dab_d2d = _copy

    def dab_fill(self, ctx, dtype, x, n, value):
        dt = _NP[int(dtype)]
        _view(x, int(n), dt)[:] = _view(value, 1, dt)[0]
        self.launches += 1
        return 0

    # -- the elementwise entry points the REAL run_local chooses between (so its routing, its stride tables and collapse_dims run on CPU)
    # Julia's methods (tests/julia_scalar.py), not NumPy's stand-ins: np.maximum / np.sign differ at -0.0, and ÷ through Float64 is wrong for
    # large Int64 values and zero divisors
    _UN = {0: lambda v: v, 1: lambda v: jl.vun("abs", v), 2: lambda v: jl.vun("abs2", v), 3: lambda v: jl.vun("neg", v),
           4: lambda v: jl.vun("sqrt", v), 5: lambda v: jl.vun("inv", v), 6: lambda v: jl.vun("floor", v), 7: lambda v: jl.vun("ceil", v),
           8: lambda v: jl.vun("sign", v)}
    _BINOPS = ("add", "sub", "mul", "div", "rem", "max", "min", "mod", "idiv", "and", "or", "xor")

    @staticmethod
    def _bin(op, a, b):
        a, b = np.asarray(a), np.asarray(b)
        return jl.vbin(HostMemABI._BINOPS[op], a, b).astype(a.dtype)

    def dab_affine(self, ctx, dtype, y, x, a, b, n):
        dt = _NP[int(dtype)]
        xv = _view(x, int(n), dt).copy()
        with np.errstate(all="ignore"):
            _view(y, int(n), dt)[:] = (_view(a, 1, dt)[0] * xv) + _view(b, 1, dt)[0]     # two roundings: NumPy does not contract
        self.launches += 1
        return 0

    def dab_unary(self, ctx, dtype, fn, y, x, n):
        dt = _NP[int(dtype)]
        with np.errstate(all="ignore"):
            _view(y, int(n), dt)[:] = self._UN[int(fn)](_view(x, int(n), dt).copy())
        self.launches += 1
        return 0

    def dab_binary(self, ctx, dtype, op, z, x, y, n):
        dt = _NP[int(dtype)]
        _view(z, int(n), dt)[:] = self._bin(int(op), _view(x, int(n), dt).copy(), _view(y, int(n), dt).copy())
        self.launches += 1
        return 0

    def dab_binary_scalar(self, ctx, dtype, op, z, x, sc, scalar_left, n):
        dt = _NP[int(dtype)]
        xv, sv = _view(x, int(n), dt).copy(), _view(sc, 1, dt)[0]
        _view(z, int(n), dt)[:] = self._bin(int(op), sv, xv) if int(scalar_left) else self._bin(int(op), xv, sv)
        self.launches += 1
        return 0

    def dab_broadcast_expr(self, ctx, src, out_dtype, out, shape, out_strides, nargs, dts, ptrs, strides, scal):
        """The 4-D box walk of the NVRTC kernel: every array argument is read through its own (element) strides, 0 = extruded dimension."""
        from numpy.lib.stride_tricks import as_strided
        expr = self.exprs[src]
        shp = tuple(_sz4(shape))
        npt = {F32: np.float32, F64: np.float64, I32: np.int32, I64: np.int64, U8: np.bool_}
        args = []
        for k in range(int(nargs)):
            dt = np.dtype(npt[int(dts[k])])
            if ptrs[k]:
                st = [int(strides[4 * k + d]) for d in range(4)]
                span = 1 + sum((shp[d] - 1) * st[d] for d in range(4))
                args.append(as_strided(_view(ptrs[k], span, dt), shape=shp, strides=[v * dt.itemsize for v in st]).copy())
            else:
                args.append(np.frombuffer(int(scal[k]).to_bytes(8, "little"), dtype=dt)[0])
        odt = np.dtype(npt[int(out_dtype)])
        ost = _sz4(out_strides)
        ospan = 1 + sum((shp[d] - 1) * ost[d] for d in range(4))
        dest = as_strided(_view(out, ospan, odt), shape=shp, strides=[v * odt.itemsize for v in ost])
        dest[...] = np.broadcast_to(np.asarray(eval_expr(expr, args)), shp).astype(odt)
        self.launches += 1
        return 0

    # -- dab_reducedim on the collapsed (inner, reduce, outer) column-major shape
    def dab_reducedim(self, ctx, dtype, op, mapc, x, inner, red, outer, out, accumulate):
        op, mapc, inner, red, outer = int(op), int(mapc), int(inner), int(red), int(outer)
        dt = _NP[int(dtype)]
        if inner * outer == 0 or (red == 0 and int(accumulate)):
            return 0
        if red == 0 and op in (2, 3):
            return 3                                               # DAB_ERR_EMPTY: max / min over an empty dimension
        v = _view(x, inner * red * outer, dt).reshape((inner, red, outer), order="F")
        code = C.c_int32()
        assert self._real().dab_reduce_result_dtype(int(dtype), op, mapc, C.byref(code)) == 0
        rdt = np.dtype(np.int64) if code.value == I64 else _NP[code.value]
        wide = np.float64 if rdt.kind == "f" else np.int64
        with np.errstate(all="ignore"):
            m = {0: lambda: v, 1: lambda: np.abs(v), 2: lambda: v * v, 3: lambda: -v}[mapc]()
            r = {0: lambda: m.astype(wide).sum(axis=1), 1: lambda: m.astype(wide).prod(axis=1), 2: lambda: jl_extreme(m, 1, True),
                 3: lambda: jl_extreme(m, 1, False)}[op]()
            o = _view(out, inner * outer, rdt).reshape((inner, outer), order="F")
            if int(accumulate):
                r = {0: np.add, 1: np.multiply, 2: lambda a, b: jl_extreme(np.stack([a, b]), 0, True),
                     3: lambda a, b: jl_extreme(np.stack([a, b]), 0, False)}[op](o.astype(r.dtype), r)
            o[...] = r.astype(rdt)
        self.launches += 1
        return 0

    # -- dab_copy_box (4-D box, column-major); refusals as the library's: an element width it has no unit for, a box past either array
    def dab_copy_box(self, ctx, elem_bytes, dst, dst_shape, dst_off, src, src_shape, src_off, extent):
        dsh, dof, ssh, sof, ext = map(_sz4, (dst_shape, dst_off, src_shape, src_off, extent))
        if int(elem_bytes) not in _UNIT:
            return 2                                               # DAB_ERR_ARG
        dt = _UNIT[int(elem_bytes)]
        for d in range(4):
            if ext[d] == 0:
                return 0
            if sof[d] + ext[d] > ssh[d] or dof[d] + ext[d] > dsh[d]:
                return 4                                           # DAB_ERR_DIM_MISMATCH
        d = _view(dst, int(np.prod(dsh)), dt).reshape(dsh, order="F")
        s = _view(src, int(np.prod(ssh)), dt).reshape(ssh, order="F")
        d[tuple(slice(o, o + e) for o, e in zip(dof, ext))] = s[tuple(slice(o, o + e) for o, e in zip(sof, ext))]
        self.launches += 1
        return 0

    # -- linear algebra tiles (NumPy stand-ins: only the HOST logic around them is under test) and small utilities
    def dab_set_option(self, ctx, key, value):
        return 0 if key in (b"ew_tma", b"combine_timeout_ms") else 2     # DAB_ERR_ARG: an unknown key, as the library

    def dab_h2d_2d(self, ctx, dptr, dpitch, hptr, hpitch, row_bytes, cols):
        for c in range(int(cols)):
            C.memmove(_addr(dptr) + c * int(dpitch), _addr(hptr) + c * int(hpitch), int(row_bytes))
        return 0

    def dab_gemv(self, ctx, dtype, trans, A, m, n, x, r):
        dt, m, n = _NP[int(dtype)], int(m), int(n)
        a = _view(A, m * n, dt).reshape((m, n), order="F")
        wide = np.float64 if dt.kind == "f" else np.int64
        with np.errstate(all="ignore"):
            if int(trans):
                _view(r, n, dt)[:] = (a.T.astype(wide) @ _view(x, m, dt).astype(wide)).astype(dt)
            else:
                _view(r, m, dt)[:] = (a.astype(wide) @ _view(x, n, dt).astype(wide)).astype(dt)
        self.launches += 1
        return 0

    def dab_gemm(self, ctx, dtype, transA, m, n, k, A, lda, B, ldb, Cp, ldc):
        dt, m, n, k, lda, ldb, ldc = _NP[int(dtype)], int(m), int(n), int(k), int(lda), int(ldb), int(ldc)
        if m == 0 or n == 0:
            return 0
        wide = np.float64 if dt.kind == "f" else np.int64
        cols_a = m if int(transA) else k
        a = _view(A, lda * cols_a, dt).reshape((lda, cols_a), order="F")[:(k if int(transA) else m)] if k else np.zeros((0, 0), dt)
        b = _view(B, ldb * n, dt).reshape((ldb, n), order="F")[:k] if k else np.zeros((0, n), dt)
        c = _view(Cp, ldc * n, dt).reshape((ldc, n), order="F")
        with np.errstate(all="ignore"):
            c[:m] = ((a.T if int(transA) else a).astype(wide) @ b.astype(wide)).astype(dt) if k else 0
        self.launches += 1
        return 0

    def dab_transpose_box(self, ctx, elem_bytes, dst, dst_ld, src, src_ld, rows, cols, conj=False):
        rows, cols, dst_ld, src_ld = int(rows), int(cols), int(dst_ld), int(src_ld)
        if rows == 0 or cols == 0:
            return 0
        if src_ld < rows or dst_ld < cols:
            return 4                                               # DAB_ERR_DIM_MISMATCH
        if int(elem_bytes) not in _UNIT:
            return 2
        dt = _UNIT[int(elem_bytes)]
        es = dt.itemsize
        s_ = _view(src, src_ld * (cols - 1) + rows, dt)
        d_ = _view(dst, dst_ld * (rows - 1) + cols, dt)
        from numpy.lib.stride_tricks import as_strided
        sv = as_strided(s_, shape=(rows, cols), strides=(es, src_ld * es))
        dv = as_strided(d_, shape=(cols, rows), strides=(es, dst_ld * es))
        dv[...] = sv.T
        if conj:                                                   # Julia's conj: the imaginary part's sign bit flipped, NaN payloads kept
            top = as_strided(_view(dst, (dst_ld * (rows - 1) + cols) * es, np.uint8)[es - 1:], shape=(cols, rows), strides=(es, dst_ld * es))
            top ^= np.uint8(0x80)
        self.launches += 1
        return 0

    def dab_adjoint_box(self, ctx, dtype, dst, dst_ld, src, src_ld, rows, cols):
        if int(dtype) not in (6, 7):
            return 6                                               # DAB_ERR_UNSUPPORTED: not a complex dtype
        return self.dab_transpose_box(ctx, 8 if int(dtype) == 6 else 16, dst, dst_ld, src, src_ld, rows, cols, conj=True)

    def dab_accumulate_stack(self, ctx, dtype, y, n, beta, alpha, stack, stride, count):
        dt, n = _NP[int(dtype)], int(n)
        yv = _view(y, n, dt)
        b, a = _view(beta, 1, dt)[0], _view(alpha, 1, dt)[0]
        with np.errstate(all="ignore"):
            acc = (yv * b) if b != 1 else yv.copy()
            if b == 0:
                acc = np.zeros(n, dtype=dt)
            for j in range(int(count)):
                t = _view(_addr(stack) + j * int(stride) * dt.itemsize, n, dt)
                acc = acc + (t * a if a != 1 else t)
            yv[:] = acc
        self.launches += 1
        return 0

    # -- dab_gather_box: per dimension the element offset of coordinate t is t * stride (possibly negative) or table[t]
    def dab_gather_box(self, ctx, elem_bytes, ndim, dst, dst_strides, dst_index, src, src_strides, src_index, extent):
        nd = int(ndim)
        if not 1 <= nd <= 8:
            return 6                                               # DAB_ERR_UNSUPPORTED
        ext = [int(extent[k]) for k in range(nd)]
        if min(ext) == 0:
            return 0
        if int(elem_bytes) not in _UNIT:
            return 2
        dt = _UNIT[int(elem_bytes)]

        def offsets(strides, index):
            total = np.zeros((), dtype=np.int64)
            for k in range(nd):
                tab = index[k] if index is not None and index else None
                o = _view(tab, ext[k], np.int64).copy() if tab else np.arange(ext[k], dtype=np.int64) * int(strides[k])
                total = total[..., None] + o                         # C-order outer sum; flattened consistently for dst and src below
            return total.reshape(-1)

        do, so = offsets(dst_strides, dst_index), offsets(src_strides, src_index)
        es = int(elem_bytes)
        dbase, sbase = _addr(dst), _addr(src)
        lo_d, lo_s = int(do.min()), int(so.min())
        dv = _view(dbase + lo_d * es, int(do.max()) - lo_d + 1, dt)
        sv = _view(sbase + lo_s * es, int(so.max()) - lo_s + 1, dt)
        dv[do - lo_d] = sv[so - lo_s]
        self.launches += 1
        return 0

    # -- K11
    def dab_sort(self, ctx, dtype, inp, out, tmp, n):
        n, u = int(n), _utype(dtype)
        src, dst, t = _addr(inp), _addr(out), _addr(tmp)
        if n and n <= 1024 and src == dst and not t:
            return 2                                               # DAB_ERR_ARG: the in-place rank sort needs tmp
        if n > 1024 and (not t or t == src or t == dst):
            return 2                                               # DAB_ERR_ARG: tmp must be a distinct buffer
        if n >= 0xFFFFF000:
            return 6                                               # DAB_ERR_UNSUPPORTED
        if n:
            raw = _view(inp, n, u).copy()
            _view(out, n, u)[:] = radix_dec(np.sort(radix_enc(raw, dtype), kind="stable"), dtype)
            self.launches += 1
        return 0

    def dab_sort_by_key_scratch_bytes(self, key_dtype, n, out):
        rounds = 2 if key_dtype in (F64, I64) else 1
        out._obj.value = (2 + rounds) * ((int(n) * 8 + 255) & ~255)
        return 0

    def dab_sort_by_key(self, ctx, key_dtype, keys, val_bytes, vals, vals_out, scratch, scratch_bytes, n):
        n = int(n)
        if n == 0:
            return 0
        if n >= 0xFFFFF000:
            return 6                                            # DAB_ERR_UNSUPPORTED
        need = C.c_size_t()
        self.dab_sort_by_key_scratch_bytes(key_dtype, n, C.byref(need))
        assert int(scratch_bytes) >= need.value and _addr(scratch) % 16 == 0 and _addr(vals) != _addr(vals_out)
        ws = (n * 8 + 255) & ~255
        base = _addr(scratch)
        words, tmp, s1, s2 = (base + k * ws for k in range(4))
        e = by_radix_key(_view(keys, n, _utype(key_dtype)), key_dtype).astype(np.uint64)
        pos = np.arange(n, dtype=np.uint64)

        def pack(h):                                            # sortby_pack_kernel
            _view(words, n, np.uint64)[:] = ((h << np.uint64(32)) | pos) ^ SIGN64

        if key_dtype in (F32, I32):
            pack(e)
            self.dab_sort(ctx, I64, words, s1, tmp, n)
            perm = (_view(s1, n, np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)
        else:
            pack(e & np.uint64(0xFFFFFFFF))
            self.dab_sort(ctx, I64, words, s1, tmp, n)
            p1 = (_view(s1, n, np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)
            pack(e[p1] >> np.uint64(32))
            self.dab_sort(ctx, I64, words, s2, tmp, n)
            perm = p1[(_view(s2, n, np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)]
        vt = {4: np.uint32, 8: np.uint64}[int(val_bytes)]
        _view(vals_out, n, vt)[:] = _view(vals, n, vt)[perm]    # sortby_gather_kernel
        self.launches += 2
        return 0

    # -- whole-chunk reductions: minimum / maximum of a chunk exact (NaN-propagating, +0.0 > -0.0, like Base);
    #    the host-only entry points (result dtype table, ordered fold) are the REAL library's -- they need no GPU
    def _real(self):
        if getattr(self, "_real_lib", None) is None:
            from darray_b200 import _lib as real
            L = C.CDLL(real.SO_PATH)
            L.dab_reduce_result_dtype.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
            L.dab_combine_ordered.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]
            self._real_lib = L
        return self._real_lib

    def dab_reduce_result_dtype(self, dtype, op, mapc, out):
        return self._real().dab_reduce_result_dtype(int(dtype), int(op), int(mapc), C.cast(C.c_void_p(_addr(out)), C.POINTER(C.c_int32)))

    def dab_combine_ordered(self, rdt, op, partials, p, out):
        return self._real().dab_combine_ordered(int(rdt), int(op), C.c_void_p(_addr(partials)), int(p), C.c_void_p(_addr(out)))

    def _reduce(self, dtype, op, mapc, param, x, n, out):
        """dab_reduce: op in SUM PROD MAX MIN ALL ANY COUNT (0..6), map in ID ABS ABS2 NEG (0..3) or a predicate (16..23, scalar parameter).
        Sums and products in the wide carrier (order-free stand-in for the kernel's tree: compared at tolerance by the tests that use it),
        max / min exact (NaN-propagating, +0.0 > -0.0, like Base)."""
        op, mapc = int(op), int(mapc)
        dt = _NP[int(dtype)] if int(dtype) != U8 else np.dtype(np.bool_)
        v = _view(x, int(n), dt)
        if op == 7:                                               # EXTREMA: [min, max] in the element type, one pass
            with np.errstate(all="ignore"):
                pair = np.asarray([jl_extreme(v, 0, False), jl_extreme(v, 0, True)], dtype=dt)
            slot = np.zeros(16, dtype=np.uint8)
            slot[:2 * dt.itemsize] = pair.view(np.uint8)
            C.memmove(_addr(out), slot.ctypes.data, 16)
            self.launches += 1
            return 0
        with np.errstate(all="ignore"):
            if mapc >= 16:
                q = _view(param, 1, dt)[0] if param is not None and _addr(param) else None
                m = {16: lambda: v == q, 17: lambda: v != q, 18: lambda: v < q, 19: lambda: v <= q, 20: lambda: v > q, 21: lambda: v >= q,
                     22: lambda: np.isnan(v), 23: lambda: v != 0}[mapc]()
            else:
                m = {0: lambda: v, 1: lambda: np.abs(v), 2: lambda: v * v, 3: lambda: -v}[mapc]()
            code = C.c_int32()
            assert self._real().dab_reduce_result_dtype(int(dtype), op, mapc, C.byref(code)) == 0
            rdt = np.dtype(np.int64) if code.value == I64 else _NP[code.value]
            wide = np.float64 if rdt.kind == "f" else np.int64
            if op in (0, 1):
                acc = (np.sum if op == 0 else np.prod)(m.astype(wide))
            elif op in (2, 3):
                acc = jl_extreme(m, 0, op == 2)
            else:
                acc = {4: lambda: int(np.all(m)), 5: lambda: int(np.any(m)), 6: lambda: int(np.count_nonzero(m))}[op]()
        slot = np.zeros(16, dtype=np.uint8)
        slot[:rdt.itemsize] = np.asarray([acc], dtype=rdt).view(np.uint8)
        slot[8:16] = np.asarray([acc], dtype=wide if op in (0, 1) else (rdt if rdt.itemsize == 8 else wide)).view(np.uint8)[:8]
        C.memmove(_addr(out), slot.ctypes.data, 16)
        self.launches += 1
        return 0

    def dab_reduce(self, ctx, dtype, op, mapc, param, x, n, out):
        return self._reduce(dtype, op, mapc, param, x, n, out)

    def dab_mapreduce_all(self, ctx, dtype, op, mapc, param, x, n, out_host):
        return self._reduce(dtype, op, mapc, param, x, n, out_host)

    dab_reduce_host = dab_mapreduce_all

    def dab_rand_u01(self, ctx, dtype, x, n, seed, offset):
        from oracle import darray_oracle as orc
        dt = _NP[int(dtype)]
        _view(x, int(n), dt)[:] = orc.rand_u01(int(seed), int(offset), int(n), dt)
        self.launches += 1
        return 0

    # -- fused map + reduce of a traced expression: the refusals of dab_mapreduce_expr with its status codes, then the result slot as
    #    mr_spec lays it out (word 0 the result, word 1 the carrier; a 16-byte carrier fills the slot)
    def dab_mapreduce_expr(self, ctx, src, val_dtype, op, n, nargs, dts, ptrs, scal, out):
        val, op, n, nargs = int(val_dtype), int(op), int(n), int(nargs)
        if not src or not _addr(out) or not 1 <= nargs <= 8 or dts is None or ptrs is None or scal is None:
            return 2                                               # DAB_ERR_ARG
        if val not in range(8):
            return 2
        if n == 0:
            return 3                                               # DAB_ERR_EMPTY
        if not _mr_served(val, op):
            return 6                                               # DAB_ERR_UNSUPPORTED
        for k in range(nargs):
            if int(dts[k]) not in _ELEM or (not ptrs[k] and int(dts[k]) == 7):
                return 2                                           # no such element type; a ComplexF64 scalar does not fit 8 bytes
        if any(ptrs[k] and _addr(ptrs[k]) % (4 * _ELEM[int(dts[k])].itemsize) for k in range(nargs)):
            return 6                                               # arrays must be aligned to 4 elements
        expr = self.exprs[src]
        args = []
        for k in range(nargs):
            dt = _ELEM[int(dts[k])]
            if ptrs[k]:
                args.append(_view(ptrs[k], n, dt).copy())
            else:
                args.append(np.frombuffer(int(scal[k]).to_bytes(8, "little")[:dt.itemsize], dtype=dt)[0])
        self.launches += 2
        if val == 5:                                               # Int128: Python integers wrapped to 128 bits
            vals = [int(v) for v in np.broadcast_to(eval_expr(expr, args), (n,))]
            mask = (1 << 128) - 1
            acc = vals[0]
            for v in vals[1:]:
                acc = {0: acc + v, 1: acc * v, 2: max(acc, v), 3: min(acc, v)}[op]
                acc &= mask
                acc = acc - (1 << 128) if acc >> 127 else acc
            C.memmove(_addr(out), (acc & mask).to_bytes(16, "little"), 16)
            return 0
        v = np.broadcast_to(np.asarray(eval_expr(expr, args)), (n,)).astype(_ELEM[val])
        slot = np.zeros(16, dtype=np.uint8)
        with np.errstate(all="ignore"):
            if val == U8:                                          # Bool values: sum / count / all / any, the count is the carrier
                c = int(np.count_nonzero(v))
                res = {0: c, 6: c, 4: int(c == n), 5: int(c != 0)}[op]
                slot.view(np.int64)[:] = [res, c]
            elif val in (6, 7):                                    # complex: the sum or product in ComplexF64, rounded once
                w = v.astype(np.complex128)
                acc = complex(w.real.sum(), w.imag.sum()) if op == 0 else complex(np.prod(w))
                R = np.float32 if val == 6 else np.float64
                pair = np.asarray([acc.real, acc.imag], dtype=np.float64).astype(R)
                slot[:pair.nbytes] = pair.view(np.uint8)
            elif v.dtype.kind == "f":
                if op in (0, 1):                                   # exact fp64 carrier, the result rounded once
                    acc = v.astype(np.float64).sum() if op == 0 else v.astype(np.float64).prod()
                    slot[:v.itemsize] = np.asarray([acc], dtype=v.dtype).view(np.uint8)
                    slot[8:] = np.asarray([acc], dtype=np.float64).view(np.uint8)
                else:                                              # Julia's max / min; the carrier is the value type
                    r = np.asarray([jl_extreme(v, 0, op == 2)], dtype=v.dtype).view(np.uint8)
                    slot[:v.itemsize] = slot[8:8 + v.itemsize] = r
            else:
                if op in (0, 1):                                   # Int32 widened, Int64 wrapping mod 2^64
                    w = v.astype(np.int64)
                    slot.view(np.int64)[:] = w.sum(dtype=np.int64) if op == 0 else w.prod(dtype=np.int64)
                else:
                    r = np.asarray([v.max() if op == 2 else v.min()], dtype=v.dtype).view(np.uint8)
                    slot[:v.itemsize] = slot[8:8 + v.itemsize] = r
        C.memmove(_addr(out), slot.ctypes.data, 16)
        return 0

    def dab_sorted_split(self, ctx, dtype, sorted_p, n, bounds_host, nb, counts):
        n, nb, u = int(n), int(nb), _utype(dtype)
        raw = _view(sorted_p, n, u)
        enc = radix_enc(raw, dtype)
        b = _view(bounds_host, nb, u).copy()
        isf = dtype in (F32, F64)
        absmask = (u(0x7FFFFFFF) if dtype == F32 else u(0x7FFFFFFFFFFFFFFF)) if isf else None
        inf = (u(0x7F800000) if dtype == F32 else u(0x7FF0000000000000)) if isf else None
        for t in range(nb):
            braw = b[t]
            if isf and (braw & absmask) > inf:                  # x > NaN is never true
                counts[t] = n
                continue
            if isf and (braw & absmask) == 0:
                braw = u(0)                                     # -0.0 bounds like +0.0
            kb = radix_enc(np.array([braw], dtype=u), dtype)[0]
            lo = int(np.searchsorted(enc, kb, side="right"))
            rest_nan = isf and lo < n and (raw[lo] & absmask) > inf
            counts[t] = n if rest_nan else lo
        self.launches += 1
        return 0


_ELEM = {**_NP, U8: np.dtype(np.bool_), 6: np.dtype(np.complex64), 7: np.dtype(np.complex128)}   # array element types


def _mr_served(val: int, op: int) -> bool:
    """mr_spec of dab_jit.cu: which (value type, op) dab_mapreduce_expr serves."""
    if val == 5:
        return op in (0, 1, 2, 3)
    if val in (6, 7):
        return op in (0, 1)
    if val == U8:
        return op in (0, 4, 5, 6)
    return op in (0, 1, 2, 3)


def jl_extreme(m, axis, is_max):
    """Base's maximum / minimum along ``axis``: any NaN gives NaN, otherwise the extreme value; a zero result is +0.0 for max when
    a +0.0 is present and -0.0 for min when a -0.0 is present.  tests/test_gpu_reduce_exact.py keeps its own copy on purpose: that
    one is the reference the kernels are checked against, this one stands in for the kernels."""
    m = np.asarray(m)
    if m.dtype.kind != "f":
        return (np.max if is_max else np.min)(m, axis=axis)
    nan = np.isnan(m)
    r = (np.max if is_max else np.min)(np.where(nan, -np.inf if is_max else np.inf, m), axis=axis)
    has = ((m == 0) & (np.signbit(m) != is_max)).any(axis=axis)
    win, lose = (m.dtype.type(0.0), m.dtype.type(-0.0)) if is_max else (m.dtype.type(-0.0), m.dtype.type(0.0))
    r = np.where(r == 0, np.where(has, win, lose), r)
    return np.where(nan.any(axis=axis), m.dtype.type(np.nan), r).astype(m.dtype)


# ---- NumPy interpreter of a traced expression (stands in for dab_unary / dab_affine / dab_broadcast_expr) ---------------------
def eval_expr(e, args):
    from darray_b200 import _broadcast as bc
    npt = bc._NPT
    if e.op == "arg":
        return args[e.val]
    if e.op == "const":
        return _wrap128(int(e.val)) if e.jt == "i128" else npt[e.jt].type(e.val)
    if e.jt == "i128" or any(x.jt == "i128" for x in e.args):
        return _eval_i128(e, args)
    if e.op == "convert":
        return np.asarray(eval_expr(e.args[0], args)).astype(npt[e.jt])
    a = [eval_expr(x, args) for x in e.args]
    with np.errstate(all="ignore"):
        if e.op == "complex":
            return _pack(np.asarray(a[0]), np.asarray(a[1])).astype(npt[e.jt])
        if e.op in ("conj", "real", "imag"):
            return {"conj": np.conj, "real": np.real, "imag": np.imag}[e.op](np.asarray(a[0])).astype(npt[e.jt])
        if e.op in ("add", "sub", "mul", "div") and len({np.iscomplexobj(v) for v in a}) == 2:
            return _mixed_complex(e.op, a[0], a[1]).astype(npt[e.jt])
        if e.op == "ifelse":
            return np.where(a[0], a[1], a[2])
        if e.op in ("add", "sub", "mul", "div", "rem", "mod", "max", "min", "and", "or", "xor", "lt", "le", "gt", "ge", "eq", "ne", "idiv"):
            r = jl.vbin(e.op, a[0], a[1])
        elif e.op == "pow":
            r = np.power(a[0], a[1])
        elif e.op == "m_copysign":
            r = np.copysign(a[0], a[1])
        elif e.op in ("m_eq", "m_ne", "m_lt", "m_le", "m_gt", "m_ge"):
            r = jl.vcmp_exact(e.op[2:], a[0], a[1])
        elif e.op == "m_powi":
            r = np.vectorize(lambda x, n: jl.pow_f32_int(np.float32(x), int(n)), otypes=[np.float32])(a[0], a[1])
        elif e.op in ("x_shl", "x_shr"):
            r = np.vectorize(lambda x, n: jl_shift(int(x), int(n), 8 * npt[e.jt].itemsize, e.op == "x_shl"), otypes=[npt[e.jt]])(a[0], a[1])
        elif e.op in ("abs", "abs2", "neg", "sign", "inv", "floor", "ceil", "x_trunc", "x_round"):
            r = jl.vun(e.op.removeprefix("x_"), np.asarray(a[0]))
        else:
            one = {"sqrt": np.sqrt, "sin": np.sin, "cos": np.cos, "tan": np.tan, "exp": np.exp, "log": np.log,
                   "tanh": np.tanh, "isnan": np.isnan, "isinf": np.isinf, "isfinite": np.isfinite, "exp2": np.exp2, "log2": np.log2,
                   "log10": np.log10, "sinh": np.sinh, "cosh": np.cosh, "atan": np.arctan, "asin": np.arcsin, "acos": np.arccos,
                   "expm1": np.expm1, "log1p": np.log1p, "cbrt": np.cbrt, "x_asinh": np.arcsinh, "x_acosh": np.arccosh, "x_atanh": np.arctanh,
                   "x_exp10": lambda x: np.power(x.dtype.type(10), x),
                   "x_sinpi": lambda x: np.sin(np.pi * np.where(x > 0.5, 1.0 - x.astype(np.float64), x.astype(np.float64))),
                   "x_cospi": lambda x: np.where(x > 0.25, np.sin(np.pi * (0.5 - x.astype(np.float64))), np.cos(np.pi * x.astype(np.float64)))}
            if e.op in ("x_erf", "x_erfc", "x_erfinv", "x_erfcinv", "x_erfcx", "x_gamma", "x_loggamma"):
                import scipy.special as sp
                one.update({"x_erf": sp.erf, "x_erfc": sp.erfc, "x_erfinv": sp.erfinv, "x_erfcinv": sp.erfcinv, "x_erfcx": sp.erfcx,
                            "x_gamma": sp.gamma, "x_loggamma": sp.gammaln})
            r = one[e.op](np.asarray(a[0]))
        return np.asarray(r).astype(npt[e.jt])


def _mixed_complex(op, a, b):
    """Julia's methods between a real and a complex operand: the real one is not promoted to complex (x*z = Complex(x*zr, x*zi), ...)."""
    a, b = np.asarray(a), np.asarray(b)
    if np.iscomplexobj(a):
        zr, zi, x = a.real, a.imag, b
        re, im = {"add": (zr + x, zi), "sub": (zr - x, zi), "mul": (zr * x, zi * x), "div": (zr / x, zi / x)}[op]
    else:
        x, zr, zi = a, b.real, b.imag
        re, im = {"add": (x + zr, zi), "sub": (x - zr, -zi), "mul": (x * zr, x * zi)}[op]
    return _pack(re, im)


def _pack(re, im):
    """Complex values from their components (re + 1j*im would turn an infinite component into NaNs)."""
    out = np.empty(np.broadcast(re, im).shape, dtype=np.result_type(re, im, np.complex64))
    out.real, out.imag = re, im
    return out


def jl_shift(x: int, n: int, bits: int, left: bool) -> int:
    """Julia's ``x << n`` (left) / ``x >> n`` on a ``bits``-wide signed integer: a negative count shifts the other way, shifting out every
    bit gives 0 (left) or the sign fill (right)."""
    if n < 0:
        left, n = not left, -n
    if left:
        v = 0 if n >= bits else (x << n) & ((1 << bits) - 1)
        return v - (1 << bits) if v >> (bits - 1) else v
    return (-1 if x < 0 else 0) if n >= bits else x >> n


def _wrap128(v: int) -> int:
    v &= (1 << 128) - 1
    return v - (1 << 128) if v >> 127 else v


def _eval_i128(e, args):
    """Int128 sub-expressions on object arrays of Python ints, wrapped to 128 bits after every operation."""
    import operator
    if e.op == "const":
        return _wrap128(int(e.val))
    a = [eval_expr(x, args) for x in e.args]
    if e.op == "convert":
        if e.jt == "i128":
            return np.vectorize(lambda v: _wrap128(int(v)), otypes=[object])(a[0])
        from darray_b200 import _broadcast as bc
        return np.vectorize(float, otypes=[np.float64])(a[0]).astype(bc._NPT[e.jt])   # Int128 -> float
    if e.op in ("lt", "le", "gt", "ge", "eq", "ne"):
        return np.vectorize(getattr(operator, e.op), otypes=[bool])(a[0], a[1])
    two = {"add": operator.add, "sub": operator.sub, "mul": operator.mul, "max": max, "min": min, "and": operator.and_, "or": operator.or_,
           "xor": operator.xor}
    if e.op in two:
        return np.vectorize(lambda x, y: _wrap128(two[e.op](int(x), int(y))), otypes=[object])(a[0], a[1])
    one = {"neg": operator.neg, "abs": abs, "abs2": lambda x: x * x}
    return np.vectorize(lambda x: _wrap128(one[e.op](int(x))), otypes=[object])(a[0])


def run_local(rt, expr, out, largs):
    """A NumPy stand-in for ``_broadcast.run_local`` (dense same-shape arguments and scalars).  No longer installed by the fixture: the REAL
    run_local now runs against the emulated elementwise entry points; kept for ad-hoc use."""
    if out.size == 0:
        return
    vals = []
    for a in largs:
        if a.arr is not None:
            assert a.arr.size == out.size
            vals.append(_view(a.arr.ptr, a.arr.size, a.arr.dtype).copy())
        else:
            vals.append(a.scalar)
    r = np.broadcast_to(np.asarray(eval_expr(expr, vals)), (out.size,)).astype(out.dtype)
    _view(out.ptr, out.size, out.dtype)[:] = r
