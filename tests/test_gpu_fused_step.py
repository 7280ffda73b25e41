"""The deferred dab_affine and the fused map-store-reduce kernel that consumes it.

``y .= a.*x .+ b`` followed by a reduction of y runs as ONE kernel (reads x, stores y, reduces y).  These tests pin that
(1) the fused result slot and y are byte-identical to the unfused two-kernel run, (2) fusion really happens (launch counts),
(3) every other entry point still sees the finished y -- the deferred kernel is queued before anything else touches the stream --
and (4) the cases that must not fuse do not.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import darray_oracle as orc

pytestmark = pytest.mark.gpu

F32 = np.float32
DTYPES = [np.float32, np.float64, np.int32, np.int64]
SIZES = [1, 5, 4097, (1 << 15) + 3, (1 << 22) + 13]


def _lib():
    from darray_b200 import _lib
    return _lib


def _coefs(dtype):
    if np.dtype(dtype).kind == "f":
        return dtype(1.5), dtype(-0.5)
    return dtype(3), dtype(-7)


def _input(dtype, n, seed=0):
    rng = np.random.default_rng(n + seed)
    if np.dtype(dtype).kind == "f":
        return (1 + rng.uniform(-1e-3, 1e-3, n)).astype(dtype)   # products stay finite for a while, sums are well conditioned
    return rng.integers(-1000, 1000, n).astype(dtype)


def _affine(ctx, code, y, x, a, b, n):
    av, bv = np.asarray(a), np.asarray(b)
    _lib().call("dab_affine", ctx, code, C.c_void_p(y), C.c_void_p(x), C.c_void_p(av.ctypes.data), C.c_void_p(bv.ctypes.data), n)


def _reduce_host(ctx, code, op, ptr, n, mapc=None):
    L = _lib()
    out = np.zeros(2, dtype=np.uint64)
    L.call("dab_reduce_host", ctx, code, op, L.MAP_ID if mapc is None else mapc, None, C.c_void_p(ptr), n, C.c_void_p(out.ctypes.data))
    return out.tobytes()


def _launches(ctx):
    n = C.c_uint64(0)
    _lib().call("dab_launch_count", ctx, C.byref(n))
    return int(n.value)


def _d2h(ctx, ptr, n, dtype):
    out = np.empty(n, dtype=dtype)
    _lib().call("dab_d2h", ctx, C.c_void_p(out.ctypes.data), C.c_void_p(ptr), n * np.dtype(dtype).itemsize)
    _lib().call("dab_sync", ctx)
    return out


def _fill(ctx, code, ptr, n, value):
    v = np.asarray(value)
    _lib().call("dab_fill", ctx, code, C.c_void_p(ptr), n, C.c_void_p(v.ctypes.data))


def _sentinel(dtype):
    return dtype(7)


# ---------------------------------------------------------------------------------------------- fused == unfused, C ABI
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_equals_unfused(dab, rt1, dtype, n, off):
    L = _lib()
    ctx, code, es = rt1.ctx, dab.dab_dtype(dtype), np.dtype(dtype).itemsize
    a, b = _coefs(dtype)
    x = _input(dtype, n)
    want = orc.affine_unfused(a, x, b)
    dx = dab.B200Array.from_numpy(rt1, np.concatenate([x[:1], x]) if off else x)
    ya, yb = dab.B200Array.empty(rt1, (n + off,), dtype), dab.B200Array.empty(rt1, (n + off,), dtype)
    px, pa, pb = dx.ptr + off * es, ya.ptr + off * es, yb.ptr + off * es
    for op in (L.SUM, L.PROD, L.MAX, L.MIN):
        _fill(ctx, code, ya.ptr, n + off, _sentinel(dtype))
        _fill(ctx, code, yb.ptr, n + off, _sentinel(dtype))
        l0 = _launches(ctx)
        _affine(ctx, code, pa, px, a, b, n)
        slot_a = _reduce_host(ctx, code, op, pa, n)            # path A: the reduction consumes the deferred affine
        l1 = _launches(ctx)
        _affine(ctx, code, pb, px, a, b, n)
        L.call("dab_sync", ctx)                                 # path B: the sync queues the affine first
        slot_b = _reduce_host(ctx, code, op, pb, n)
        l2 = _launches(ctx)
        assert (l1 - l0, l2 - l1) == (1, 2), (op, l1 - l0, l2 - l1)
        assert slot_a == slot_b, (op, np.frombuffer(slot_a, np.uint64), np.frombuffer(slot_b, np.uint64))
        got_a, got_b = _d2h(ctx, pa, n, dtype), _d2h(ctx, pb, n, dtype)
        assert got_a.tobytes() == got_b.tobytes() == want.tobytes(), op


def test_fused_in_place(dab, rt1):
    """map!(f, d, d) then sum(d) through the C ABI: x == y."""
    L = _lib()
    n = (1 << 20) + 7
    x = _input(F32, n, 1)
    a, b = _coefs(F32)
    d1, d2 = dab.B200Array.from_numpy(rt1, x), dab.B200Array.from_numpy(rt1, x)
    l0 = _launches(rt1.ctx)
    _affine(rt1.ctx, L.F32, d1.ptr, d1.ptr, a, b, n)
    s1 = _reduce_host(rt1.ctx, L.F32, L.SUM, d1.ptr, n)
    assert _launches(rt1.ctx) - l0 == 1
    _affine(rt1.ctx, L.F32, d2.ptr, d2.ptr, a, b, n)
    L.call("dab_sync", rt1.ctx)
    assert s1 == _reduce_host(rt1.ctx, L.F32, L.SUM, d2.ptr, n)
    assert d1.to_numpy().tobytes() == d2.to_numpy().tobytes() == orc.affine_unfused(a, x, b).tobytes()


# ---------------------------------------------------------------------------------------------- public API
def test_public_api_fuses(dab, rt1):
    n = (1 << 20) + 3
    x = orc.rand_u01(5, 0, n)
    a, b = F32(1.5), F32(0.25)
    f = lambda v: a * v + b  # noqa: E731
    want = orc.affine_unfused(a, x, b)
    d = dab.distribute(x)
    y = dab.similar(d)
    results = {}
    for name, red in (("sum", dab.sum), ("maximum", dab.maximum)):
        l0 = rt1.launches()
        dab.broadcast_into(y, f, d)
        r = red(y)
        assert rt1.launches() - l0 == 1, name
        assert dab.to_array(y).tobytes() == want.tobytes()
        dab.broadcast_into(y, f, d)
        rt1.launches()                      # flushes the deferred affine without a sync: the unfused launch sequence
        r_ref = red(y)
        assert np.asarray(r).tobytes() == np.asarray(r_ref).tobytes(), (name, r, r_ref)
        results[name] = r
    assert results["maximum"] == want.max()
    e = dab.distribute(x)
    l0 = rt1.launches()
    dab.map_inplace(f, e, e)
    s = dab.sum(e)
    assert rt1.launches() - l0 == 1
    assert np.asarray(s).tobytes() == np.asarray(results["sum"]).tobytes()
    assert dab.to_array(e).tobytes() == want.tobytes()


# ---------------------------------------------------------------------------------------------- ordering
@pytest.fixture()
def step(dab, rt1):
    """x (n Float32), a y pre-filled with a sentinel, and the expected y = a*x + b."""
    n = (1 << 16) + 5
    x = _input(F32, n, 2)
    a, b = _coefs(F32)
    dx = dab.B200Array.from_numpy(rt1, x)
    dy = dab.B200Array.empty(rt1, (n,), F32)
    _fill(rt1.ctx, _lib().F32, dy.ptr, n, _sentinel(F32))
    return dict(n=n, x=x, a=a, b=b, dx=dx, dy=dy, want=orc.affine_unfused(a, x, b))


def _defer(rt1, s):
    _affine(rt1.ctx, _lib().F32, s["dy"].ptr, s["dx"].ptr, s["a"], s["b"], s["n"])


def test_order_copies(dab, rt1, step):
    L, s, n = _lib(), step, step["n"]
    _defer(rt1, s)
    assert _d2h(rt1.ctx, s["dy"].ptr, n, F32).tobytes() == s["want"].tobytes()          # dab_d2h
    _fill(rt1.ctx, L.F32, s["dy"].ptr, n, _sentinel(F32))
    z = dab.B200Array.empty(rt1, (n,), F32)
    _defer(rt1, s)
    L.call("dab_d2d", rt1.ctx, C.c_void_p(z.ptr), C.c_void_p(s["dy"].ptr), 4 * n)        # dab_d2d
    assert z.to_numpy().tobytes() == s["want"].tobytes()
    _fill(rt1.ctx, L.F32, s["dy"].ptr, n, _sentinel(F32))
    _fill(rt1.ctx, L.F32, z.ptr, n, F32(0))
    _defer(rt1, s)
    zero = L.sz4((0, 0, 0, 0))
    L.call("dab_copy_box", rt1.ctx, 4, C.c_void_p(z.ptr), L.sz4((n,)), zero, C.c_void_p(s["dy"].ptr), L.sz4((n,)), zero,
           L.sz4((n,)))                                                                   # dab_copy_box
    assert z.to_numpy().tobytes() == s["want"].tobytes()
    _fill(rt1.ctx, L.F32, s["dy"].ptr, n, _sentinel(F32))
    _defer(rt1, s)
    _affine(rt1.ctx, L.F32, z.ptr, s["dy"].ptr, s["a"], s["b"], n)                        # a chained dab_affine that reads y
    assert z.to_numpy().tobytes() == orc.affine_unfused(s["a"], s["want"], s["b"]).tobytes()


def test_order_reductions_that_do_not_fuse(dab, rt1, step):
    L, s, n, ctx = _lib(), step, step["n"], rt1.ctx
    want_x = _reduce_host(ctx, L.F32, L.SUM, s["dx"].ptr, n)
    want_d = dab.B200Array.from_numpy(rt1, s["want"])
    want_short = _reduce_host(ctx, L.F32, L.SUM, want_d.ptr, n - 1)
    want_abs = _reduce_host(ctx, L.F32, L.SUM, want_d.ptr, n, L.MAP_ABS)
    cases = [(s["dx"].ptr, n, None, want_x), (s["dy"].ptr, n - 1, None, want_short), (s["dy"].ptr, n, L.MAP_ABS, want_abs)]
    for ptr, m, mapc, want in cases:
        _fill(ctx, L.F32, s["dy"].ptr, n, _sentinel(F32))
        l0 = _launches(ctx)
        _defer(rt1, s)
        got = _reduce_host(ctx, L.F32, L.SUM, ptr, m, mapc)
        assert _launches(ctx) - l0 == 2, (m, mapc)
        assert got == want, (m, mapc)
        assert s["dy"].to_numpy().tobytes() == s["want"].tobytes()
        assert s["dx"].to_numpy().tobytes() == s["x"].tobytes()


def test_order_mapreduce_expr(dab, rt1):
    n = (1 << 16) + 5
    x = orc.rand_u01(11, 0, n)
    a, b = F32(1.5), F32(0.25)
    d = dab.distribute(x)
    y = dab.similar(d)
    g = lambda v: v * v + F32(1)  # noqa: E731  (a general closure: one NVRTC map-reduce kernel, dab_mapreduce_expr)
    dab.broadcast_into(y, lambda v: a * v + b, d)
    rt1.sync()
    want = dab.mapreduce(g, "max", y)
    _fill(rt1.ctx, _lib().F32, dab.localpart(y).ptr, n, _sentinel(F32))
    dab.broadcast_into(y, lambda v: a * v + b, d)
    got = dab.mapreduce(g, "max", y)
    assert np.asarray(got).tobytes() == np.asarray(want).tobytes()
    w = orc.affine_unfused(a, x, b)
    assert got == (w * w + F32(1)).max()


def test_order_free_and_reuse(dab, rt1, step):
    L, s, n = _lib(), step, step["n"]
    _defer(rt1, s)
    s["dx"].free()                                   # the block goes back to the allocator's cache ...
    z = dab.B200Array.empty(rt1, (n,), F32)          # ... and may come straight back: it must not be overwritten before the affine ran
    z.copy_from_host(np.full(n, F32(-3)))
    assert s["dy"].to_numpy().tobytes() == s["want"].tobytes()
    assert z.to_numpy().tobytes() == np.full(n, F32(-3)).tobytes()


def test_order_event_record(dab, rt1):
    """An event recorded after the deferred affine completes after it: the elapsed time covers a 256 MiB stream."""
    L = _lib()
    n = 1 << 26
    dx = dab.B200Array.empty(rt1, (n,), F32)
    dy = dab.B200Array.empty(rt1, (n,), F32)
    _fill(rt1.ctx, L.F32, dx.ptr, n, F32(2))
    rt1.sync()
    e0, e1 = rt1.event(), rt1.event()
    try:
        rt1.record(e0)
        _affine(rt1.ctx, L.F32, dy.ptr, dx.ptr, F32(1.5), F32(0.25), n)
        rt1.record(e1)
        ms = rt1.elapsed_ms(e0, e1)
        assert ms > 0.05, ms                         # 512 MB through HBM: ~0.2 ms; an empty interval is a few microseconds
        got = _d2h(rt1.ctx, dy.ptr, 1 << 10, F32)
        assert np.all(got == F32(3.25))
    finally:
        rt1.event_destroy(e0)
        rt1.event_destroy(e1)


# ---------------------------------------------------------------------------------------------- no fusion where it does not apply
def test_no_fusion_mismatched_alignment(dab, rt1):
    L = _lib()
    n = (1 << 18) + 1
    x = _input(F32, n + 1, 3)
    a, b = _coefs(F32)
    dx = dab.B200Array.from_numpy(rt1, x)
    dy = dab.B200Array.empty(rt1, (n,), F32)
    l0 = _launches(rt1.ctx)
    _affine(rt1.ctx, L.F32, dy.ptr, dx.ptr + 4, a, b, n)            # x one element off, y aligned: the scalar kernel, launched at once
    got = _reduce_host(rt1.ctx, L.F32, L.MAX, dy.ptr, n)
    assert _launches(rt1.ctx) - l0 == 2
    want = orc.affine_unfused(a, x[1:], b)
    assert dy.to_numpy().tobytes() == want.tobytes()
    assert np.frombuffer(got[:4], F32)[0] == want.max()


def test_no_fusion_with_tma_variant(dab, rt1):
    L = _lib()
    n = 8192 * 64                                                    # whole 32 KiB tiles: one TMA launch, no ragged tail
    x = _input(F32, n, 4)
    a, b = _coefs(F32)
    dx = dab.B200Array.from_numpy(rt1, x)
    dy = dab.B200Array.empty(rt1, (n,), F32)
    want_d = dab.B200Array.from_numpy(rt1, orc.affine_unfused(a, x, b))
    want = _reduce_host(rt1.ctx, L.F32, L.SUM, want_d.ptr, n)
    rt1.set_option("ew_tma", 1)
    try:
        l0 = _launches(rt1.ctx)
        _affine(rt1.ctx, L.F32, dy.ptr, dx.ptr, a, b, n)
        got = _reduce_host(rt1.ctx, L.F32, L.SUM, dy.ptr, n)
        assert _launches(rt1.ctx) - l0 == 2
    finally:
        rt1.set_option("ew_tma", 0)
    assert got == want
    assert dy.to_numpy().tobytes() == orc.affine_unfused(a, x, b).tobytes()


def test_no_fusion_after_dab_stream(dab, rt1):
    """dab_stream hands out the raw stream: from then on every dab_affine is queued when it is called.  A ctx of its own, so the
    switch does not outlive this test."""
    L = _lib()
    ctx = C.c_void_p()
    L.call("dab_init", 0, C.byref(ctx))
    try:
        n = (1 << 18) + 3
        x = _input(F32, n, 5)
        a, b = _coefs(F32)
        dx = dab.B200Array.from_numpy(rt1, x)
        dy = dab.B200Array.empty(rt1, (n,), F32)
        want_d = dab.B200Array.from_numpy(rt1, orc.affine_unfused(a, x, b))
        want = _reduce_host(rt1.ctx, L.F32, L.SUM, want_d.ptr, n)
        l0 = _launches(ctx)
        _affine(ctx, L.F32, dy.ptr, dx.ptr, a, b, n)
        stream = C.c_void_p()
        L.call("dab_stream", ctx, C.byref(stream))                   # queues the pending affine ...
        assert _launches(ctx) - l0 == 1
        got = _reduce_host(ctx, L.F32, L.SUM, dy.ptr, n)
        assert got == want
        for _ in range(2):                                             # ... and nothing is held back afterwards
            l0 = _launches(ctx)
            _affine(ctx, L.F32, dy.ptr, dx.ptr, a, b, n)
            got = _reduce_host(ctx, L.F32, L.SUM, dy.ptr, n)
            assert _launches(ctx) - l0 == 2
            assert got == want
        assert _d2h(ctx, dy.ptr, n, F32).tobytes() == orc.affine_unfused(a, x, b).tobytes()
    finally:
        L.call("dab_shutdown", ctx)
