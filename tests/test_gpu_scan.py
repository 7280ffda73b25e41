"""GPU tier of the scans (K17, ``dab_scan`` / ``dab_scan_totals``) on one H100.

Bit-exact through the ABI on every kernel path against the sequential model in tests/scan_oracle.py, on inputs whose results are exact
in any order: integers of any value, float sums on the 2^-10 grid, float products of +-1 with a few +-2 / +-0.5, max / min with NaN,
+-0 and +-Inf.  Then the public API on 1, 2 and 8 workers, and one 2^31 + 5 element in-place scan for 64-bit indexing.
The multi-rank path needs a box with two or more GPUs; its carry plan is executed over gloo in tests/test_cpu_scan.py."""
import ctypes as C

import numpy as np
import pytest

import scan_oracle as so

pytestmark = pytest.mark.gpu

TILE = 4096
F32, F64, I32, I64, U8 = range(5)
SUM, PROD, MAX, MIN = range(4)
NP = so._NP
CASES = [(F32, SUM, F32), (F64, SUM, F64), (F32, PROD, F32), (F64, PROD, F64), (I32, SUM, I64), (I32, SUM, I32), (I32, PROD, I32),
         (I32, PROD, I64), (I64, SUM, I64), (I64, PROD, I64), (U8, SUM, I64), (U8, PROD, U8), (F32, MAX, F32), (F64, MIN, F64),
         (F32, MIN, F32), (F64, MAX, F64), (I32, MAX, I32), (I64, MIN, I64), (U8, MAX, U8), (U8, MIN, U8)]
SHAPES = [(1, 1, 1), (1, 2, 1), (1, 3, 2), (1, TILE - 1, 2), (1, TILE, 3), (1, TILE + 1, 2), (1, 5 * TILE + 17, 1), (1, 10, 3001),
          (1, 7, 1500), (1, 1, 5000), (2, 5000, 1), (3, 700, 2), (5, 64, 3), (1000, 300, 2), (1000, 20, 3), (4097, 40, 2), (4097, 100, 1),
          (1024, 200, 1), (1024, 20, 2), (2, 140000, 1)]   # 16-byte vectors for every element size; > 4096 segments


def values(code, op, n, rng):
    if code == U8:
        return rng.random(n) < (0.9 if op in (PROD, MIN) else 0.1)
    if code in (I32, I64):
        info = np.iinfo(NP[code])
        return rng.integers(info.min, info.max, n, dtype=NP[code], endpoint=True)
    dt = NP[code]
    if op == SUM:
        return (rng.integers(-8, 9, n) * 2.0 ** -10).astype(dt)
    if op == PROD:
        v = rng.choice([1.0, -1.0], n)
        k = rng.random(n)
        v[k < 0.01] *= 2.0
        v[(k >= 0.01) & (k < 0.02)] *= 0.5
        return v.astype(dt)
    v = rng.standard_normal(n).astype(dt)
    edges = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], dtype=dt)
    pos = rng.random(n) < 0.05
    v[pos] = rng.choice(edges, int(pos.sum()))
    for p in (TILE - 1, TILE, TILE + 1, 2 * TILE - 1):               # edge values at tile boundaries
        if p < n:
            v[p] = edges[p % 4]
    v[(rng.random(n) < 0.0005)] = np.nan                          # rare: most fibres stay NaN-free
    return v


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint8), b[~nb].view(np.uint8))


def model(code, op, out_code, x, inner, ln, outer, carry):
    """Julia's sequential fold of every fibre (seeded by the carry, an exact value on these inputs), in the result type."""
    name = {SUM: "+", PROD: "*", MAX: "max", MIN: "min"}[op]
    v = x.reshape((inner, ln, outer), order="F")
    R = NP[out_code]
    W = np.dtype(np.int64) if (code == U8 and op == SUM) else R
    rows = np.moveaxis(v, 1, 0)
    if carry is not None:
        rows = np.concatenate([carry.reshape((1, inner, outer), order="F").astype(W), rows.astype(W)])
    out = so._fold_rows(name, rows, W)
    if carry is not None:
        out = out[1:]
    return np.moveaxis(out, 0, 1).astype(R).reshape(-1, order="F")


def run_abi(dab, rt, code, op, out_code, x, inner, ln, outer, carry=None, off=0, inplace=False):
    from darray_b200 import B200Array, _lib
    n = inner * ln * outer
    isz = NP[code].itemsize
    xb = B200Array.from_numpy(rt, np.concatenate([np.zeros(off, NP[code]), x]))
    xp = xb.ptr + off * isz
    yb = xb if inplace else B200Array.empty(rt, (n + off,), NP[out_code])
    yp = xp if inplace else yb.ptr + off * NP[out_code].itemsize
    cb = B200Array.from_numpy(rt, carry) if carry is not None else None
    _lib.call("dab_scan", rt.ctx, code, op, out_code, C.c_void_p(xp), inner, ln, outer, C.c_void_p(cb.ptr) if cb else None, C.c_void_p(yp))
    got = yb.to_numpy()[off:]
    tot = B200Array.empty(rt, (inner * outer,), so.carrier(code, op))
    xb2 = B200Array.from_numpy(rt, x)
    _lib.call("dab_scan_totals", rt.ctx, code, op, out_code, C.c_void_p(xb2.ptr), inner, ln, outer, C.c_void_p(tot.ptr))
    tv = tot.to_numpy()
    for b in (xb, tot, xb2) + (() if inplace else (yb,)) + ((cb,) if cb else ()):
        b.free()
    return got, tv


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}")
def test_abi_bit_exact_every_path(rt1, dab, case):
    code, op, out_code = case
    rng = np.random.default_rng(1000 * code + 10 * op + out_code)
    for si, (inner, ln, outer) in enumerate(SHAPES):
        n = inner * ln * outer
        x = values(code, op, n, rng)
        A = so.carrier(code, op)
        carry = None
        if si % 3 == 1:                                           # an exact carry in the carrier type
            carry = values(code, op, inner * outer, rng).astype(A) if code != U8 else (rng.random(inner * outer) < 0.5).astype(A)
        off = 0 if inner % 16 == 0 else si % 4                  # inner = 1024 stays aligned: the 16-byte strided kernel
        inplace = si % 5 == 2 and NP[code].itemsize == NP[out_code].itemsize
        got, tot = run_abi(dab, rt1, code, op, out_code, x, inner, ln, outer, carry, off, inplace)
        want = model(code, op, out_code, x, inner, ln, outer, carry)
        assert same(got, want), (case, inner, ln, outer, off, inplace, carry is not None)
        want_tot = so.emulate_scan(code, op, out_code, x, inner, ln, outer, None)[:, -1, :].reshape(-1, order="F")
        assert same(tot, want_tot.astype(A)), (case, inner, ln, outer, "totals")


def test_abi_refusals_and_empty(rt1, dab):
    from darray_b200 import B200Array, _lib
    x = B200Array.from_numpy(rt1, np.ones(8, np.float32))
    for bad in ((F32, SUM, F64), (I32, MAX, I64), (U8, SUM, U8), (I64, 4, I64), (5, SUM, 5)):
        with pytest.raises(dab.UnsupportedError):
            _lib.call("dab_scan", rt1.ctx, bad[0], bad[1], bad[2], C.c_void_p(x.ptr), 1, 8, 1, None, C.c_void_p(x.ptr))
    _lib.call("dab_scan", rt1.ctx, F32, SUM, F32, C.c_void_p(x.ptr), 1, 0, 1, None, C.c_void_p(x.ptr))
    t = B200Array.empty(rt1, (3,), np.float64)
    _lib.call("dab_scan_totals", rt1.ctx, F32, SUM, F32, C.c_void_p(x.ptr), 3, 0, 1, C.c_void_p(t.ptr))
    assert np.array_equal(t.to_numpy().view(np.uint64), np.full(3, -0.0).view(np.uint64))
    x.free()
    t.free()


def test_float32_fp64_carrier_deviation(rt1, dab):
    """Float32 prefixes run in fp64 and are rounded once: [3f38, 3f38, -3f38] gives [3f38, Inf, 3f38] (Julia's Float32 fold: Inf)."""
    d = dab.distribute(np.array([3e38, 3e38, -3e38], dtype=np.float32))
    r = dab.to_array(dab.cumsum(d))
    assert r[0] == np.float32(3e38) and np.isinf(r[1]) and r[2] == np.float32(3e38)
    assert np.isinf(so.jl_accumulate("+", np.array([3e38, 3e38, -3e38], dtype=np.float32), 1, cum=True)[2])


def _pairs(dab, A, pids, dist=None):
    return dab.distribute(A, procs=pids, dist=dist)


@pytest.mark.parametrize("fixture", ["rt1", "rt2", "rt8"])
def test_public_api_layouts(request, dab, fixture):
    request.getfixturevalue(fixture)
    rng = np.random.default_rng(3)
    pids = dab.workers()
    P = len(pids)
    for shape in [(50000,), (300, 257), (40, 33, 9)]:
        for dt in (np.float32, np.float64, np.int32, np.int64, np.bool_):
            if dt == np.bool_:
                A = rng.random(shape) < 0.5
            elif np.dtype(dt).kind == "i":
                A = rng.integers(-1000, 1000, shape).astype(dt)
            else:
                A = (rng.integers(-8, 9, shape) * 2.0 ** -10).astype(dt)
            for dist in [None] + ([[1] * (len(shape) - 1) + [P]] if len(shape) > 1 else []):
                d = _pairs(dab, A, pids, dist)
                for dims in range(1, len(shape) + 2):
                    for fn, op, cum in ((dab.cumsum, "+", True), (dab.cumprod, "*", True)):
                        if op == "*" and dt in (np.float32, np.float64):
                            continue
                        r = fn(d, dims=dims)
                        assert r.dtype == so.result_type(dt, op, cum)
                        assert same(dab.to_array(r), so.jl_accumulate(op, A, dims, cum=cum)), (shape, dt, dist, dims, op)
                        assert r.layout.same_as(dab.similar(d, r.dtype).layout)
                    for op in ("max", "min", "+"):
                        init = 3 if op == "+" else None
                        r = dab.accumulate(op, d, dims=dims, init=init)
                        want = so.jl_accumulate(op, A, dims, init=init if dims <= len(shape) else None)
                        assert same(dab.to_array(r), want), (shape, dt, dist, dims, op)
                d.close()
            dab.d_closeall()


def test_public_api_random_floats_and_split_layouts(rt8, dab):
    """Random floats: within n*eps*sum|x| of the extended-precision prefix; Float32 results within 1 ulp between one chunk and the dims
    split over 8 workers; in place and into another layout."""
    rng = np.random.default_rng(9)
    A = rng.standard_normal((4000, 24)).astype(np.float32)
    exact = np.cumsum(A.astype(np.longdouble), axis=0)
    bound = 4000 * np.finfo(np.float32).eps * np.cumsum(np.abs(A).astype(np.float64), axis=0)
    one = dab.distribute(A, procs=[1])
    split = dab.distribute(A, procs=dab.workers(), dist=[8, 1])
    r1 = dab.to_array(dab.cumsum(one, dims=1))
    r8 = dab.to_array(dab.cumsum(split, dims=1))
    assert np.all(np.abs(r1.astype(np.float64) - exact.astype(np.float64)) <= bound)
    ulp = np.abs(r1.view(np.int32).astype(np.int64) - r8.view(np.int32).astype(np.int64))
    assert ulp.max() <= 1
    dab.cumsum_(split, split, dims=1)                              # in place, dims split
    assert np.array_equal(dab.to_array(split), r8)
    dest = dab.distribute(np.zeros_like(A), procs=dab.workers(), dist=[1, 8])
    dab.accumulate_("max", dest, one, dims=1)
    assert same(dab.to_array(dest), so.jl_accumulate("max", A, 1))
    view = dab.distribute(A, procs=dab.workers())[10:3000, 2:20]
    assert np.array_equal(dab.to_array(dab.cumsum(view, dims=2)),
                          dab.to_array(dab.cumsum(dab.distribute(A[10:3000, 2:20].copy()), dims=2)))


def test_index_width_inplace_2_31(rt1, dab):
    """cumsum! in place of 2^31 + 5 Float32 grid values on one worker (8 GiB): sampled positions and the last element exact."""
    from oracle import darray_oracle as orc
    n = 2 ** 31 + 5
    if rt1.device_info()["free_bytes"] < 20 * 2 ** 30:
        pytest.skip("needs 20 GiB of free device memory")
    d = dab.drand((n,), dtype=np.float32, seed=77)
    dab.broadcast_into(d, lambda u: (dab.floor(u * np.float32(17)) - np.float32(8)) * np.float32(2.0 ** -10), d)

    def host_x(lo, cnt):
        u = orc.rand_u01(77, lo, cnt)
        return (np.floor(u * np.float32(17)) - np.float32(8)) * np.float32(2.0 ** -10)

    total = float(dab.sum(d))
    head = np.cumsum(host_x(0, 3 * TILE).astype(np.float64))
    tail_x = host_x(2 ** 31 - 2, n - (2 ** 31 - 2)).astype(np.float64)
    dab.cumsum_(d, d)
    got_head = np.asarray(d[0:3 * TILE]).astype(np.float64)
    assert np.array_equal(got_head, head)
    got_tail = np.asarray(d[2 ** 31 - 2:n]).astype(np.float64)
    want_tail = total - (np.sum(tail_x) - np.cumsum(tail_x))
    assert np.array_equal(got_tail, want_tail), (got_tail, want_tail)
    assert got_tail[-1] == total
    for p in (2 ** 30 + 12345, 2 ** 31 - 4097):
        seg = np.asarray(d[p - 1:p + 2]).astype(np.float64)
        assert np.array_equal(np.diff(seg), host_x(p, 2).astype(np.float64)), p
    d.close()
