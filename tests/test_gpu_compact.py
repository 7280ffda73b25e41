"""GPU tests of ``d[mask]``, ``findall`` and ``filter`` (row f13): K23 (``dab_compact_count`` / ``dab_compact``) through the C ABI on
every dispatch path against a byte-exact model, the distributed flow against Julia's logical indexing, the compositions with K22 and
broadcast masks, every element type, and a mask chunk of more than 2^31 elements.  The kernels only move bytes: every result must
equal the model exactly."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:                                                     # the emulated C ABI gets K23 (with the K17 scans) and K22 too
    import compact_hostmem
    import take_hostmem
    compact_hostmem.install()
    take_hostmem.install()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 4096
UNITS = {1: np.uint8, 4: np.uint32, 8: np.uint64, 16: np.complex128}   # carriers of 1-, 4-, 8- and 16-byte elements
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128]


def model(a, m):
    """Julia's ``A[M]`` for a Bool array ``M`` of ``A``'s size."""
    return np.asarray(a).ravel(order="F")[np.asarray(m).ravel(order="F")]


def model_findall(m):
    return np.flatnonzero(np.asarray(m).ravel(order="F")).astype(np.int64) + 1


def _bits(es, n, rng):
    """n elements of random bit patterns (NaNs with payloads, -0.0, denormals included) in the carrier of ``es`` bytes."""
    return rng.integers(0, 256, n * es, dtype=np.uint8).view(UNITS[es])


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def _mask_bytes(n, density, rng):
    """Mask bytes: 0 for false and any nonzero byte for true (true is "nonzero", not only 1)."""
    t = rng.random(n) < density
    return np.where(t, rng.integers(1, 256, n), 0).astype(np.uint8)


def _compact(dab, rt, mask, vals, run_len, runs, es, out_cuts, mask_off=0, src_off=0, out_off=0):
    """K23 on one chunk of ``runs`` runs of ``run_len`` elements through the C ABI: dab_compact_count, the tile offsets from the host
    (so that only K23 is under test), then dab_compact into an output of ``len(out_cuts) - 1`` chunks (``es == 0``: index mode with run
    r starting at linear index 1000 * r).  ``*_off``: elements between each allocation's start and the pointer passed.  Returns the
    counts, the output (sentinel fill where nothing is written) and the model of both."""
    from darray_b200 import _lib
    n = run_len * runs
    tpr = -(-run_len // TILE)
    tiles = tpr * runs
    mb = _up(dab, rt, np.concatenate([np.full(mask_off, 7, np.uint8), mask, np.zeros(1, np.uint8)]))
    carrier = np.int64 if es == 0 else UNITS[es]
    usz = np.dtype(carrier).itemsize
    sb = None if es == 0 else _up(dab, rt, np.concatenate([np.zeros(src_off, carrier), vals]).astype(carrier))
    cb = dab.B200Array.from_numpy(rt, np.full(max(tiles, 1), -5, np.int32))
    l0 = rt.launches()
    _lib.call("dab_compact_count", rt.ctx, C.c_void_p(mb.ptr + mask_off), run_len, runs, C.c_void_p(cb.ptr))
    launched = rt.launches() - l0
    counts = cb.to_numpy()[:tiles]
    want_counts = np.array([np.count_nonzero(mask[(b // tpr) * run_len + (b % tpr) * TILE:][:min(TILE, run_len - (b % tpr) * TILE)])
                            for b in range(tiles)], dtype=np.int32)
    incl = np.cumsum(want_counts.reshape(runs, tpr) if tiles else np.zeros((0, 0), np.int32), axis=1).reshape(-1).astype(np.int64)
    run_tot = incl.reshape(runs, tpr)[:, -1] if tiles else np.zeros(runs, np.int64)
    run_off = np.concatenate([[0], np.cumsum(run_tot)])[:-1].astype(np.int64) if runs else np.zeros(0, np.int64)
    info = np.stack([run_off, 1000 * np.arange(runs, dtype=np.int64)]).reshape(-1, order="F")
    ib = dab.B200Array.from_numpy(rt, np.concatenate([incl, [0]]).astype(np.int64))
    rb = dab.B200Array.from_numpy(rt, np.concatenate([info, [0]]).astype(np.int64))
    sel = mask.astype(bool)
    if es == 0:
        want = np.concatenate([1000 * r + np.flatnonzero(sel[r * run_len:(r + 1) * run_len]) + 1 for r in range(runs)] or
                              [np.zeros(0, np.int64)]).astype(np.int64)
    else:
        want = vals[sel]
    fill = _bits(usz, int(out_cuts[-1]), np.random.default_rng(1)).view(carrier)
    chunks, ptrs = [], []
    for c in range(len(out_cuts) - 1):
        k = out_cuts[c + 1] - out_cuts[c]
        if k:
            ob = _up(dab, rt, np.concatenate([np.zeros(out_off, carrier), fill[out_cuts[c]:out_cuts[c + 1]]]).astype(carrier))
            chunks.append((ob, c, out_off + k))
            ptrs.append(ob.ptr + out_off * usz)
        else:
            ptrs.append(None)
    l1 = rt.launches()
    _lib.call("dab_compact", rt.ctx, es, C.c_void_p(mb.ptr + mask_off), C.c_void_p(sb.ptr + src_off * usz) if sb else None, run_len, runs,
              C.c_void_p(ib.ptr), C.c_void_p(rb.ptr), len(out_cuts) - 1, (C.c_size_t * len(out_cuts))(*out_cuts),
              (C.c_void_p * len(ptrs))(*ptrs))
    launched += rt.launches() - l1
    out = fill.copy()
    for ob, c, k in chunks:
        h = _down(rt, ob, k, carrier)
        assert np.array_equal(h[:out_off].view(np.uint8), np.zeros(out_off, carrier).view(np.uint8))   # nothing before the chunk
        out[out_cuts[c]:out_cuts[c + 1]] = h[out_off:]
    expect = fill.copy()
    expect[:want.size] = want
    for x in [mb, cb, ib, rb] + ([sb] if sb else []) + [ob for ob, _, _ in chunks]:
        x.free()
    return counts, want_counts, out, expect, launched


def _up(dab, rt, a):
    """A device copy of the bytes of the host array ``a`` (any element type)."""
    from darray_b200 import _lib
    a = np.ascontiguousarray(a)
    b = dab.B200Array.empty(rt, (max(a.nbytes, 1),), np.bool_)
    if a.nbytes:
        _lib.call("dab_h2d", rt.ctx, C.c_void_p(b.ptr), C.c_void_p(a.ctypes.data), a.nbytes)
        rt.sync()
    return b


def _down(rt, b, n, dt):
    from darray_b200 import _lib
    out = np.empty(n, dtype=dt)
    if out.nbytes:
        _lib.call("dab_d2h", rt.ctx, C.c_void_p(out.ctypes.data), C.c_void_p(b.ptr), out.nbytes)
        rt.sync()
    return out


def _cuts(total, g, rng):
    inner = np.sort(rng.integers(0, total + 1, g - 1)) if g > 1 else np.zeros(0, np.int64)
    return [0] + [int(x) for x in inner] + [int(total)]


@pytest.mark.parametrize("es", [0, 1, 4, 8, 16])
@pytest.mark.parametrize("run_len", [1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_kernel_sizes_and_alignment(dab, rt1, es, run_len):
    """Every element size and index mode, runs of 1, tile - 1, tile, tile + 1 and several tiles, aligned and misaligned mask, value
    and output pointers, random mask bytes, a 3-chunk output (one empty)."""
    rng = np.random.default_rng(run_len * 5 + es)
    for runs in (1, 3):
        n = run_len * runs
        mask = _mask_bytes(n, 0.5, rng)
        vals = None if es == 0 else _bits(es, n, rng)
        cnt = int(np.count_nonzero(mask))
        total = cnt + 5
        for mo, so, oo in ((0, 0, 0), (1, 0, 0), (3, 1, 1), (16, 0, 1)):
            cuts = [0, cnt // 3, cnt // 3, total]
            counts, want_counts, out, expect, launched = _compact(dab, rt1, mask, vals, run_len, runs, es, cuts, mo, so, oo)
            _same(counts, want_counts)
            _same(out, expect)
            assert launched == 2


@pytest.mark.parametrize("es", [0, 1, 4, 8, 16])
def test_kernel_many_short_runs(dab, rt1, es):
    """Runs shorter than a tile (3 elements) and many of them (2000), densities 0, 1 and random, an output of 7 chunks."""
    rng = np.random.default_rng(es)
    for run_len, runs in ((3, 2000), (1, 5000), (100, 300)):
        for density in (0.0, 1.0, 0.37):
            n = run_len * runs
            mask = _mask_bytes(n, density, rng)
            vals = None if es == 0 else _bits(es, n, rng)
            cnt = int(np.count_nonzero(mask))
            counts, want_counts, out, expect, _ = _compact(dab, rt1, mask, vals, run_len, runs, es, _cuts(cnt, 7, rng) if cnt else [0, 1], 1)
            _same(counts, want_counts)
            _same(out, expect)


@pytest.mark.parametrize("es", [0, 4, 16])
def test_kernel_size_zero(dab, rt1, es):
    """run_len == 0 or runs == 0: no launch, and nothing written."""
    rng = np.random.default_rng(0)
    for run_len, runs in ((0, 5), (7, 0)):
        _, _, out, expect, launched = _compact(dab, rt1, np.zeros(0, np.uint8), None if es == 0 else _bits(es, 0, rng), run_len, runs, es, [0, 4])
        _same(out, expect)
        assert launched == 0


def test_kernel_refusals(dab, rt1):
    """Unserved element sizes, more than 1024 output chunks, decreasing cuts and a NULL non-empty chunk: status codes, no launch."""
    from darray_b200 import _lib
    m = dab.B200Array.from_numpy(rt1, np.ones(8, np.bool_))
    v = dab.B200Array.from_numpy(rt1, np.arange(8.0))
    t = dab.B200Array.from_numpy(rt1, np.array([8], np.int64))
    info = dab.B200Array.from_numpy(rt1, np.array([0, 0], np.int64))
    out = dab.B200Array.empty(rt1, (8,), np.float64)

    def call(es=8, cuts=(0, 8), ptrs=None):
        ptrs = ptrs if ptrs is not None else [out.ptr] * (len(cuts) - 1)
        return _lib.lib().dab_compact(rt1.ctx, es, C.c_void_p(m.ptr), C.c_void_p(v.ptr), 8, 1, C.c_void_p(t.ptr), C.c_void_p(info.ptr),
                                      len(cuts) - 1, (C.c_size_t * len(cuts))(*cuts), (C.c_void_p * len(ptrs))(*ptrs))
    l0 = rt1.launches()
    assert call(es=2) == _lib.ERR_ARG
    assert call(cuts=(0,) * 1025 + (8,)) == _lib.ERR_UNSUPPORTED
    assert call(cuts=(0, 9, 8)) == _lib.ERR_ARG
    assert call(cuts=(1, 8)) == _lib.ERR_ARG
    assert call(cuts=(0, 4, 8), ptrs=[out.ptr, None]) == _lib.ERR_ARG
    assert rt1.launches() == l0
    assert call() == _lib.OK and rt1.launches() == l0 + 1
    _same(out.to_numpy(), np.arange(8.0))


# ---- the distributed flow ----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("shape,dist", [((100003,), None), ((37, 29), [3, 2]), ((6, 5, 7), [2, 1, 3]), ((301, 47), [1, 8]),
                                        ((64, 50), [8, 1]), ((5, 4, 3, 2, 2, 3), [2, 2, 1, 1, 1, 2])])
@pytest.mark.parametrize("density", [0.0, 1.0, 0.5, 0.01])
def test_distributed_flow(dab, rt8, shape, dist, density):
    """d[m] and findall(m) on 8 workers against a.ravel('F')[m.ravel('F')] and flatnonzero + 1, d and m in the same layout and in
    different ones."""
    rng = np.random.default_rng(len(shape) * 7 + int(density * 100))
    a = rng.standard_normal(shape)
    mh = rng.random(shape) < density
    lays = [dict()] + ([dict(procs=list(range(1, int(np.prod(dist)) + 1)), dist=dist)] if dist else [])
    for dl in lays:
        d = dab.distribute(a, **dl)
        for ml in lays:
            m = dab.distribute(mh, **ml)
            R = d[m]
            S = dab.similar(d, dims=R.dims)
            assert R.layout.pids == S.layout.pids and R.layout.indices == S.layout.indices
            _same(dab.to_array(R), model(a, mh))
            _same(dab.to_array(dab.findall(m)), model_findall(mh))


def test_compositions(dab, rt8):
    """d[findall(m)] == d[m] byte for byte through K22, v[v > 0] with a broadcast mask, filter and findall with a predicate."""
    rng = np.random.default_rng(2)
    h = rng.standard_normal((203, 41))
    h[rng.random(h.shape) < 0.05] = -0.0
    d = dab.distribute(h, procs=list(range(1, 9)), dist=[4, 2])
    mh = rng.random(h.shape) < 0.3
    m = dab.distribute(mh)
    _same(dab.to_array(d[dab.findall(m)]), dab.to_array(d[m]))
    v = dab.distribute(rng.standard_normal(50001))
    vh = dab.to_array(v)
    _same(dab.to_array(v[dab.broadcast(lambda x: x > 0, v)]), vh[vh > 0])
    _same(dab.to_array(dab.filter(lambda x: x > 0, d)), model(h, h > 0))
    _same(dab.to_array(dab.findall(lambda x: x < -1, d)), model_findall(h < -1))
    _same(dab.to_array(dab.findall(lambda x: dab.isnan(x), v)), np.zeros(0, np.int64))


@pytest.mark.parametrize("T", ELTYPES)
def test_every_element_type(dab, rt8, T):
    """Every element type on a 2-d d split along dim 1, random bit patterns compared byte for byte."""
    rng = np.random.default_rng(np.dtype(T).itemsize)
    es = np.dtype(T).itemsize
    h = (rng.random((97, 61)) < 0.5) if T == np.bool_ else _bits(es, 97 * 61, rng).view(T).reshape(97, 61)
    mh = rng.random((97, 61)) < 0.45
    for dist in ([8, 1], [2, 4]):
        d = dab.distribute(h, procs=list(range(1, 9)), dist=dist)
        R = d[dab.distribute(mh)]
        assert R.dtype == np.dtype(T)
        _same(dab.to_array(R), model(h, mh))


def test_refusals_leave_nothing(dab, rt8):
    """A Bool key of other dims stays UnsupportedError; non-Bool findall and predicates raise Julia's TypeError; nothing launched."""
    d = dab.distribute(np.arange(16.0).reshape(4, 4))
    keys = [dab.distribute(np.array([True, False])), dab.distribute(np.ones(16, dtype=bool))]
    l0, r0 = rt8.launches(), dab.registry_size()
    for k in keys:
        with pytest.raises(dab.UnsupportedError):
            d[k]
    with pytest.raises(TypeError, match=r"non-boolean \(Float64\)"):
        dab.findall(d)
    with pytest.raises(TypeError, match=r"non-boolean \(Float64\)"):
        dab.filter(lambda x: x + 1, d)
    assert rt8.launches() == l0 and dab.registry_size() == r0


@pytest.mark.skipif(HOSTMEM, reason="a chunk of more than 2^31 elements is a device-memory case")
def test_chunk_past_2_pow_31(dab, rt1):
    """One Bool chunk of 2^31 + 2^20 + 5 elements with trues before and past 2^31: findall(m) and m[m]."""
    from darray_b200 import _lib
    n = (1 << 31) + (1 << 20) + 5
    m = dab.dfill(False, (n,), procs=[1])
    pos = np.array([0, 12345, (1 << 31) - 1, 1 << 31, (1 << 31) + 4097, n - 1], dtype=np.int64)
    one = np.ones(1, np.uint8)
    ch = m.chunks[1]
    for p in pos:
        _lib.call("dab_h2d", rt1.ctx, C.c_void_p(ch.ptr + int(p)), C.c_void_p(one.ctypes.data), 1)
    rt1.sync()
    _same(dab.to_array(dab.findall(m)), pos + 1)
    R = m[m]
    assert R.dims == (pos.size,) and bool(dab.to_array(R).all())


def test_multi_gpu():
    """tools/multi_gpu_compact.py under torchrun on two GPUs: d split across ranks, the mask in a different layout, results whose
    chunks live on the other rank."""
    import torch
    if HOSTMEM or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.join(ROOT, "tools", "multi_gpu_compact.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "multi-gpu compact passed" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
