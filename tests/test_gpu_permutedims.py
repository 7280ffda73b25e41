"""K28 ``dab_permute_box`` against a byte-exact model on every dispatch path, and ``permutedims`` / ``permutedims_`` end to end.

The ABI cases follow tests/test_gpu_data_movement.py: operands at chosen byte offsets from 256-byte aligned allocations, between
canary bytes, filled with random bytes that include (viewed as floats) NaNs with payloads, +-0, +-Inf and subnormals.  The expected
destination is computed from the bytes alone: every element of the box holds its source element's bytes, every other byte (the gaps of
a strided destination, the canaries) is unchanged.  ``permute_labels`` mirrors the host side of the kernel (the 16-byte path
conditions and the tile shape of ``launch_permute``), so that ``test_case_table_reaches_every_path`` shows which paths the table takes.
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from test_gpu_data_movement import Dev, diff_report, rand_bytes

pytestmark = pytest.mark.gpu

HOSTMEM = os.environ.get("DAB_HOSTMEM") == "1"
if HOSTMEM:
    import permute_hostmem
    permute_hostmem.install()

WIDTHS = (1, 2, 4, 8, 16)
ELTYPES = [np.float32, np.float64, np.int32, np.int64, np.bool_, np.complex64, np.complex128, np.float16]


def _lib():
    from darray_b200 import _lib as L
    return L


# ---------------------------------------------------------------------------------------------------------- dispatch mirror
def tile_shape(es, vec, e0, eq):
    """launch_permute (dab_permute.cu): log2 of the tile extents along q and along 0."""
    V = 16 // es if vec else 1
    lnt = {(1, True): 14, (1, False): 12, (2, True): 12, (2, False): 12, (4, True): 12, (4, False): 12, (8, True): 10, (8, False): 10,
           (16, False): 10}[(es, vec)]
    le = lnt // 2
    seg = max(32 // es, V)
    lmin = seg.bit_length() - 1
    lq, l0 = max(eq - 1, 0).bit_length(), max(e0 - 1, 0).bit_length()
    if lq >= le and l0 >= le:
        return le, le
    if lq <= l0:
        lq = max(lq, lmin)
        return lq, lnt - lq
    l0 = max(l0, lmin)
    return lnt - l0, l0


def permute_labels(es, dptr, dstr, sptr, sstr, ext, strided_dst):
    q = [k for k in range(1, len(ext)) if sstr[k] == 1][0]
    V = 16 // es if es < 16 else 1
    vec = (V > 1 and dptr % 16 == 0 and sptr % 16 == 0 and ext[0] % V == 0 and ext[q] % V == 0
           and all(sstr[k] % V == 0 for k in range(len(ext)) if k != q) and all(dstr[k] % V == 0 for k in range(1, len(ext))))
    lq, l0 = tile_shape(es, vec, ext[0], ext[q])
    out = {f"{es}B {'16-byte' if vec else 'one-element'} accesses", f"batch of {len(ext) - 2} dims"}
    out.add("ragged last tile" if ext[0] % (1 << l0) or ext[q] % (1 << lq) else "whole tiles")
    if lq < l0:
        out.add("tile narrowed along q")
    if l0 < lq:
        out.add("tile narrowed along 0")
    if ext[0] == 1 or ext[q] == 1:
        out.add("plane extent 1")
    if q != 1:
        out.add("q != 1")
    if strided_dst:
        out.add("strided destination")
    if min(dstr) < 0 or min(sstr) < 0:
        out.add("negative strides")
    return out


REQUIRED = ({f"{es}B 16-byte accesses" for es in (1, 2, 4, 8)} | {f"{es}B one-element accesses" for es in WIDTHS}
            | {f"batch of {n} dims" for n in range(0, 7)}
            | {"ragged last tile", "whole tiles", "tile narrowed along q", "tile narrowed along 0", "plane extent 1", "q != 1",
               "strided destination", "negative strides"})


# ---------------------------------------------------------------------------------------------------------- case table
# (extents in destination order, source memory order (its first dim is q), destination padding per dim, source padding per step)
GEOMS = {
    "2d_ragged": ((70, 45), (1, 0), (0, 0), (0, 0)),
    "2d_whole_tiles": ((128, 128), (1, 0), (0, 0), (0, 0)),
    "2d_padded_both": ((37, 53), (1, 0), (3, 0), (5, 0)),
    "3d_q2": ((40, 3, 36), (2, 0, 1), (0, 0, 0), (0, 0, 0)),
    "3d_q1_batch": ((33, 17, 5), (1, 2, 0), (0, 0, 0), (1, 0, 0)),
    "3d_vec": ((64, 5, 32), (2, 0, 1), (0, 0, 0), (0, 0, 0)),
    "3d_vec_strided_dst": ((48, 6, 32), (2, 1, 0), (16, 0, 0), (0, 16, 0)),
    "narrow_q": ((200, 3, 4), (1, 0, 2), (0, 0, 0), (0, 0, 0)),
    "narrow_0": ((2, 150, 3), (1, 2, 0), (0, 0, 0), (0, 0, 0)),
    "extent1_dim0": ((1, 50, 6), (1, 2, 0), (0, 0, 0), (0, 0, 0)),
    "extent1_q": ((20, 1, 7), (1, 0, 2), (0, 0, 0), (0, 0, 0)),
    "4d": ((9, 4, 11, 3), (2, 3, 0, 1), (1, 0, 2, 0), (0, 1, 0, 0)),
    "5d": ((6, 5, 3, 4, 2), (3, 1, 4, 0, 2), (0, 0, 0, 0, 0), (0, 0, 0, 0, 0)),
    "6d_strided": ((5, 3, 4, 2, 3, 2), (4, 5, 0, 2, 1, 3), (2, 1, 0, 0, 1, 0), (0, 0, 0, 0, 0, 0)),
    "7d": ((4, 3, 2, 3, 2, 2, 3), (6, 2, 0, 4, 1, 5, 3), (0, 0, 0, 0, 0, 0, 0), (0, 0, 0, 0, 0, 0, 0)),
    "8d": ((5, 4, 2, 3, 2, 2, 3, 2), (3, 7, 1, 0, 5, 2, 6, 4), (0, 0, 0, 0, 0, 0, 0, 0), (0, 0, 0, 0, 0, 0, 0, 0)),
    "8d_vec_q7": ((16, 2, 2, 1, 2, 3, 2, 16), (7, 0, 2, 1, 4, 3, 6, 5), (0, 0, 0, 0, 0, 0, 0, 0), (0, 0, 0, 0, 0, 0, 0, 0)),
    "3d_vec_negative_batch": ((64, 5, 32), (2, 0, 1), (0, 0, 0), (0, 0, 0)),
    "4d_negative": ((9, 4, 11, 3), (2, 3, 0, 1), (1, 0, 2, 0), (0, 1, 0, 0)),
}
# dimensions whose stride is negated (destination, source): the operand pointer then addresses coordinate 0 from inside the allocation
NEGATED = {"3d_vec_negative_batch": ((1,), (1,)), "4d_negative": ((2,), (0, 3))}


def geometry(name):
    """Strides (elements) and spans of one geometry: destination column-major over padded extents, source in its memory order."""
    ext, order, dpad, spad = GEOMS[name]
    N = len(ext)
    dstr, r = [], 1
    for k in range(N):
        dstr.append(r)
        r *= ext[k] + dpad[k]
    sstr, r = [0] * N, 1
    for i, k in enumerate(order):
        sstr[k] = r
        r *= ext[k] + spad[i]
    dspan = 1 + sum((e - 1) * s for e, s in zip(ext, dstr))
    sspan = 1 + sum((e - 1) * s for e, s in zip(ext, sstr))
    dneg, sneg = NEGATED.get(name, ((), ()))
    dbase = sum((ext[k] - 1) * dstr[k] for k in dneg)          # element offset of coordinate 0 from the start of the span
    sbase = sum((ext[k] - 1) * sstr[k] for k in sneg)
    dstr = [-v if k in dneg else v for k, v in enumerate(dstr)]
    sstr = [-v if k in sneg else v for k, v in enumerate(sstr)]
    return list(ext), dstr, sstr, dspan, sspan, any(dpad), dbase, sbase


def cases(es):
    """Every geometry with both operands 16-byte aligned and, below 16-byte elements, with each operand misaligned by one element."""
    out = [(name, 0, 0) for name in GEOMS]
    if es < 16:
        out += [(name, es, 0) for name in GEOMS] + [(name, 0, es) for name in ("2d_whole_tiles", "3d_vec", "8d_vec_q7", "3d_vec_negative_batch")]
    return out


def offsets(ext, strides):
    tot = np.zeros((), dtype=np.int64)
    for e, s in zip(ext, strides):
        tot = tot[..., None] + np.arange(e, dtype=np.int64) * s
    return tot.reshape(-1)


def test_case_table_reaches_every_path(capsys):
    got = set()
    for es in WIDTHS:
        for name, ps, pd in cases(es):
            ext, dstr, sstr, dspan, sspan, strided, dbase, sbase = geometry(name)
            assert sum(1 for k in range(1, len(ext)) if sstr[k] == 1) == 1 and dstr[0] == 1, name
            do, so = offsets(ext, dstr) + dbase, offsets(ext, sstr) + sbase
            assert np.unique(do).size == int(np.prod(ext)), name                       # the destination box does not overlap itself
            assert do.min() == so.min() == 0 and do.max() == dspan - 1 and so.max() == sspan - 1, name
            got |= permute_labels(es, 8192 + pd + dbase * es, dstr, 4096 + ps + sbase * es, sstr, ext, strided)
    with capsys.disabled():
        print("\npaths reached by the case table:\n  " + "\n  ".join(sorted(got)))
    assert REQUIRED <= got, sorted(REQUIRED - got)


@pytest.mark.parametrize("es", WIDTHS)
def test_permute_box_bit_exact(dab, rt1, es):
    """Every case: one launch, the box's bytes equal their source bytes, every other destination byte and the source unchanged."""
    rng = np.random.default_rng(2800 + es)
    L = _lib()
    bad = []
    for name, ps, pd in cases(es):
        ext, dstr, sstr, dspan, sspan, _, dbase, sbase = geometry(name)
        nd = len(ext)
        src = Dev(rt1, rand_bytes(rng, es * sspan), ps, rng)
        dst = Dev(rt1, rand_bytes(rng, es * dspan), pd, rng)
        try:
            n0 = rt1.launches()
            LL = C.c_longlong * nd
            L.call("dab_permute_box", rt1.ctx, es, nd, C.c_void_p(dst.ptr + dbase * es), LL(*dstr), C.c_void_p(src.ptr + sbase * es), LL(*sstr),
                   (C.c_size_t * nd)(*ext))
            rt1.sync()
            nl = rt1.launches() - n0
            got = dst.get()
            want = dst.img.copy()
            d_el = want[dst.at:dst.at + es * dspan].reshape(dspan, es)
            s_el = src.img[src.at:src.at + es * sspan].reshape(sspan, es)
            d_el[offsets(ext, dstr) + dbase] = s_el[offsets(ext, sstr) + sbase]
            if not np.array_equal(got, want):
                bad.append(f"{name} phases {ps}/{pd}: {diff_report(got, want, dst.at)}")
            if not np.array_equal(src.get(), src.img):
                bad.append(f"{name}: the source changed")
            if nl != 1:
                bad.append(f"{name}: {nl} launches")
        finally:
            src.free()
            dst.free()
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:8])


def test_permute_box_refusals_write_nothing(dab, rt1):
    """A null pointer, ndim outside 2..8, an element width other than 1, 2, 4, 8, 16, destination dim 0 not contiguous, and zero or two
    other source-contiguous dims: ArgumentError, no launch, the destination byte for byte unchanged; a zero extent launches nothing."""
    L = _lib()
    rng = np.random.default_rng(28)
    src = Dev(rt1, rand_bytes(rng, 4096), 0, rng)
    dst = Dev(rt1, rand_bytes(rng, 4096), 0, rng)
    LL, SZ = C.c_longlong * 9, C.c_size_t * 9
    ok_d, ok_s, ok_e = [1, 8] + [64] * 7, [8, 1] + [64] * 7, [8, 8] + [1] * 7

    def call(es=4, nd=2, ds=ok_d, ss=ok_s, ext=ok_e, dp=None, sp=None):
        return lambda: L.call("dab_permute_box", rt1.ctx, es, nd, C.c_void_p(dst.ptr if dp is None else dp), LL(*ds),
                              C.c_void_p(src.ptr if sp is None else sp), LL(*ss), SZ(*ext))

    try:
        refused = [call(es=e) for e in (0, 3, 32, -4)] + [call(nd=n) for n in (0, 1, 9)] + [
            call(ds=[2, 8] + [64] * 7), call(ss=[8, 16] + [64] * 7), call(nd=3, ds=[1, 8, 64] + [0] * 6, ss=[64, 1, 1] + [0] * 6, ext=[8, 8, 1] + [1] * 6),
            call(dp=0), call(sp=0)]
        for k, f in enumerate(refused + [call(ext=[8, 0] + [1] * 7), call(nd=3, ds=[1, 8, 64] + [0] * 6, ss=[8, 1, 64] + [0] * 6, ext=[0, 8, 2] + [1] * 6)]):
            n0 = rt1.launches()
            if k < len(refused):
                with pytest.raises(L.ArgumentError):
                    f()
            else:
                f()
            rt1.sync()
            assert rt1.launches() == n0, k
            assert np.array_equal(dst.get(), dst.img), k
    finally:
        src.free()
        dst.free()


# ---------------------------------------------------------------------------------------------------------- public forms
def _values(T, shape, rng):
    """Random bits of the element type (NaN payloads, -0.0, subnormals and Infs among them for the float types; 0 / 1 for Bool)."""
    T = np.dtype(T)
    n = int(np.prod(shape))
    if T == np.bool_:
        return (rng.random(n) > 0.5).reshape(shape, order="F")
    return rand_bytes(rng, n * T.itemsize).view(T).reshape(shape, order="F")


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def _plan_len(dab, src_layout, dims, procs, dist=None, es=8):
    from darray_b200._permute import permute_plan
    from darray_b200.layout import make_layout
    return lambda perm: len(permute_plan(src_layout, make_layout(dims, procs, dist), perm, es))


ND_CASES = [((24, 10, 13), (3, 1, 2), [2, 1, 3]), ((12, 7, 9, 5), (2, 4, 3, 1), [1, 2, 1, 3]), ((6, 5, 7, 4, 3), (5, 3, 1, 4, 2), None),
            ((4, 3, 5, 2, 3, 4), (6, 1, 5, 2, 4, 3), [1, 1, 2, 1, 1, 4]), ((65, 33, 3), (2, 1, 3), [3, 2, 1]), ((40, 3, 48), (1, 3, 2), None)]


@pytest.mark.parametrize("rtname", ["rt1", "rt2", "rt8"])
@pytest.mark.parametrize("T", ELTYPES, ids=[np.dtype(t).name for t in ELTYPES])
def test_public_forms_bit_exact(dab, request, rtname, T):
    """3-d to 6-d arrays in irregular layouts: ``permutedims`` equals ``np.transpose`` bit for bit with one launch per plan piece and the
    layout of ``similar``; ``permutedims_`` into a destination with another grid; ``permutedims(v)``; ``permutedims(M)`` equals
    ``copy(transpose(M))`` with as many launches; nothing is left registered."""
    rt = request.getfixturevalue(rtname)
    nw = len(rt.workers())
    rng = np.random.default_rng(zlib.crc32(f"{rtname} {np.dtype(T).name}".encode()))
    r0 = dab.registry_size()
    for dims, perm, dist in ND_CASES:
        a = _values(T, dims, rng)
        procs = list(range(1, nw + 1))
        if dist is not None and int(np.prod(dist)) > nw:
            dist = None
        A = dab.distribute(a, procs=procs, dist=dist)
        pd = tuple(dims[p - 1] for p in perm)
        l0 = rt.launches()
        B = dab.permutedims(A, perm)
        nl = rt.launches() - l0
        _same(dab.to_array(B), np.transpose(a, [p - 1 for p in perm]))
        S = dab.similar(A, dims=pd)
        assert B.layout.same_as(S.layout)
        assert nl == _plan_len(dab, A.layout, pd, list(A.layout.pids), es=np.dtype(T).itemsize)(perm)
        D = dab.distribute(np.zeros(pd, dtype=T), procs=procs[::-1], dist=[min(nw, pd[0])] + [1] * (len(pd) - 1))
        l0 = rt.launches()
        dab.permutedims_(D, A, perm)
        assert rt.launches() - l0 == _plan_len(dab, A.layout, pd, procs[::-1], D.layout.grid, es=np.dtype(T).itemsize)(perm)
        _same(dab.to_array(D), np.transpose(a, [p - 1 for p in perm]))
        for x in (A, B, S, D):
            x.close()
    v = _values(T, (1001,), rng)
    V = dab.distribute(v)
    R = dab.permutedims(V)
    _same(dab.to_array(R), v.reshape(1, -1))
    m = _values(T, (130, 67), rng)
    M = dab.distribute(m)
    l0 = rt.launches()
    P = dab.permutedims(M)
    l1 = rt.launches()
    Q = dab.copy_transposed(dab.transpose(M))
    assert l1 - l0 == rt.launches() - l1
    _same(dab.to_array(P), m.T)
    _same(dab.to_array(Q), dab.to_array(P))
    for x in (V, R, M, P, Q):
        x.close()
    rt.sync()
    assert dab.registry_size() == r0


def test_refusals_launch_nothing(dab, rt8):
    """Every error of the contract raises before any allocation or launch and leaves the registry unchanged."""
    A = dab.distribute(np.arange(60.0).reshape(3, 4, 5))
    D = dab.dzeros((5, 3, 4))
    D32 = dab.dzeros((5, 3, 4), dtype=np.float32)
    D2 = dab.dzeros((5, 12))
    cases = [(dab.ArgumentError, lambda: dab.permutedims(A, (1, 2))),
             (dab.ArgumentError, lambda: dab.permutedims(A, (2, 2, 1))),
             (dab.ArgumentError, lambda: dab.permutedims(A, (1, 2, 4))),
             (dab.DimensionMismatch, lambda: dab.permutedims_(D, A, (1, 2, 3))),
             (dab.DimensionMismatch, lambda: dab.permutedims_(D2, A, (3, 1, 2))),
             (dab.ArgumentError, lambda: dab.permutedims_(A, A, (1, 2, 3))),
             (dab.UnsupportedError, lambda: dab.permutedims_(D32, A, (3, 1, 2))),
             (dab.UnsupportedError, lambda: dab.permutedims(A[0:2, :, :], (3, 1, 2))),
             (TypeError, lambda: dab.permutedims(A))]
    for exc, f in cases:
        rt8.sync()
        l0, r0 = rt8.launches(), dab.registry_size()
        with pytest.raises(exc):
            f()
        assert (rt8.launches(), dab.registry_size()) == (l0, r0), exc
