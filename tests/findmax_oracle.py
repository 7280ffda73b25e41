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


def global_index(pos: np.ndarray, cdims=(), offs=(), gdims=()) -> np.ndarray:
    """Chunk-local 0-based positions -> 1-based global linear indices (``FmGlobal``): column-major unravel in the chunk dims, plus the
    offsets, ravel in the global dims.  No dims: the position plus one."""
    pos = np.asarray(pos, dtype=np.int64)
    if not len(cdims):
        return pos + 1
    c = np.unravel_index(pos, [int(v) for v in cdims], order="F")
    return np.ravel_multi_index(tuple(cc + int(o) for cc, o in zip(c, offs)), [int(v) for v in gdims], order="F").astype(np.int64) + 1


def find_carried(which: int, m: np.ndarray, ii: np.ndarray):
    """The dims reduction over axis 1 of (inner, red, outer) values ``m`` that carry the indices ``ii`` (a later pass, or the fold on the
    owner): the largest key, then the smallest carried index; -1 marks "no element" and is skipped.  A fibre with no element gives (0, -1),
    the kernels' empty accumulator.  Of two entries with equal key that carry the same index, the one at the smaller position is kept.
    The kernels keep it only where they meet the two in position order: along one thread's walk, or in two splits (the finish fold runs
    in split order).  Within one split of the lead kernel, entries in different lanes are folded lane by lane, so the lower lane's entry
    is kept even at a larger position; that is not a contract, and no test should rely on either outcome there.
    Returns (values, indices), each (inner, outer)."""
    keys = order_keys(which, m.ravel(order="F")).reshape(m.shape, order="F")
    ok = ii != -1
    kk = np.where(ok, keys, np.uint64(0))
    top = kk.max(axis=1, keepdims=True)
    cand = ok & (kk == top)
    small = np.where(cand, ii, np.iinfo(np.int64).max).min(axis=1, keepdims=True)
    pos = np.argmax(cand & (ii == small), axis=1)                   # the first position of the winning (key, index)
    rows = np.arange(m.shape[0])[:, None], np.arange(m.shape[2])[None, :]
    vals = m[rows[0], pos, rows[1]]
    idx = ii[rows[0], pos, rows[1]]
    none = ~ok.any(axis=1)
    vals[none] = 0
    idx[none] = -1
    return vals, idx


# ---- launch model of dab_findminmax.cu ----------------------------------------------------------------------------------------------
# A mirror of the host-side dispatch: flat_grid (dab_reduce_traits.cuh), dim_nsplit and launch_fmdim.  tests/test_gpu_findmax_paths.py
# builds each case to reach one of its labels and asserts that premise here.
RD_THREADS, RD_UNROLL = 256, 4
MAX_REDUCE_BLOCKS = 262144
CTAS_PER_SM = 8                 # the most 256-thread CTAs an SM holds: a grid beyond sm_count * 8 CTAs loops whatever the occupancy
MIN_SM_COUNT = 9                # the fewest SMs at which case_table reaches every label (an empty split needs 258 or more splits)


def _ceil(a: int, b: int) -> int:
    return -(-a // b)


def dim_nsplit(have: int, target: int, max_split: int) -> int:
    max_split = max(max_split, 1)
    want = 1 if have >= target else _ceil(target, have)
    return min(want, max_split, 1024)


def flat_grid(dtype, addr16: int, n: int) -> dict:
    """The whole-chunk kernel's geometry for n elements at an address that is ``addr16`` mod 16: the unaligned head, the tiles of
    RD_THREADS * RD_UNROLL 16-byte vectors, the grid and tiles per CTA, the vectors after the last whole tile and the tail elements."""
    size = np.dtype(dtype).itemsize
    vpt = 16 // size
    head = min(((16 - addr16) & 15) // size, n)
    tiles = (n - head) // (vpt * RD_THREADS * RD_UNROLL)
    k = 2
    if _ceil(tiles, k) > MAX_REDUCE_BLOCKS:
        k = _ceil(tiles, MAX_REDUCE_BLOCKS)
    nvec = (n - head) // vpt
    return dict(head=head, tiles=tiles, grid=max(1, _ceil(tiles, k)), tiles_per_cta=k, rem_vecs=nvec - tiles * RD_THREADS * RD_UNROLL,
                tail=n - head - nvec * vpt, vpt=vpt, tile=vpt * RD_THREADS * RD_UNROLL)


def fmdim_plan(dtype, inner: int, red: int, outer: int, addr16: int, has_idx: bool, sm_count: int) -> dict:
    """What launch_fmdim runs for one (inner, red, outer) pass: the kernel ("whole", "lead", "strided", "vec"), the lanes G per run of
    the lead kernel, the split count and the splits' [lo, hi) (hi <= lo: an empty split), the launch count, and whether the persistent
    grid certainly loops (more than sm_count * 8 CTAs of work)."""
    size = np.dtype(dtype).itemsize
    vpt = 16 // size
    nout = inner * outer
    target = sm_count * 8
    if not has_idx and inner == 1 and outer == 1 and red >= 1 << 16:
        return dict(kernel="whole", G=0, vec=False, nsplit=1, bounds=[(0, red)], empty=False, launches=2, loops=False,
                    flat=flat_grid(dtype, addr16, red))
    vec = not has_idx and size >= 4 and inner > 1 and inner % vpt == 0 and addr16 == 0 and nout // vpt >= 4096
    if inner == 1:
        G = 32 if red >= 64 else 4
        nsplit = dim_nsplit(outer, target * (RD_THREADS // G), red // (G * 64))
        ctas = _ceil(outer * nsplit, RD_THREADS // G)
        kernel = "lead"
    else:
        G = 0
        base = _ceil(nout // vpt, RD_THREADS) if vec else _ceil(nout, RD_THREADS)
        nsplit = dim_nsplit(base, 4 * target, red // 256)
        ctas = base * nsplit
        kernel = "vec" if vec else "strided"
    L = _ceil(red, nsplit)
    bounds = [(s * L, min(s * L + L, red)) for s in range(nsplit)]
    return dict(kernel=kernel, G=G, vec=vec, nsplit=nsplit, bounds=bounds, empty=any(hi <= lo for lo, hi in bounds),
                launches=2 if nsplit > 1 else 1, loops=ctas > sm_count * CTAS_PER_SM)


def plan_labels(plan: dict, dtype, inner: int, outer: int, addr16: int, has_idx: bool) -> set:
    """The labels a plan reaches: its kernel (lead4 / lead32 / strided / vec / whole), "_split" and "_idx" suffixes, and "empty_split",
    "grid_loop" and "bool_vec_shape" (a Bool pass of a shape that would take the 16-byte kernel at 4 bytes)."""
    k = plan["kernel"]
    name = f"lead{plan['G']}" if k == "lead" else k
    name += "_split" if plan["nsplit"] > 1 else ""
    name += "_idx" if has_idx else ""
    out = {name}
    if plan["empty"]:
        out.add("empty_split")
    if plan["loops"]:
        out.add("grid_loop")
    if np.dtype(dtype) == np.bool_ and not has_idx and inner > 1 and inner % 16 == 0 and addr16 == 0 and inner * outer // 16 >= 4096:
        out.add("bool_vec_shape")
    return out


ALL_LABELS = {"whole", "lead4", "lead32", "lead32_split", "strided", "strided_split", "vec", "vec_split", "lead4_idx", "lead32_idx",
              "lead32_split_idx", "strided_idx", "strided_split_idx", "empty_split", "grid_loop", "bool_vec_shape"}


def case_table(sm_count: int):
    """The dims cases of tests/test_gpu_findmax_paths.py: (name, label the case is built to reach, dtype -> (inner, red, outer, element
    phase), index input).  Sizes follow the SM count; boundaries are taken on both sides (red 63 / 64 and 65535 / 65536, nout / VPT 4095 /
    4096, inner % VPT != 0, a base one element off 16 bytes).

    An empty split: a strided pass of one CTA of outputs gets n = min(4 * sm_count * 8, 1024) splits when red >= 256 n.  With red =
    256 n + 1 each split holds 257 elements, so the last n - ceil(red / 257) splits are empty; there are some once n >= 258, that is from
    MIN_SM_COUNT SMs on (3 of 1024 on 32 SMs or more).  Fewer SMs cannot leave a split empty: every split then holds at least 256
    elements and there are at most 256 of them."""
    if sm_count < MIN_SM_COUNT:
        raise ValueError(f"the case table needs {MIN_SM_COUNT} or more SMs, not {sm_count}")
    v = lambda dt: 16 // np.dtype(dt).itemsize
    t = sm_count * CTAS_PER_SM
    red_empty = 256 * min(4 * t, 1024) + 1
    return [
        ("lead4_red63", "lead4", lambda dt: (1, 63, 37, 0), False),
        ("lead32_red64", "lead32", lambda dt: (1, 64, 37, 1), False),
        ("lead32_split", "lead32_split", lambda dt: (1, 2048 * 6 + 5, 3, 0), False),
        ("lead32_split_red65535", "lead32_split", lambda dt: (1, 65535, 1, 0), False),
        ("whole_red65536", "whole", lambda dt: (1, 65536, 1, 0), False),
        ("whole_misaligned", "whole", lambda dt: (1, 3 * 65536 + 77, 1, 1), False),
        ("lead4_loop", "grid_loop", lambda dt: (1, 5, t * 64 + 101, 0), False),
        ("lead32_loop", "grid_loop", lambda dt: (1, 64, t * 8 + 9, 0), False),
        ("strided", "strided", lambda dt: (3, 300, 5, 0), False),
        ("strided_split", "strided_split", lambda dt: (5, 256 * 8 + 3, 7, 1), False),
        ("strided_empty_split", "empty_split", lambda dt: (2, red_empty, 1, 0), False),
        ("strided_loop", "grid_loop", lambda dt: (256 * t + 1, 2, 1, 0), False),
        ("vec_nout4096", "vec", lambda dt: (8 * v(dt), 3, 512, 0), False),
        ("strided_nout4095", "strided", lambda dt: (4095 * v(dt), 3, 1, 0), False),
        ("strided_inner_mod_vpt", "strided", lambda dt: (4097 * v(dt) - 1, 3, 1, 0), False),
        ("strided_base_misaligned", "strided", lambda dt: (8 * v(dt), 3, 512, 1), False),
        ("vec_split", "vec_split", lambda dt: (4096 * v(dt), 512, 1, 0), False),
        ("strided_split_nout4095", "strided_split", lambda dt: (4095 * v(dt), 512, 1, 0), False),
        ("vec_loop", "grid_loop", lambda dt: (v(dt) * 256 * (t + 1), 2, 1, 0), False),
        ("lead4_idx", "lead4_idx", lambda dt: (1, 63, 37, 0), True),
        ("lead32_idx", "lead32_idx", lambda dt: (1, 64, 37, 1), True),
        ("lead32_split_idx", "lead32_split_idx", lambda dt: (1, 2048 * 6 + 5, 3, 0), True),
        ("lead32_split_idx_red65536", "lead32_split_idx", lambda dt: (1, 65536, 1, 0), True),
        ("strided_idx", "strided_idx", lambda dt: (3, 300, 5, 1), True),
        ("strided_split_idx", "strided_split_idx", lambda dt: (5, 256 * 8 + 3, 7, 0), True),
        ("strided_empty_split_idx", "empty_split", lambda dt: (2, red_empty, 1, 0), True),
    ]


def case_labels(case, dtype, sm_count: int) -> set:
    name, want, shape, idx = case
    inner, red, outer, phase = shape(dtype)
    addr16 = (phase * np.dtype(dtype).itemsize) % 16
    return plan_labels(fmdim_plan(dtype, inner, red, outer, addr16, idx, sm_count), dtype, inner, outer, addr16, idx)


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
    if not hm._addr(x) or not hm._addr(out) or hm._addr(x) % np.dtype(_DT[int(dtype)]).itemsize:
        return 2                                                                           # DAB_ERR_ARG: null or misaligned
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
    has_idx = idx_in is not None and bool(hm._addr(idx_in))
    if nd < 0 or nd > 8 or (nd > 0 and not (hm._addr(cdims) and hm._addr(offs) and hm._addr(gdims))):
        return 2
    if inner * outer == 0:
        return 0
    if red == 0:
        return 3
    if not hm._addr(x) or not hm._addr(out_v) or not hm._addr(out_i) or hm._addr(x) % np.dtype(dt).itemsize:
        return 2
    cd = [int(cdims[k]) for k in range(nd)]
    of = [int(offs[k]) for k in range(nd)]
    gd = [int(gdims[k]) for k in range(nd)]
    if any(c <= 0 or o < 0 or g < o + c for c, o, g in zip(cd, of, gd)):
        return 2                                                                           # a dim that does not fit its global extent
    if has_idx and int(mapc) != 0:
        return 2                                                                           # an index input goes with the identity map
    xs = hm._view(x, inner * red * outer, dt).copy().reshape((inner, red, outer), order="F")
    f = _mapf(dtype, mapc)
    m = xs if f is None else _apply(f, xs.ravel(order="F")).reshape(xs.shape, order="F")
    if has_idx:
        ii = hm._view(idx_in, inner * red * outer, np.int64).copy().reshape((inner, red, outer), order="F")
    else:
        ii = global_index(np.arange(inner * red * outer, dtype=np.int64), cd, of, gd).reshape((inner, red, outer), order="F")
    vals, idx = find_carried(int(which), m, ii)
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
