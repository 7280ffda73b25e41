"""CPU tests of the samplesort restatement (reference src/sort.jl; its own test is test/darray.jl:1015-1025:
``sort(Array(d)) == Array(sort(d; sample=s))`` for 10^0..10^6 elements, T in (Int, Float64), four kinds of ``sample``)."""
import numpy as np
import pytest

from oracle import darray_oracle as orc


def _data(T, n, rng):
    if np.dtype(T).kind == "i":
        return rng.integers(np.iinfo(T).min, np.iinfo(T).max, n, dtype=T)      # rand(Int, n): the full range
    return rng.random(n).astype(T)


@pytest.mark.parametrize("T", [np.int64, np.float64])
@pytest.mark.parametrize("i", range(0, 6))
def test_oracle_sort_reference_test(T, i):
    rng = np.random.default_rng(100 + i)
    n = 10 ** i
    a = _data(T, n, rng)
    for nw in (1, 2, 8):
        d = orc.distribute(a, nworkers=nw)
        for sample in (True, False, (a.min(), a.max()), _data(T, min(n, 512), rng)):
            d2, b = orc.darray_sort(d, sample)
            a2 = orc.to_array(d2)
            assert len(a2) == n and np.array_equal(np.sort(a), a2)
            assert len(b) == len(d.pids) + 1 and np.all(b[1:-1][:-1] <= b[1:-1][1:])
            assert d2.pids == [d.pids[k] for k in range(len(d.pids)) if k in [d.pids.index(p) for p in d2.pids]]
            assert all(len(c) > 0 for c in d2.chunks) and sum(len(c) for c in d2.chunks) == n
            assert d2.cuts[0][0] == 1 and d2.cuts[0][-1] == n + 1


def test_oracle_sort_details():
    # the sample picks sorted[1:div(llp,ss):llp]: more than 512 keys when 512 < llp < 1024 (step 1)
    assert list(orc.sort_sample_indices(1000)) == list(range(1000))
    assert list(orc.sort_sample_indices(2048)) == list(range(0, 2048, 4))
    assert len(orc.sort_sample_indices(1025)) == 513
    with pytest.raises(ZeroDivisionError):
        orc.sort_sample_indices(0)
    # boundaries: first sample replaced by typemin, typemax appended
    b = orc.sort_boundaries_from_samples(np.array([5, 1, 9, 3, 7, 2], dtype=np.int64), 3, np.int64)
    assert list(b) == [np.iinfo(np.int64).min, 3, 7, np.iinfo(np.int64).max]
    # split scan: piece i = leading run of elements NOT > boundaries[i+1]
    s = np.array([1, 2, 3, 3, 4, 8, 9], dtype=np.int64)
    assert orc.sort_split_points(s, b) == [4, 5, 7]
    # isless order: -0.0 before +0.0, NaN last, and a NaN never exceeds a boundary (it stays in the piece being scanned)
    v = np.array([0.0, np.nan, -0.0, 1.0, -np.inf], dtype=np.float64)
    sv = orc.jl_sort(v)
    assert np.signbit(sv[1]) and not np.signbit(sv[2]) and sv[0] == -np.inf and np.isnan(sv[-1])
    bf = np.array([-np.inf, 0.0, np.inf])
    assert orc.sort_split_points(sv, bf) == [3, 5]
    # uniform sample with a full-range Int64 min/max: abs(ub - lb) wraps like the reference's machine arithmetic
    lo, hi = np.int64(-9 * 10 ** 18), np.int64(9 * 10 ** 18)
    u = orc.sort_uniform_sample(lo, hi, 4, np.int64)
    wrapped = (int(hi) - int(lo) + 2 ** 63) % 2 ** 64 - 2 ** 63
    assert u[0] == lo and u[1] == np.int64(np.rint(float(lo) + abs(wrapped) / 4))
    with pytest.raises(ValueError):
        orc.sort_uniform_sample(-np.inf, 1.0, 2, np.float64)


def test_host_boundary_logic_matches_oracle():
    from darray_b200 import _sort
    rng = np.random.default_rng(3)
    for T in (np.int64, np.float64, np.float32, np.int32):
        dt = np.dtype(T)
        s = _data(T, 700, rng)
        for nparts in (1, 2, 3, 8):
            assert np.array_equal(_sort.boundaries_from_samples(s, nparts, dt), orc.sort_boundaries_from_samples(s, nparts, dt))
            assert np.array_equal(_sort.uniform_sample(s.min(), s.max(), nparts, dt), orc.sort_uniform_sample(s.min(), s.max(), nparts, dt))


# ---- sort(d; by = f): oracle, the dab_sort_by_key composition, and the host flow of _sort.py over the host-memory ABI emulation ----

def _by_cases(T):
    """(traced closure for the product, NumPy-vectorised twin for the oracle)."""
    import darray_b200 as dab
    cases = [(lambda x: -x, lambda v: -v), (lambda x: abs(x), lambda v: np.abs(v)), (lambda x: x, lambda v: v)]
    if np.dtype(T).kind == "i":
        cases += [(lambda x: dab.rem(x, 7), lambda v: np.fmod(v, np.dtype(T).type(7))),              # many equal keys: stability
                  (lambda x: x * 0.5, lambda v: v * 0.5),                                            # Float64 keys of Int values
                  (lambda x: x > 3, lambda v: (v > 3).astype(np.int32))]                             # Bool keys
    else:
        cases += [(lambda x: dab.floor(x * 4), lambda v: np.floor(v * np.dtype(T).type(4))),
                  (lambda x: dab.ifelse(x > 0.5, x, 1 - x), lambda v: np.where(v > 0.5, v, 1 - v))]
    return cases


def _by_data(T, n, rng):
    if np.dtype(T).kind == "i":
        return rng.integers(-50, 50, n).astype(T)
    a = rng.random(n).astype(T)
    if n >= 8:                                                                   # signed zeros, infinities and NaNs among the values
        a[rng.integers(0, n, 3)] = [-0.0, np.inf, -np.inf]
    return a


def _multiset_contains(big, small):
    ub, cb = np.unique(big.view(np.uint8).reshape(len(big), -1), axis=0, return_counts=True)
    us, cs = np.unique(small.view(np.uint8).reshape(len(small), -1), axis=0, return_counts=True)
    have = {bytes(r): c for r, c in zip(ub, cb)}
    return all(have.get(bytes(r), 0) >= c for r, c in zip(us, cs))


def test_oracle_sort_by():
    rng = np.random.default_rng(5)
    for T in (np.int64, np.float64, np.float32, np.int32):
        tmax = np.array([orc._typemax(np.dtype(T))], dtype=T)
        for n in (1, 10, 1000, 5000):
            a = _by_data(T, n, rng)
            for _, nby in _by_cases(T):
                ka = nby(a)
                with np.errstate(invalid="ignore"):
                    kept = ~(ka > nby(tmax)[0])                 # the reference never ships an element whose key exceeds by(typemax(T))
                want = a[kept][orc.jl_sortperm_stable(ka[kept])]
                for nw in (1, 3, 8):
                    if n < nw:
                        continue
                    # one worker: ONE piece, cut at the first key above by(typemax(T)); several workers: only the tail behind the LAST
                    # split point is lost, so a key function whose maximum is by(typemax(T)) loses nothing
                    try:
                        d2, b = orc.darray_sort(orc.distribute(a, nworkers=nw), True, by=nby)
                    except ValueError:
                        assert not kept.all()
                        continue
                    got = orc.to_array(d2)
                    k = nby(got)
                    assert _multiset_contains(a, got) and (len(got) == n if kept.all() else len(got) <= n)
                    with np.errstate(invalid="ignore"):
                        assert not np.any(k[1:] < k[:-1])                             # ordered by key
                    if nw == 1:
                        assert np.array_equal(got, want, equal_nan=True)              # sort(a; by) of the shipped elements, stable
    # NaN keys are equal to each other: they keep input order at the end; -0.0 keys sort before +0.0 keys
    v = np.array([3.0, np.nan, -0.0, 0.0, 1.0, np.nan, -0.0], dtype=np.float64)
    tag = np.arange(7, dtype=np.float64)
    assert list(orc.jl_sortperm_stable(v)) == [2, 6, 3, 4, 0, 1, 5]
    assert list(orc.jl_sort_by(tag, lambda t: v[t.astype(int)])) == [2, 6, 3, 4, 0, 1, 5]


def test_sort_by_key_composition_matches_stable_order():
    """The packed-word composition of dab_sortby.cu (emulated step by step in tests/hostmem_abi.py) against a stable isless argsort."""
    import ctypes as C

    import hostmem_abi as hm
    fake = hm.HostMemABI()
    rng = np.random.default_rng(11)
    for code, kt in ((hm.F32, np.float32), (hm.F64, np.float64), (hm.I32, np.int32), (hm.I64, np.int64)):
        for n in (1, 2, 33, 4097):
            if np.dtype(kt).kind == "f":
                keys = rng.standard_normal(n).astype(kt)
                keys[rng.integers(0, n, max(1, n // 8))] = rng.choice(np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf], dtype=kt), max(1, n // 8))
                keys = np.round(keys, 1)                                            # many ties
                if n > 30:                                                          # NaNs with different payloads are still ONE key
                    raw = keys.view(np.uint32 if kt == np.float32 else np.uint64)
                    raw[5] = raw.dtype.type(0x7FC00123 if kt == np.float32 else 0x7FF8000000000123)
                    raw[9] = raw.dtype.type(0xFFC00001 if kt == np.float32 else 0xFFF8000000000001)
            else:
                keys = rng.integers(np.iinfo(kt).min, np.iinfo(kt).max, n, dtype=kt)
                keys[rng.integers(0, n, max(1, n // 2))] = kt(7)
                if n > 30:
                    keys[:4] = [np.iinfo(kt).min, np.iinfo(kt).max, -1, 0]
            for vt in (np.float32, np.int64):
                vals = np.arange(n).astype(vt)
                out = np.empty_like(vals)
                need = C.c_size_t()
                fake.dab_sort_by_key_scratch_bytes(code, n, C.byref(need))
                scratch = np.zeros(need.value + 16, dtype=np.uint8)
                sp = (scratch.ctypes.data + 15) & ~15
                assert fake.dab_sort_by_key(None, code, keys.ctypes.data, vals.itemsize, vals.ctypes.data, out.ctypes.data, sp, need.value, n) == 0
                assert np.array_equal(out, vals[orc.jl_sortperm_stable(keys)]), (kt, vt, n)
    # the radix-key bijection itself: monotone in isless order and invertible
    f = np.array([-np.inf, -1.5, -0.0, 0.0, 1e-30, 2.0, np.inf, np.nan], dtype=np.float32)
    e = hm.radix_enc(f.view(np.uint32), hm.F32)
    assert np.all(e[1:] > e[:-1]) and np.array_equal(hm.radix_dec(e, hm.F32), f.view(np.uint32))
    d = f.astype(np.float64)
    e = hm.radix_enc(d.view(np.uint64), hm.F64)
    assert np.all(e[1:] > e[:-1]) and np.array_equal(hm.radix_dec(e, hm.F64), d.view(np.uint64))


@pytest.mark.parametrize("T", [np.int64, np.float64, np.float32, np.int32])
@pytest.mark.parametrize("nw", [1, 2, 8])
def test_host_sort_flow_with_and_without_by(hostmem, dab, T, nw):
    """_sort.py end to end on the host-memory ABI: result, boundaries and result layout equal the oracle's, for every `sample` kind."""
    rt = dab.init(workers_per_rank=nw, use_dist=False)
    rng = np.random.default_rng(17 + nw)
    for n in (nw, 97, 3000):
        a = _by_data(T, n, rng)
        od = orc.distribute(a, nworkers=nw)
        d = dab.distribute(a)
        assert d.layout.indices == od.indices
        smp = _by_data(T, 64, rng)
        lohi = (T(-60), T(60)) if np.dtype(T).kind == "i" else (T(0), T(1))
        for sample in (True, False, lohi, smp):
            for tby, nby in [(None, None)] + _by_cases(T):
                try:
                    want, wb = orc.darray_sort(od, sample, by=nby)
                except ValueError:                              # every key exceeds by(typemax(T)): nothing is shipped (see the oracle's docstring)
                    with pytest.raises(dab.ArgumentError):
                        dab.sort_with_boundaries(d, sample, tby)
                    continue
                got, gb = dab.sort_with_boundaries(d, sample, tby)
                assert np.array_equal(gb, wb, equal_nan=True), (n, sample is True, tby)
                assert got.layout.indices == want.indices and list(got.layout.pids) == list(want.pids)
                ga, wa = dab.to_array(got), orc.to_array(want)
                assert ga.dtype == wa.dtype and np.array_equal(ga.view(np.uint8), wa.view(np.uint8)), (n, sample is True, tby)
                got.close()
        d.close()
    assert hostmem.launches > 0
    rt.shutdown()


def test_sort_by_key_element_code_host_replay(tmp_path):
    """tools/sortby_host_check.cu: the per-element code the sort-by-key KERNELS run (dab_sortby_core.cuh, __host__ __device__) replayed on
    the host -- words packed by ``sortby_word``, std::sort in place of K11, permutation by ``sortby_source`` -- against std::stable_sort
    in isless order, for the four key types (ties, signed zeros, infinities, NaN payloads, integer extremes)."""
    import os
    import shutil
    import subprocess
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "sortby_host_check")
    subprocess.check_call([nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "distributedarrays.jl_b200", "csrc"),
                           "-o", exe, os.path.join(root, "tools", "sortby_host_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "sortby_host_check: ok" in out.stdout, out.stdout + out.stderr


def test_host_sort_flow_by_with_nan_values_and_nan_keys(hostmem, dab):
    """NaN values, NaN keys (sqrt of negatives) and signed zeros through the keyed samplesort: NaN keys tie and keep input order behind
    everything else, a NaN key never exceeds a boundary -- product flow (emulated kernels) and oracle agree bit for bit."""
    rng = np.random.default_rng(4)
    for nw in (1, 3, 8):
        dab.init(workers_per_rank=nw, use_dist=False)
        for T in (np.float64, np.float32):
            for n in (nw, 50, 2000):
                a = rng.standard_normal(n).astype(T)
                a[rng.integers(0, n, max(1, n // 10))] = np.nan
                a[rng.integers(0, n, max(1, n // 10))] = -0.0
                od, d = orc.distribute(a, nworkers=nw), dab.distribute(a)
                for tby, nby in [(lambda x: x * 1, lambda v: v * 1), (lambda x: abs(x), np.abs), (lambda x: dab.sqrt(x), lambda v: np.sqrt(v)),
                                 (lambda x: dab.ifelse(x > 0, x, 0 * x), lambda v: np.where(v > 0, v, 0 * v))]:
                    for sample in (True, a[rng.integers(0, n, min(n, 32))]):
                        try:
                            with np.errstate(all="ignore"):
                                want, wb = orc.darray_sort(od, sample, by=nby)
                        except ValueError:
                            with pytest.raises(dab.ArgumentError):
                                dab.sort_with_boundaries(d, sample, tby)
                            continue
                        got, gb = dab.sort_with_boundaries(d, sample, tby)
                        assert np.array_equal(gb, wb, equal_nan=True) and got.layout.indices == want.indices
                        assert np.array_equal(dab.to_array(got).view(np.uint8), orc.to_array(want).view(np.uint8)), (nw, T, n)
                d.close()


# ---- tests/test_gpu_sort_paths.py: its digit-set data, its model and its tile-shape premise, checked without a GPU ---------------

def test_sort_paths_digit_set_generator():
    """Every named case of the onesweep path tests has exactly its intended non-constant digits, for every dtype, keys only and pairs;
    for pairs of floats only the NaN case holds NaNs (several payloads, both signs), and those are exactly the keys that collapse to the
    top radix key.  The outliers differ from the rest in one key, and one-digit-per-tile data is constant in digit 0 inside every tile."""
    import test_gpu_sort_paths as sp
    rng = np.random.default_rng(31)
    for T in map(np.dtype, sp.DTYPES):
        w, U = T.itemsize, sp.UINT[T.itemsize]
        sets = sp.digit_sets(w)
        assert sets["odd"][0] > 0 and sets["odd"][-1] < w - 1 and len(sets["odd"]) % 2 == 1
        assert sets["even"][0] > 0 and sets["even"][-1] < w - 1 and len(sets["even"]) % 2 == 0
        for pairs in (False, True):
            tile = (sp.PAIRS_TILE if pairs else sp.KEYS_TILE)[w]
            for n in (1025, 3 * tile + 1):
                for name in sp.SMALL_NAMES:
                    a, act, outl = sp.make_case(T, name, n, tile, rng, pairs)
                    assert a.dtype == T and a.size == n
                    sp.check_premise(a, act, outl, pairs)
                    if name in sets:
                        assert act == sets[name]
                    r = sp.pairs_radix(a) if pairs else sp.keys_radix(a)
                    if outl is not None:                                    # one key differs from the n - 1 others
                        assert sorted(np.unique(r, return_counts=True)[1]) == [1, n - 1]
                    if name == "tile_digit":
                        d0 = (r & U(0xFF)).astype(np.int64)
                        t = np.arange(n) // tile
                        assert np.array_equal(d0, t * 97 % 256)
                    if pairs and T.kind == "f":
                        nan = np.isnan(a)
                        assert np.array_equal(nan, r == ~U(0))
                        if name == "all_nan":
                            raw = a.view(U)
                            assert nan.any() and np.unique(raw[nan]).size > 10 and np.unique(raw[nan] >> U(8 * w - 1)).size == 2
                        else:
                            assert not nan.any()
    # the premise check itself: a digit with one odd key out is non-constant, a constant one is not
    k = np.full(5000, 0x11223344, dtype=np.uint32)
    assert sp.active_digits(k) == ()
    k[4999] = 0x11223345
    assert sp.active_digits(k) == (0,) and sp.largest_bin(k, 0) == 4999


def test_sort_paths_model_matches_oracle():
    """The model of the path tests against the oracle: dec(sort(enc)) is Julia's sort on NaN-free data (signed zeros, infinities, ties),
    and the stable argsort of the collapsed key is Julia's stable sortperm (NaNs equal to each other) with or without NaNs."""
    import hostmem_abi as hm
    import test_gpu_sort_paths as sp
    rng = np.random.default_rng(32)
    for T in map(np.dtype, sp.DTYPES):
        for name in ("all", "odd", "low_top", "outlier_first", "tile_digit"):
            a, _, _ = sp.make_case(T, name, 20000, sp.PAIRS_TILE[T.itemsize], rng, pairs=True)     # NaN-free
            a = a.copy()
            a[rng.integers(0, a.size, 2000)] = a[rng.integers(0, a.size, 2000)]                   # ties
            if T.kind == "f":
                a[rng.integers(0, a.size, 300)] = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf], dtype=T), 300)
            U = sp.UINT[T.itemsize]
            assert np.array_equal(sp.model_sort(a), orc.jl_sort(a).view(U)), (T, name)
            perm, ek = sp.model_pairs(a)
            assert np.array_equal(perm, orc.jl_sortperm_stable(a)), (T, name)
            assert np.array_equal(hm.radix_dec(ek, sp.CODE[T]), orc.jl_sort(a).view(U))
        if T.kind == "f":
            a, _, _ = sp.make_case(T, "all_nan", 20000, sp.PAIRS_TILE[T.itemsize], rng, pairs=True)
            assert np.isnan(a).any()
            assert np.array_equal(sp.model_pairs(a)[0], orc.jl_sortperm_stable(a))


def test_sort_paths_tile_shapes_match_the_kernel():
    """The tile sizes and residency the path tests build their size classes from are the ones dab_sort.cu instantiates: keys only 256 x 32
    (4-byte keys) and 256 x 16 (8-byte), pairs 256 x 16 and 256 x 10, each at most 3 CTAs per SM by its shared memory (228 KiB per H100
    SM, 1 KiB of it reserved per CTA), so that the persistent class really gives every resident CTA 4 or more tiles."""
    import os
    import re

    import test_gpu_sort_paths as sp
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "distributedarrays.jl_b200", "csrc", "dab_sort.cu")).read()
    body = src[src.index("int32_t sort_t("):]
    body = body[:body.index("\n}\n")]
    pairs_part = body[body.index("if constexpr (!std::is_void<P>::value)"):body.index("} else if constexpr (sizeof(U) == 8)")]
    keys_part = body[body.index("} else if constexpr (sizeof(U) == 8)"):]
    inst = r"sort_passes<T, P, (\d+), (\d+), (\d+)>"
    smem_line = ("constexpr size_t smem = 2 * (size_t)TILE * (sizeof(U) + (PAIRS ? 4 : 0)) + (size_t)(THREADS / 32) * 1024 + 1024 + 32;")
    assert smem_line in src
    for part, tiles, pair_bytes in ((pairs_part, sp.PAIRS_TILE, 4), (keys_part, sp.KEYS_TILE, 0)):
        got = [tuple(map(int, m)) for m in re.findall(inst, part)]
        assert len(got) == 2, got
        for (threads, kpt, minb), width in zip(got, (8, 4)):                # the 8-byte branch comes first in both
            assert threads * kpt == tiles[width] and minb == sp.CTAS_PER_SM
            smem = 2 * threads * kpt * (width + pair_bytes) + threads // 32 * 1024 + 1024 + 32
            assert smem <= 227 * 1024 and (228 * 1024) // (smem + 1024) <= sp.CTAS_PER_SM, (width, pair_bytes, smem)
