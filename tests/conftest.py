import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with `-m gpu`)")


@pytest.fixture(scope="session", autouse=True)
def _hostmem_session():
    """``DAB_HOSTMEM=1`` (never set by the driver's tiers; used by tests/test_cpu_host.py in a subprocess): install the host-memory
    emulation of the C ABI (tests/hostmem_abi.py) for the whole session, so that the ``-m gpu`` test modules can be executed on a
    CPU-only machine as a regression test of the HOST runtime (tracer, kernel routing, stride tables, layouts, halo / exchange plans,
    error contracts).  Says nothing about the CUDA kernels."""
    if os.environ.get("DAB_HOSTMEM") != "1":
        yield None
        return
    import darray_b200  # noqa: F401
    import hostmem_abi

    lib_mod = sys.modules["darray_b200._lib"]
    bc_mod = sys.modules["darray_b200._broadcast"]
    fake = hostmem_abi.HostMemABI()
    lib_mod._lib = fake
    real_codegen = bc_mod.codegen

    def recording_codegen(e):
        src = real_codegen(e)
        fake.exprs[src.encode()] = e
        return src

    bc_mod.codegen = recording_codegen
    yield fake


@pytest.fixture(scope="session")
def dab():
    import darray_b200

    return darray_b200


@pytest.fixture()
def rt8(dab):
    """8 workers on the one visible GPU: multi-chunk layouts (grids, fibres, halos) on a single-GPU box."""
    rt = dab.init(workers_per_rank=8, use_dist=False)
    yield rt
    dab.d_closeall()


@pytest.fixture()
def rt1(dab):
    rt = dab.init(workers_per_rank=1, use_dist=False)
    yield rt
    dab.d_closeall()


@pytest.fixture()
def rt2(dab):
    rt = dab.init(workers_per_rank=2, use_dist=False)
    yield rt
    dab.d_closeall()


@pytest.fixture()
def hostmem(dab, monkeypatch):
    """CPU-only runs of the HOST logic above the C ABI: installs ``tests/hostmem_abi.py`` (an emulation of the entry points that
    ``sort`` drives, over host memory) in place of libdab200.so for one test, and removes every trace of it afterwards.  Test
    infrastructure; the product never sees it."""
    import sys

    import hostmem_abi

    lib_mod = sys.modules["darray_b200._lib"]
    rt_mod = sys.modules["darray_b200.runtime"]
    bc_mod = sys.modules["darray_b200._broadcast"]
    if rt_mod._RT is not None:                              # a real runtime left by an earlier GPU test: close it properly first,
        dab.d_closeall()                                     # the emulation must not share process state with it
        rt_mod._RT.shutdown()
    saved_lib, saved_rt = lib_mod._lib, None
    fake = hostmem_abi.HostMemABI()
    lib_mod._lib = fake
    real_codegen = bc_mod.codegen

    def recording_codegen(e):                                  # lets the emulated dab_mapreduce_expr find the tree behind a source string
        src = real_codegen(e)
        fake.exprs[src.encode()] = e
        return src

    monkeypatch.setattr(bc_mod, "codegen", recording_codegen)
    try:
        yield fake
    finally:
        try:
            dab.d_closeall()
            if rt_mod._RT is not None:
                rt_mod._RT.shutdown()                      # ctx = None: late finalizers become no-ops instead of reaching the real library
        finally:
            rt_mod._RT = saved_rt
            lib_mod._lib = saved_lib
