"""CPU tests of the NSGA-II survival entry points: workspace sizing and argument checks answer without a GPU (every
rejected call returns before any CUDA call), and DeviceNSGA2 rejects an unsupported population before touching a device."""
import ctypes

import pytest

from hebo_b200 import _lib
from hebo_b200.evolution import DeviceNSGA2


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_workspace_bytes_range_and_monotone(lib):
    for pop in (0, -1, 16385, 1 << 20):
        assert lib.hb_nsga2_workspace_bytes(pop, 8) < 0
    assert lib.hb_nsga2_workspace_bytes(100, 0) < 0
    sizes = [lib.hb_nsga2_workspace_bytes(p, 32) for p in range(1, 16385, 37)] + [lib.hb_nsga2_workspace_bytes(16384, 32)]
    assert all(s >= 0 for s in sizes)
    assert all(b >= a for a, b in zip(sizes, sizes[1:]))


def test_survive_ex_rejects_bad_arguments_before_any_cuda_call(lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    null = None
    ok = dict(X=p, F=p, C=p, FC=p, pop=300, D=4, d=3, Xn=p, Fn=p, Xcn=p, Xen=p, ws=p,
              ws_bytes=lib.hb_nsga2_workspace_bytes(300, 4), stream=null)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.hb_nsga2_survive_ex(a["X"], a["F"], a["C"], a["FC"], a["pop"], a["D"], a["d"], a["Xn"], a["Fn"],
                                       a["Xcn"], a["Xen"], a["ws"], a["ws_bytes"], a["stream"])
    for name in ("X", "F", "C", "FC", "Xn", "Fn", "Xcn", "Xen"):
        assert call(**{name: null}) == _lib.HB_ERR_INVALID, name
    assert call(pop=16385, ws_bytes=1 << 30) == _lib.HB_ERR_INVALID
    assert call(pop=0) == _lib.HB_ERR_INVALID
    assert call(d=5) == _lib.HB_ERR_INVALID
    assert call(ws=null) == _lib.HB_ERR_INVALID                                  # pop > 256 needs the workspace
    assert call(ws_bytes=ok["ws_bytes"] - 1) == _lib.HB_ERR_INVALID             # short workspace
    # the workspace-free entry keeps its pop <= 256 limit
    assert lib.hb_nsga2_survive(p, p, p, p, 300, 4, 3, p, p, p, p, null) == _lib.HB_ERR_INVALID


@pytest.mark.parametrize("pop", [16385, 1, 0])
def test_device_nsga2_rejects_unsupported_population_before_touching_a_device(pop):
    with pytest.raises(ValueError):
        DeviceNSGA2(["real", "real"], [0.0, 0.0], [1.0, 1.0], 2, lambda xc, xe, g: None, pop=pop, device="cuda:63")
