"""CPU tests of hb_ehvi's C ABI: argument rejections before any launch, m = 0, and the workspace query.  The pointers are
fake and never dereferenced."""
import ctypes

import pytest

from hebo_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


P = ctypes.c_void_p(256)


def call(lib, front=P, n=10, K=3, samples=P, m=5, n_mc=10, ref=P, base=P, ehvi=P, ws=P, ws_bytes=None):
    if ws_bytes is None:
        ws_bytes = max(lib.hb_ehvi_workspace_bytes(n, K, m, n_mc), 0)
    return lib.hb_ehvi(front, n, K, samples, m, n_mc, ref, base, ehvi, ws, ws_bytes, None)


def test_bad_arguments_are_rejected_before_any_launch(lib):
    bad = _lib.HB_ERR_INVALID
    for K in (-1, 0, 1, _lib.HB_MAX_OBJ + 1):
        assert lib.hb_ehvi_workspace_bytes(10, K, 5, 10) < 0
        assert call(lib, K=K, ws_bytes=1 << 30) == bad, K
    for kw in (dict(n=-1), dict(m=-1), dict(n_mc=0), dict(n_mc=-3)):
        args = {**dict(n=10, K=3, m=5, n_mc=10), **kw}
        assert lib.hb_ehvi_workspace_bytes(args["n"], args["K"], args["m"], args["n_mc"]) < 0, kw
        assert call(lib, ws_bytes=1 << 30, **kw) == bad, kw
    for name in ("front", "samples", "ref", "base", "ehvi", "ws"):
        assert call(lib, **{name: None}) == bad, name
    need = lib.hb_ehvi_workspace_bytes(10, 3, 5, 10)
    assert call(lib, ws_bytes=need - 1) == bad
    assert call(lib, ws_bytes=-1) == bad
    assert call(lib, n=(1 << 31), ws_bytes=1 << 62) == bad               # row ids are int32


def test_zero_candidates_launch_nothing(lib):
    assert call(lib, m=0) == _lib.HB_OK
    assert call(lib, m=0, n=0, front=None) == _lib.HB_OK                 # an empty front needs no pointer


def test_workspace_is_monotone(lib):
    for K in range(2, _lib.HB_MAX_OBJ + 1):
        w = [lib.hb_ehvi_workspace_bytes(n, K, 100, 10) for n in range(0, 300)]
        assert all(b > 0 for b in w) and all(a <= b for a, b in zip(w, w[1:])), K
    for n in (0, 1, 31, 100, 1000):
        w = [lib.hb_ehvi_workspace_bytes(n, K, 100, 10) for K in range(2, _lib.HB_MAX_OBJ + 1)]
        assert all(a <= b for a, b in zip(w, w[1:])), n
    for K in (2, 5):
        w = [lib.hb_ehvi_workspace_bytes(50, K, m, 10) for m in (0, 1, 100, 6553, 6554, 16384, 100000)]
        assert all(a <= b for a, b in zip(w, w[1:])), K
        w = [lib.hb_ehvi_workspace_bytes(50, K, 100, n_mc) for n_mc in (1, 10, 655, 656, 10000)]
        assert all(a <= b for a, b in zip(w, w[1:])), K
    # the hypervolume of every item is held, and K - 2 level sets of n + 1 row ids per resident item
    assert lib.hb_ehvi_workspace_bytes(100, 4, 100, 10) >= (100 * 10 + 1) * 8 + 100 * 4 * 8 + 2 * 101 * 1001 * 4
