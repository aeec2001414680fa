"""Argument checks of hb_posterior_mace_ex / hb_posterior_mace, CPU only.

Every call passes fake device pointers that must never be dereferenced: each one has to fail its argument checks before
any launch.  The workspace size is an int64 and is compared as one, so a negative size is refused like a short one."""
import ctypes

import pytest

from hebo_b200 import _lib

N, D, M, MC = 300, 2, 100, 128
POINTERS = ("Xs", "x_mul", "x_add", "Zt", "alpha", "Linv", "hyp", "ws")


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def _spec(num_enum=0):
    u, e = (ctypes.c_int32 * 1)(3), (ctypes.c_int32 * 1)(2)
    spec = _lib.ModelSpec(1, num_enum, u, e, 0)
    spec._keep = (u, e)
    return spec


def _call(lib, spec=None, m=M, d=D, kern=0, m_chunk=MC, ws_bytes=None, Xe=None, meta=None, tab=None, hi=True, lo=True,
          F=True, mu=True, var=True, **null):
    p = ctypes.c_void_p(16)
    a = {k: p for k in POINTERS}
    a.update(null)
    if ws_bytes is None:
        ws_bytes = int(lib.hb_posterior_workspace_bytes(N, max(d, 1), max(m_chunk, 1)))
    sp = None if spec is None else ctypes.byref(spec)
    opt = lambda on: p if on else None
    return lib.hb_posterior_mace_ex(a["Xs"], Xe, m, 0, N, d, sp, meta, tab, a["x_mul"], a["x_add"], a["Zt"], a["alpha"],
                                    a["Linv"], opt(hi), opt(lo), a["hyp"], kern, 0.0, 1.0, 0, 0.0, 2.0, 1e-4, None, None, 7,
                                    opt(F), opt(mu), opt(var), a["ws"], ws_bytes, m_chunk, None)


@pytest.mark.parametrize("tensor", [True, False], ids=["tensor", "simt"])
def test_posterior_mace_rejects_bad_arguments(lib, tensor):
    bad = _lib.HB_ERR_INVALID
    path = dict(hi=tensor, lo=tensor)
    for name in POINTERS:
        assert _call(lib, **path, **{name: None}) == bad, name
        assert _call(lib, _spec(), **path, **{name: None}) == bad, name
    need = int(lib.hb_posterior_workspace_bytes(N, D, MC))
    assert need > 0
    for ws in (need - 1, 0, -1, -need, -(1 << 62)):                       # short or negative
        assert _call(lib, ws_bytes=ws, **path) == bad, ws
    for mc in (0, -1):
        assert _call(lib, m_chunk=mc, ws_bytes=1 << 40, **path) == bad, mc
    for m in (0, -1):
        assert _call(lib, m=m, **path) == bad, m
    for kern in (-1, 3, 7):
        assert _call(lib, kern=kern, **path) == bad, kern
    assert _call(lib, F=False, mu=False, var=False, **path) == bad           # nothing to write
    p = ctypes.c_void_p(16)
    mixed = _spec(num_enum=1)                                              # a categorical column needs Xe / meta / tables
    for Xe, meta, tab in ((None, p, p), (p, None, p), (p, p, None)):
        assert _call(lib, mixed, Xe=Xe, meta=meta, tab=tab, **path) == bad


def test_posterior_mace_needs_both_operand_halves_or_neither(lib):
    """Linv_hi and Linv_lo select the tensor path together; exactly one of them is a caller error, not a silent SIMT run."""
    bad = _lib.HB_ERR_INVALID
    assert _call(lib, hi=True, lo=False) == bad
    assert _call(lib, hi=False, lo=True) == bad


def test_posterior_mace_null_spec_form_rejects_bad_arguments(lib):
    """hb_posterior_mace is hb_posterior_mace_ex with spec = NULL: numeric models only (d = 0 is refused), same checks."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    need = int(lib.hb_posterior_workspace_bytes(N, D, MC))

    def call(m=M, d=D, kern=0, ws_bytes=need, hi=p, lo=p, mc=MC, F=p, mu=p, var=p):
        return lib.hb_posterior_mace(p, m, N, d, p, p, p, p, p, hi, lo, p, kern, 0.0, 1.0, 0, 0.0, 2.0, 1e-4, None, None, 7,
                                     F, mu, var, p, ws_bytes, mc, None)
    for d in (0, -1):
        assert call(d=d, ws_bytes=1 << 40) == bad, d
    assert call(m=0) == bad
    assert call(kern=3) == bad
    assert call(mc=0, ws_bytes=1 << 40) == bad
    assert call(ws_bytes=need - 1) == bad
    assert call(ws_bytes=-1) == bad
    assert call(hi=None) == bad and call(lo=None) == bad
    assert call(F=None, mu=None, var=None) == bad
