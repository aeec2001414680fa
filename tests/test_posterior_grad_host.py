"""Argument checks of hb_posterior_grad_ex / hb_posterior_grad, CPU only.

Every call passes fake device pointers that must never be dereferenced: each one has to fail its argument checks before
any launch.  A warped spec is rejected because post_grad_kernel differentiates through x_mul / l only -- the caller
applies the Kumaraswamy warp in front (hebo_b200.GP._predict_autograd) and passes spec->warp = 0."""
import ctypes

import pytest

from hebo_b200 import _lib

N, D, M = 300, 2, 100
POINTERS = ("Xs", "x_mul", "x_add", "Zt", "alpha", "Linv", "hyp", "mu", "var", "dmu", "dvar", "ws")


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def _call(lib, spec=None, m=M, d=D, kern=0, m_chunk=128, ws_bytes=None, Xe=None, meta=None, tab=None, **null):
    p = ctypes.c_void_p(16)
    a = {k: p for k in POINTERS}
    a.update(null)
    if ws_bytes is None:
        ws_bytes = int(lib.hb_posterior_workspace_bytes(N, max(d, 1), max(m_chunk, 1)))
    sp = None if spec is None else ctypes.byref(spec)
    return lib.hb_posterior_grad_ex(a["Xs"], Xe, m, N, d, sp, meta, tab, a["x_mul"], a["x_add"], a["Zt"], a["alpha"], a["Linv"],
                                    a["hyp"], kern, 0.0, 1.0, 0, a["mu"], a["var"], a["dmu"], a["dvar"], a["ws"], ws_bytes,
                                    m_chunk, None)


def _spec(warp=0, num_enum=0):
    u, e = (ctypes.c_int32 * 1)(3), (ctypes.c_int32 * 1)(2)
    spec = _lib.ModelSpec(1, num_enum, u, e, warp)
    spec._keep = (u, e)
    return spec


@pytest.mark.parametrize("warp", [1, 2])
def test_posterior_grad_rejects_a_warped_spec(lib, warp):
    """Learned (1) and fixed (2) warps: the kernel would compare unwarped candidate features with the warped training
    features and drop dw/dx, so the call refuses the spec; a warped model's caller passes warp = 0."""
    assert _call(lib, _spec(warp)) == _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    assert _call(lib, _spec(warp, num_enum=1), Xe=p, meta=p, tab=p) == _lib.HB_ERR_INVALID


def test_posterior_grad_rejects_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    for name in POINTERS:
        assert _call(lib, **{name: None}) == bad, name
        assert _call(lib, _spec(0), **{name: None}) == bad, name
    for m in (0, -1):
        assert _call(lib, m=m) == bad, m
    for mc in (0, -1):
        assert _call(lib, m_chunk=mc, ws_bytes=1 << 40) == bad, mc
    for d in (0, -1):
        assert _call(lib, d=d, ws_bytes=1 << 40) == bad, d
    for kern in (-1, 3, 7):
        assert _call(lib, kern=kern) == bad, kern
    need = int(lib.hb_posterior_workspace_bytes(N, D, 128))
    assert need > 0
    assert _call(lib, ws_bytes=need - 1) == bad                            # one byte short
    assert _call(lib, ws_bytes=-1) == bad                                  # negative: not a huge unsigned size
    p = ctypes.c_void_p(16)
    mixed = _spec(0, num_enum=1)                                           # a categorical column needs Xe / meta / tables
    for Xe, meta, tab in ((None, p, p), (p, None, p), (p, p, None)):
        assert _call(lib, mixed, Xe=Xe, meta=meta, tab=tab) == bad


def test_posterior_grad_null_spec_form_rejects_bad_arguments(lib):
    """hb_posterior_grad is hb_posterior_grad_ex with spec = NULL: it inherits the same checks."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    need = int(lib.hb_posterior_workspace_bytes(N, D, 128))

    def call(m=M, d=D, kern=0, ws_bytes=need, dvar=p):
        return lib.hb_posterior_grad(p, m, N, d, p, p, p, p, p, p, kern, 0.0, 1.0, 0, p, p, p, dvar, p, ws_bytes, 128, None)
    assert call(m=0) == bad
    assert call(d=0, ws_bytes=1 << 40) == bad
    assert call(kern=3) == bad
    assert call(ws_bytes=need - 1) == bad
    assert call(ws_bytes=-1) == bad
    assert call(dvar=None) == bad
