"""Host-side checks of the batched multi-output fit: workspace arithmetic and argument checks of hb_fit_multi_* (no CUDA
call is made), and which MultiTaskModel fits take the batched path."""
import ctypes as C

import pytest
import torch

from hebo_b200 import _lib
from hebo_b200.gp import MultiTaskModel


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_workspace_is_num_out_single_output_slices(lib):
    u, e = (C.c_int32 * 2)(5, 9), (C.c_int32 * 2)(3, 5)
    spec = _lib.ModelSpec(1, 2, u, e, 1)
    for n, d, sp in [(300, 6, None), (1100, 32, None), (257, 2, C.byref(spec))]:
        one = lib.hb_fit_workspace_bytes_ex(n, d, sp)
        assert one > 0 and one % 256 == 0
        for B in (1, 2, 7, _lib.HB_MAX_OUTPUTS):
            assert lib.hb_fit_multi_workspace_bytes(n, d, sp, B) == B * one
    assert lib.hb_fit_multi_workspace_bytes(0, 6, None, 2) < 0
    assert lib.hb_fit_multi_workspace_bytes(300, 0, None, 2) < 0


@pytest.mark.parametrize("B", [0, -1, _lib.HB_MAX_OUTPUTS + 1])
def test_num_out_outside_the_range_is_rejected(lib, B):
    assert lib.hb_fit_multi_workspace_bytes(300, 6, None, B) < 0
    dummy = C.c_void_p(256)                        # never dereferenced: the arguments are checked first
    losses = (C.c_float * 64)()
    status = (C.c_int32 * 64)()
    st = lib.hb_fit_multi_ex(dummy, None, dummy, 300, 6, None, B, dummy, 0, None, 1e-4, 0.01, 0.03, 1, None, losses, status,
                             dummy, 1 << 40, None)
    assert st == _lib.HB_ERR_INVALID


def test_null_status_and_short_workspace_are_rejected(lib):
    dummy = C.c_void_p(256)
    status = (C.c_int32 * 2)()
    assert lib.hb_fit_multi_ex(dummy, None, dummy, 300, 6, None, 2, dummy, 0, None, 1e-4, 0.01, 0.03, 1, None, None, None,
                               dummy, 1 << 40, None) == _lib.HB_ERR_INVALID
    short = lib.hb_fit_multi_workspace_bytes(300, 6, None, 2) - 1
    assert lib.hb_fit_multi_ex(dummy, None, dummy, 300, 6, None, 2, dummy, 0, None, 1e-4, 0.01, 0.03, 1, None, None, status,
                               dummy, short, None) == _lib.HB_ERR_INVALID


def _y(n, B):
    return torch.randn(n, B, generator=torch.Generator().manual_seed(0))


def test_batched_path_selection():
    y = _y(50, 3)
    assert MultiTaskModel(2, 0, 3)._batched(y)
    assert MultiTaskModel(2, 0, 3, optimizer="psgld")._batched(y)
    assert not MultiTaskModel(2, 0, 3, optimizer="lbfgs")._batched(y)
    assert not MultiTaskModel(2, 0, 3, optimizer="adam")._batched(y)
    assert not MultiTaskModel(2, 0, 1)._batched(y[:, :1])
    assert not MultiTaskModel(2, 0, _lib.HB_MAX_OUTPUTS + 1)._batched(_y(50, _lib.HB_MAX_OUTPUTS + 1))


def test_nan_patterns_select_the_path():
    y = _y(50, 3)
    y[[4, 9]] = float("nan")                       # the same rows in every output: one training set
    assert MultiTaskModel(2, 0, 3)._batched(y)
    y[11, 1] = float("inf")                        # output 1 loses one more row than the others
    assert not MultiTaskModel(2, 0, 3)._batched(y)
