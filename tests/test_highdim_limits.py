"""The feature-count bound d + sum(emb_sizes) <= HB_MAX_FEATURES (4096), host only: the Python model and the C ABI's
parameter / workspace queries agree on it."""
import ctypes
import os
import re

import pytest

import hebo_b200
from hebo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_header_and_binding_state_the_same_bound():
    with open(os.path.join(ROOT, "include", "hebo_b200.h")) as fh:
        m = re.search(r"#define\s+HB_MAX_FEATURES\s+(\d+)", fh.read())
    assert m and int(m.group(1)) == _lib.HB_MAX_FEATURES == 4096


def test_gp_accepts_the_bound_and_rejects_one_more():
    gp = hebo_b200.GP(4096, 0, 1)
    assert gp.num_cont + gp.De == 4096
    with pytest.raises(NotImplementedError, match="4096"):
        hebo_b200.GP(4097, 0, 1)
    # numeric columns plus the embedding widths (min(50, 1 + u // 2) per categorical column) count together
    hebo_b200.GP(4096 - 100, 2, 1, num_uniqs=[200, 200])
    with pytest.raises(NotImplementedError, match="4096"):
        hebo_b200.GP(4096 - 99, 2, 1, num_uniqs=[200, 200])
    with pytest.raises(NotImplementedError, match="4096"):
        hebo_b200.GP(4000, 1, 1, num_uniqs=[300], emb_sizes=[97])


def test_abi_queries_accept_the_bound_and_reject_one_more(lib):
    assert lib.hb_num_params(4096, None) == 4096 + 3
    assert lib.hb_num_params(4097, None) < 0
    n = 512
    w = lib.hb_fit_workspace_bytes_ex(n, 4096, None)
    assert w > 0 and lib.hb_fit_workspace_bytes_ex(n, 4097, None) < 0
    # Zt [d, NP] and the per-block gradient partials, sized for the widest row (3 d + 3 slots: a learned warp)
    nblocks = (n // 128) * (n // 128 + 1) // 2
    assert w >= 4096 * n * 4 + nblocks * (3 * 4096 + 3) * 4
    # learned warp: the derivative rows dZa, dZb [d, NP] on top
    warp = _lib.ModelSpec(1, 0, None, None, 1)
    ww = lib.hb_fit_workspace_bytes_ex(n, 4096, ctypes.byref(warp))
    assert ww >= w + 2 * 4096 * n * 4
    assert lib.hb_fit_workspace_bytes_ex(n, 4097, ctypes.byref(warp)) < 0
    # mixed: d + De counts, and the embedding-row gradient buffer [NP / 128][De][NP] is part of the workspace
    u, e = (ctypes.c_int32 * 2)(100, 100), (ctypes.c_int32 * 2)(48, 48)
    mixed = _lib.ModelSpec(1, 2, u, e)
    wm = lib.hb_fit_workspace_bytes_ex(n, 4000, ctypes.byref(mixed))
    assert wm >= (n // 128) * 96 * n * 4 + 4096 * n * 4
    assert lib.hb_num_params(4000, ctypes.byref(mixed)) > 0
    assert lib.hb_num_params(4001, ctypes.byref(mixed)) < 0
    assert lib.hb_fit_workspace_bytes_ex(n, 4001, ctypes.byref(mixed)) < 0
    assert lib.hb_sample_workspace_bytes(n, 4001, ctypes.byref(mixed), 64) < 0
