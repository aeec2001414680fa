"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol include/hebo_b200.h
declares; host-only entry points answer without a GPU.  (No compute calls here.)"""
import ctypes
import os
import re

import pytest

from hebo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "hebo_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(hb_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_header_and_binding_table_agree():
    names = declared_functions()
    assert len(names) >= 18
    assert sorted(_lib.SIGNATURES.keys()) == names


def test_library_exports_every_declared_symbol(lib):
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared_functions():
        assert hasattr(raw, name), f"{name} declared in include/hebo_b200.h but not exported"


def test_host_only_entry_points(lib):
    assert lib.hb_version() >= 200
    # parameter counts / workspace of the general (mixed, non-ARD) models, host only
    assert lib.hb_num_params(32, None) == 35
    u, e = (ctypes.c_int32 * 2)(5, 9), (ctypes.c_int32 * 2)(3, 5)
    spec = _lib.ModelSpec(1, 2, u, e)
    assert lib.hb_num_params(2, ctypes.byref(spec)) == 66 and lib.hb_num_params(0, ctypes.byref(spec)) == 64
    spec0 = _lib.ModelSpec(0, 0, None, None)
    assert lib.hb_num_params(7, ctypes.byref(spec0)) == 4
    assert lib.hb_num_params(0, None) < 0
    assert lib.hb_fit_workspace_bytes_ex(1000, 2, ctypes.byref(spec)) > lib.hb_fit_workspace_bytes(1000, 2)
    assert lib.hb_vnorm_operand_kind() == 0
    assert lib.hb_padded_n(1) == 128 and lib.hb_padded_n(128) == 128 and lib.hb_padded_n(129) == 256
    assert lib.hb_padded_n(4096) == 4096
    w = lib.hb_fit_workspace_bytes(4096, 32)
    assert w >= 3 * 4096 * 4096 * 4          # L, Linv, scratch
    assert lib.hb_fit_workspace_bytes(0, 3) < 0
    assert lib.hb_posterior_workspace_bytes(4096, 32, 8192) >= 8192 * 4096 * 4
    assert lib.hb_pareto_workspace_bytes(1 << 20) >= (1 << 20) * 5
    assert isinstance(lib.hb_last_error(), bytes)


def test_invalid_arguments_are_reported_not_crashed(lib):
    # NULL pointers / bad sizes must come back as HB_ERR_INVALID before any CUDA call
    assert lib.hb_gram(None, 10, 2, None, 0, None, 0.0, None, None) == _lib.HB_ERR_INVALID
    assert lib.hb_cholesky(None, 128, None, None, None) == _lib.HB_ERR_INVALID
    assert lib.hb_pareto_front3(None, 10, None, None, None, 0, None) == _lib.HB_ERR_INVALID
    assert lib.hb_fit_state(None, 10, 2, None) == _lib.HB_ERR_INVALID
    assert lib.hb_fit_ex(None, None, None, 10, 2, None, None, 0, None, 0.0, 0.01, 0.01, 1, None, None, None, 0, None) == _lib.HB_ERR_INVALID
    assert lib.hb_mll_fwd_bwd(None, None, None, 10, 2, None, None, 0, None, 0.0, 0.01, 0.0, None, None, None, None, 0, None) == _lib.HB_ERR_INVALID


def test_linalg_stages_reject_bad_sizes_and_null_pointers(lib):
    """hb_tri_inverse, hb_kinv and hb_solve_logdet refuse NP <= 0 or not a multiple of 128, n <= 0 or n > NP, and every
    NULL pointer with HB_ERR_INVALID before any launch.  The pointers are fake and never dereferenced."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    for np_ in (0, -128, 100, 129, 200):
        assert lib.hb_tri_inverse(p, np_, p, p, None) == bad, np_
        assert lib.hb_kinv(p, np_, p, None) == bad, np_
        assert lib.hb_solve_logdet(p, p, p, 10, np_, p, p, p, p, None) == bad, np_
    for n, np_ in ((0, 128), (-1, 128), (-(1 << 40), 256), (129, 128), (257, 256)):
        assert lib.hb_solve_logdet(p, p, p, n, np_, p, p, p, p, None) == bad, (n, np_)
    for k in range(3):
        args = [p, p, p]
        args[k] = None
        assert lib.hb_tri_inverse(args[0], 128, args[1], args[2], None) == bad, k
    for k in range(2):
        args = [p, p]
        args[k] = None
        assert lib.hb_kinv(args[0], 128, args[1], None) == bad, k
    for k in range(7):
        args = [p] * 7                      # L, Linv, y, hyp, alpha, scal, ws
        args[k] = None
        L, Linv, y, hyp, alpha, scal, ws = args
        assert lib.hb_solve_logdet(L, Linv, y, 10, 128, hyp, alpha, scal, ws, None) == bad, k


def test_tensor_core_stages_reject_bad_sizes_null_pointers_and_short_workspaces(lib):
    """hb_cholesky_tc, hb_tri_inverse_tc and hb_kinv_tc refuse NP <= 0 or not a multiple of 128, every NULL pointer, and a
    tensor-core workspace one byte short or of negative size, with HB_ERR_INVALID before any launch.  The workspace size is
    the fit workspace's tensor-core block: 8 NP^2 + 2 * 512 NP floats (every block a multiple of 256 bytes here).  The
    pointers are fake and never dereferenced."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    for np_ in (128, 640, 4224):
        assert lib.hb_tc_workspace_bytes(np_) == 4 * (8 * np_ * np_ + 2 * 512 * np_), np_
    big = lib.hb_tc_workspace_bytes(4224)
    for np_ in (0, -128, 100, 129, 200):
        assert lib.hb_tc_workspace_bytes(np_) < 0, np_
        assert lib.hb_cholesky_tc(p, np_, p, p, p, big, None) == bad, np_
        assert lib.hb_tri_inverse_tc(p, np_, p, p, big, None) == bad, np_
        assert lib.hb_kinv_tc(np_, p, p, big, None) == bad, np_
    for k in range(4):
        args = [p] * 4                      # A, ws, info, tc_ws
        args[k] = None
        assert lib.hb_cholesky_tc(args[0], 128, args[1], args[2], args[3], big, None) == bad, k
    for k in range(3):
        args = [p] * 3                      # L, Linv, tc_ws
        args[k] = None
        assert lib.hb_tri_inverse_tc(args[0], 128, args[1], args[2], big, None) == bad, k
    for k in range(2):
        args = [p] * 2                      # Kinv, tc_ws
        args[k] = None
        assert lib.hb_kinv_tc(128, args[0], args[1], big, None) == bad, k
    need = lib.hb_tc_workspace_bytes(640)
    for short in (need - 1, -1, -(1 << 40)):
        assert lib.hb_cholesky_tc(p, 640, p, p, p, short, None) == bad, short
        assert lib.hb_tri_inverse_tc(p, 640, p, p, short, None) == bad, short
        assert lib.hb_kinv_tc(640, p, p, short, None) == bad, short


def test_front_pack_rejects_row_offsets_outside_the_id_range(lib):
    """hb_front_pack stores a global id row_offset + row (row < 2^31) as two 24-bit fp32 halves, exact below 2^48: a
    negative row_offset, or one above 2^48 - 2^31, is refused before any launch.  The pointers are fake and never
    dereferenced."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    top = (1 << 48) - (1 << 31)
    for off in (-1, -(1 << 31), top + 1, 1 << 48, (1 << 62)):
        assert lib.hb_front_pack(p, p, p, p, p, off, 64, p, None) == bad, off


@pytest.mark.parametrize("ws_bytes", ["short", -1, -(1 << 40)])
def test_workspace_size_is_checked_as_a_signed_count(lib, ws_bytes):
    """A workspace one byte short, or of negative size, is refused before any launch.  A negative int64 must not pass the
    check as a huge size_t.  The pointers are fake and never dereferenced."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)

    def ws(need):
        assert need > 0
        return need - 1 if ws_bytes == "short" else ws_bytes
    m = 5000
    need = int(lib.hb_pareto_workspace_bytes(m))
    assert lib.hb_pareto_front3(p, m, p, p, p, ws(need), None) == bad
    for k in (1, 3, 8):
        assert lib.hb_pareto_front_k(p, m, k, p, p, p, ws(need), None) == bad, k
    need = int(lib.hb_front_merge_workspace_bytes(4, 64))
    assert lib.hb_front_merge(p, 4, 64, p, p, ws(need), None) == bad
    n, d = 300, 2
    need = int(lib.hb_sample_workspace_bytes(n, d, None, 100))
    assert lib.hb_sample_y(p, None, 100, n, d, None, None, None, p, p, p, p, p, p, p, 0, 0.0, 1.0, 0, p, 3, p, None, p,
                           ws(need), None) == bad


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.HeboB200Error):
        _lib.lib()
