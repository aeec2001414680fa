"""Host-side contract of hebo_b200.RF (no GPU): the reference's constructor key and default, flags and noise, the
single-output and envelope checks, category range checks, and register() into a HEBO model registry."""
import sys
import types

import pytest
import torch

from hebo_b200 import RF, _lib
from hebo_b200.gp import GP, register


def test_defaults_and_flags():
    m = RF(2, 0, 1)
    assert m.n_estimators == 100
    assert RF(2, 0, 1, n_estimators=20).n_estimators == 20
    assert not (m.support_ts or m.support_grad or m.support_multi_output or m.support_warm_start)
    assert torch.equal(m.noise, torch.zeros(1)) and not m.fitted
    with pytest.raises(NotImplementedError):
        m.sample_f()
    mixed = RF(1, 2, 1, num_uniqs=[3, 4])
    assert mixed.width == 8 and mixed.num_uniqs == [3, 4]


def test_num_out_and_envelope():
    with pytest.raises(NotImplementedError):
        RF(2, 0, 2)
    with pytest.raises(NotImplementedError):
        RF(2, 0, 1, n_estimators=_lib.HB_RF_MAX_TREES + 1)
    with pytest.raises(NotImplementedError):
        RF(2, 0, 1, n_estimators=0)
    RF(_lib.HB_RF_MAX_WIDTH, 0, 1)
    with pytest.raises(NotImplementedError):
        RF(_lib.HB_RF_MAX_WIDTH - 2, 1, 1, num_uniqs=[3])
    with pytest.raises(NotImplementedError):
        RF(1, 0, 1, device="cpu").fit(torch.zeros(_lib.HB_RF_MAX_ROWS + 1, 1), None, torch.zeros(_lib.HB_RF_MAX_ROWS + 1, 1))


def test_input_checks_before_any_launch():
    m = RF(1, 1, 1, num_uniqs=[3], device="cpu")
    with pytest.raises(IndexError):
        m.fit(torch.zeros(4, 1), torch.tensor([[0], [1], [3], [2]]), torch.zeros(4, 1))
    with pytest.raises(IndexError):
        m.fit(torch.zeros(4, 1), torch.tensor([[0], [-1], [2], [2]]), torch.zeros(4, 1))
    with pytest.raises(AssertionError):                       # filter_nan: no finite target
        m.fit(torch.zeros(2, 1), torch.zeros(2, 1).long(), torch.full((2, 1), float("nan")))
    with pytest.raises(AssertionError):                       # filter_nan: non-finite inputs
        m.fit(torch.tensor([[0.0], [float("inf")]]), torch.zeros(2, 1).long(), torch.zeros(2, 1))
    with pytest.raises(IndexError):
        m.predict(torch.zeros(2, 1), torch.tensor([[0], [5]]))
    for v in (float("inf"), float("-inf")):                  # sklearn refuses infinite candidates
        with pytest.raises(ValueError):
            m.predict(torch.tensor([[0.0], [v]]), torch.zeros(2, 1).long())
        with pytest.raises(ValueError):
            m.sample_y(torch.tensor([[v]]), torch.zeros(1, 1).long())


def test_abi_rejects_outside_the_envelope():
    if not _lib.available():
        pytest.skip("library not built")
    import ctypes as C
    lib = _lib.lib()
    u = (C.c_int32 * 2)(3, 4)
    spec = _lib.RfSpec(2, 2, u)
    assert lib.hb_rf_fit_workspace_bytes(100, C.byref(spec), 1, 20) > 0
    assert lib.hb_rf_forest_bytes(C.byref(spec), 199, 1, 20) > 0
    assert lib.hb_rf_fit_workspace_bytes(_lib.HB_RF_MAX_ROWS + 1, C.byref(spec), 1, 20) < 0
    assert lib.hb_rf_fit_workspace_bytes(100, C.byref(spec), _lib.HB_MAX_OUTPUTS + 1, 20) < 0
    assert lib.hb_rf_fit_workspace_bytes(100, C.byref(spec), 1, _lib.HB_RF_MAX_TREES + 1) < 0
    wide = _lib.RfSpec(_lib.HB_RF_MAX_WIDTH, 1, u)
    assert lib.hb_rf_forest_bytes(C.byref(wide), 10, 1, 1) < 0
    assert lib.hb_rf_fit(None, None, None, 10, C.byref(spec), 1, 1, None, 0, None, None, None, 0, None) == _lib.HB_ERR_INVALID
    assert lib.hb_rf_predict(None, None, 10, C.byref(spec), None, 1, 1, None, None, None, 0, 0, 0, None, None) == \
        _lib.HB_ERR_INVALID
    assert lib.hb_rf_load(None, None, None, None, None, None, C.byref(spec), 1, 10, None, None) == _lib.HB_ERR_INVALID


@pytest.fixture
def registry(monkeypatch):
    sentinel_rf, sentinel_gp = object(), object()
    factory = types.ModuleType("hebo.models.model_factory")
    factory.model_dict = {"gp": sentinel_gp, "rf": sentinel_rf}
    factory.model_names = list(factory.model_dict)
    hebo = types.ModuleType("hebo")
    models = types.ModuleType("hebo.models")
    hebo.models, models.model_factory = models, factory
    monkeypatch.setitem(sys.modules, "hebo", hebo)
    monkeypatch.setitem(sys.modules, "hebo.models", models)
    monkeypatch.setitem(sys.modules, "hebo.models.model_factory", factory)
    return factory, sentinel_gp, sentinel_rf


def test_register_adds_rf_b200_and_keeps_rf(registry):
    factory, gp, rf = registry
    assert register()
    assert factory.model_dict["rf_b200"] is RF and factory.model_dict["rf"] is rf and factory.model_dict["gp"] is gp
    assert "rf_b200" in factory.model_names


def test_register_override_rf(registry):
    factory, gp, rf = registry
    assert register(override_rf=True)
    assert factory.model_dict["rf"] is RF and factory.model_dict["gp"] is gp
    assert register(override_gp=True, override_rf=True) and factory.model_dict["gp"] is GP
