"""Host-side checks of the feature-selecting deep ensemble (hebo_b200.FeDeepEnsemble): conf defaults, FeNet's gate-last
parameter layout, the weights-only L1 set, the concrete layers' temperature schedule against the reference's recorded
temperatures, the argument checks of hb_fe_fit / hb_fe_predict (no CUDA call is made), and that the optimisers outside
HEBO and BO still reject the name."""
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import FeDeepEnsemble, _lib
from hebo_b200.bo import BO, HEBO_VectorContextual
from hebo_b200.embedding import HEBO_Embedding
from hebo_b200.ensemble import fe_epoch_temperature, init_params
from hebo_b200.general import GeneralBO
from hebo_b200.gp import MultiTaskModel
from hebo_b200.noisy import NoisyOpt
from hebo_b200.suggest import HEBO
from tests.util import load_golden

SPACE = [{"name": "x0", "type": "num", "lb": -3, "ub": 7}, {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}]


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_defaults_match_the_reference():
    m = FeDeepEnsemble(3, 0, 1)
    assert (m.fe_layer, m.temperature, m.mask_reg, m.start_temp, m.end_temp, m.anneal_base) == ("stg", None, 0.1, 1.0, 0.1, 0.99)
    assert m.support_grad is False and m.support_warm_start and m.num_ensembles == 5 and m.num_epochs == 500
    assert m.gate_temperature == 1.0
    assert FeDeepEnsemble(3, 0, 1, fe_layer="concrete").gate_temperature == float(np.float32(0.1))
    assert FeDeepEnsemble(3, 0, 1, fe_layer="hard_concrete", temperature=0.3).gate_temperature == float(np.float32(0.3))
    assert FeDeepEnsemble(3, 0, 1, temperature=0).gate_temperature == 1.0        # FeNet: `if self.temperature:`


def test_unknown_fe_layer_is_rejected():
    with pytest.raises(KeyError):
        FeDeepEnsemble(3, 0, 1, fe_layer="gumbel")


def test_gate_is_the_last_parameter_of_fenet_layout():
    m = FeDeepEnsemble(2, 2, 2, num_uniqs=[4, 7], num_hiddens=8, rand_prior=True, fe_layer="concrete")
    names = [n for n, _ in m.layout]
    # FeNet's state_dict: BaseNet's registration order, then feature_select (fe_deep_ensemble.py:20-27)
    assert names == ["enum_layer.emb.0.weight", "enum_layer.emb.1.weight", "hidden.0.weight", "hidden.0.bias",
                     "mu.weight", "mu.bias", "sigma2.0.weight", "sigma2.0.bias", "prior_net.0.weight", "prior_net.0.bias",
                     "prior_net.prior_net_out.weight", "prior_net.prior_net_out.bias", "feature_select.logits"]
    assert m.layout[-1][1] == (m.din,) and m.din == 2 + 3 + 4
    assert m.P == sum(int(np.prod(s)) for _, s in m.layout)
    assert FeDeepEnsemble(3, 0, 1).layout[-1][0] == "feature_select.mu"
    torch.manual_seed(0)
    raw = init_params(m.layout)
    assert raw.numel() == m.P and float(raw[-m.din:].abs().max()) < 0.05 and bool((raw[-m.din:] != 0).all())


def test_layout_matches_the_reference_fixture(lib):
    ref = load_golden("ref_fe_deep_ensemble.npz")
    inputs = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]
    for vi in range(int(ref["num_variants"])):
        li, noise, inp, O, prior = (int(v) for v in ref[f"v{vi}_cfg"])
        dc, uniqs, trans = inputs[inp]
        m = FeDeepEnsemble(dc, len(uniqs), O, num_ensembles=2, num_epochs=3, batch_size=8, num_hiddens=8,
                           output_noise=bool(noise), rand_prior=bool(prior), enum_trans=trans, num_uniqs=uniqs,
                           fe_layer=["stg", "concrete", "hard_concrete"][li])
        assert ref[f"v{vi}_init"].shape[1] == m.P
        assert lib.hb_fe_num_params(C.byref(m._spec)) == m.P
        assert lib.hb_fe_fit_workspace_bytes(C.byref(m._spec), 5) == 3 * 5 * m.P * 4
        assert ref[f"v{vi}_draws"].shape == m.draws_shape(ref[f"v{vi}_ys_fit"].shape[0])


def test_l1_covers_weights_only():
    """FeDeepEnsemble.fit_one takes the L1 term over parameters whose name contains 'weight': embedding tables and every
    weight matrix, the prior net's included; not the biases and not the gate."""
    m = FeDeepEnsemble(2, 1, 1, num_uniqs=[5], num_hiddens=8, num_layers=2, rand_prior=True)
    l1 = [n for n, _ in m.layout if "weight" in n]
    assert l1 == ["enum_layer.emb.0.weight", "hidden.0.weight", "hidden.2.weight", "mu.weight", "sigma2.0.weight",
                  "prior_net.0.weight", "prior_net.2.weight", "prior_net.prior_net_out.weight"]
    assert not any(n.startswith("feature_select") for n in l1)


def test_temperature_schedule_matches_the_reference():
    ref = load_golden("ref_fe_deep_ensemble.npz")
    seen = 0
    for vi in range(int(ref["num_variants"])):
        li = int(ref[f"v{vi}_cfg"][0])
        temps = ref[f"v{vi}_temps"]
        for ep in range(temps.shape[1]):
            want = 1.0 if li == 0 else fe_epoch_temperature(1.0, 0.1, 0.99, ep)
            assert (temps[:, ep] == np.float32(want)).all()
            seen += 1
        if li:
            assert float(ref[f"v{vi}_eval_temp"][0]) == fe_epoch_temperature(1.0, 0.1, 0.99, temps.shape[1] - 1)
    assert seen > 0
    # the clamp at end_temp, and the product taken in double before the fp32 rounding
    assert fe_epoch_temperature(1.0, 0.1, 0.99, 499) == float(np.float32(0.1))
    assert fe_epoch_temperature(1.0, 0.1, 0.99, 100) == float(np.float32(0.99 ** 100))


def test_batch_envelope_counts_the_gate_buffers():
    de_rows = FeDeepEnsemble(2, 0, 1, num_hiddens=256, num_layers=3)
    rows = 32
    assert de_rows.batch_floats(rows) == super(FeDeepEnsemble, de_rows).batch_floats(rows) + 2 * rows * (de_rows.din | 1)
    m = FeDeepEnsemble(256, 0, 8, num_layers=3, num_hiddens=256, rand_prior=True, batch_size=32)
    assert m.batch_floats(32) > _lib.HB_DE_MAX_BATCH_FLOATS
    with pytest.raises(NotImplementedError, match="HB_DE_MAX_BATCH_FLOATS"):
        m.fit(torch.randn(100, 256), None, torch.randn(100, 8))


def test_c_argument_checks(lib):
    u = (C.c_int32 * 1)(3)
    spec = _lib.DeSpec(4, 1, u, 0, 1, 16, 1, 1, 0, 1e-4)
    P = lib.hb_fe_num_params(C.byref(spec))
    assert P == lib.hb_de_num_params(C.byref(spec)) + 4 + 2
    assert C.sizeof(_lib.FeGate) == 40
    ws = C.c_void_p(16)
    for kind, T in ((3, 1.0), (-1, 1.0), (0, 0.0), (1, float("nan"))):
        g = _lib.FeGate(kind, T, 1.0, 0.1, 0.99, 0.1)
        rc = lib.hb_fe_fit(ws, ws, ws, 10, C.byref(spec), C.byref(g), 2, ws, 5e-3, 1e-3, 32, 1, None, None, 0, ws, ws,
                           1 << 30, None)
        assert rc != 0
        rc = lib.hb_fe_predict(ws, ws, 10, C.byref(spec), C.byref(g), 2, ws, ws, ws, ws, ws, -1, None, 0, 0, ws, ws, None)
        assert rc != 0
    g = _lib.FeGate(0, 1.0, 1.0, 0.1, 0.99, 0.1)
    assert lib.hb_fe_fit(ws, ws, ws, 10, C.byref(spec), None, 2, ws, 5e-3, 1e-3, 32, 1, None, None, 0, ws, ws, 1 << 30,
                         None) != 0
    need = lib.hb_fe_fit_workspace_bytes(C.byref(spec), 2)
    assert lib.hb_fe_fit(ws, ws, ws, 10, C.byref(spec), C.byref(g), 2, ws, 5e-3, 1e-3, 32, 1, None, None, 0, ws, ws,
                         need - 1, None) != 0
    assert lib.hb_fe_predict(ws, ws, 10, C.byref(spec), C.byref(g), 2, ws, ws, ws, ws, ws, 2, None, 0, 0, ws, ws, None) != 0
    assert lib.hb_fe_fit(ws, ws, ws, 10, C.byref(spec), C.byref(g), 2, ws, 5e-3, 1e-3, 32, 0, None, None, 0, None, ws,
                         need, None) == 0           # num_epochs = 0 changes nothing and launches nothing


def test_only_hebo_and_bo_take_the_name():
    assert HEBO(SPACE, model_name="fe_deep_ensemble").model_name == "fe_deep_ensemble"
    assert HEBO(SPACE, model_name="fe_deep_ensemble").model_config == {"num_uniqs": [3]}
    assert BO(SPACE, model_name="fe_deep_ensemble").model_name == "fe_deep_ensemble"
    with pytest.raises(NotImplementedError):
        GeneralBO(SPACE, 2, 1, model_name="fe_deep_ensemble")
    with pytest.raises(NotImplementedError):
        NoisyOpt(SPACE, model_name="fe_deep_ensemble")
    box = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(4)]
    with pytest.raises(NotImplementedError):
        HEBO_Embedding(box, model_name="fe_deep_ensemble", eff_dim=2, device="cpu")
    with pytest.raises(NotImplementedError):
        HEBO_VectorContextual(SPACE, {"one": {"x1": "a"}}, model_name="fe_deep_ensemble")
    with pytest.raises(NotImplementedError):
        MultiTaskModel(2, 0, 2, base_model_name="fe_deep_ensemble", device="cpu")
