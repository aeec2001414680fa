"""GumbelDeepEnsemble's host side without a GPU: defaults, parameter layout and initialisation, the temperature schedule,
the rand_prior rule, the C argument checks, and the optimiser gates."""
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import GumbelDeepEnsemble, _lib
from hebo_b200.acq import _batchable
from hebo_b200.ensemble import EnsembleBatch, gumbel_epoch_temperature


def _m(dc=5, ne=0, **kw):
    if ne:
        kw.setdefault("num_uniqs", [3] * ne)
    return GumbelDeepEnsemble(dc, ne, 1, device="cpu", **kw)


def test_defaults_and_reduced_dim():
    m = _m(5)
    assert m.reduced_dim == 3 and m.conf["reduced_dim"] == 3 and m.support_grad is False
    assert _m(0, 2).reduced_dim == 1 and _m(5, reduced_dim=1).reduced_dim == 1
    assert m.num_epochs == 500 and m.batch_size == 32 and m.l1 == 1e-3 and m.temperature == 0.1


def test_layout_and_init():
    m = _m(6, 2, num_layers=2, num_hiddens=16)
    names = [n for n, _ in m.layout]
    assert names[-1] == "feature_select.logits" and dict(m.layout)["feature_select.logits"] == (4, 6)
    assert dict(m.layout)["hidden.0.weight"] == (16, 4 + 4)         # selected width + two embeddings of 2
    assert m.P == sum(int(np.prod(s)) for _, s in m.layout)
    torch.manual_seed(0)
    raw = m.init_member()
    sd = {}
    o = 0
    for n, s in m.layout:
        k = int(np.prod(s))
        sd[n] = raw[o:o + k].reshape(s)
        o += k
    assert (sd["feature_select.logits"] == 0).all() and (sd["mu.bias"] == 0).all()
    # rebuilt hidden layers: nn.Linear's default, biases in U(+-1/sqrt(fan_in)) and nonzero
    assert (sd["hidden.0.bias"] != 0).any() and sd["hidden.0.bias"].abs().max() <= 1 / np.sqrt(8)
    assert sd["hidden.0.weight"].abs().max() <= 1 / np.sqrt(8)
    # without numeric columns nothing is rebuilt: BaseNet's zero biases
    m0 = _m(0, 2)
    assert dict(m0.layout)["feature_select.logits"] == (1, 0)
    raw0 = m0.init_member()
    b0 = dict(m0.layout)
    off = sum(int(np.prod(s)) for n, s in m0.layout[:[n for n, _ in m0.layout].index("hidden.0.bias")])
    assert (raw0[off:off + b0["hidden.0.bias"][0]] == 0).all()


def test_temperature_schedule():
    assert gumbel_epoch_temperature(0) == float(np.float32(1.1))
    assert gumbel_epoch_temperature(10) == float(np.float32(0.8 ** 10 + 0.1))


def test_rand_prior_rule():
    with pytest.raises(NotImplementedError):
        _m(5, rand_prior=True)
    assert _m(5, rand_prior=True, reduced_dim=5).rand_prior
    assert _m(0, 2, rand_prior=True).rand_prior


def test_c_argument_checks():
    lib = _lib.lib()
    m = _m(5)
    assert lib.hb_gumbel_num_params(C.byref(m._spec), 3) == m.P
    assert lib.hb_gumbel_num_params(C.byref(m._spec), 0) == -1
    assert lib.hb_gumbel_num_params(C.byref(m._spec), 300) == -1
    mp = _m(5, rand_prior=True, reduced_dim=5)
    assert lib.hb_gumbel_num_params(C.byref(mp._spec), 4) == -1
    assert lib.hb_gumbel_fit_workspace_bytes(C.byref(m._spec), 3, 2) == 4 * (3 * 2 * m.P + 2 * 3 * 5)
    assert lib.hb_gumbel_fit_workspace_bytes(C.byref(m._spec), 3, 0) == -1
    rc = lib.hb_gumbel_fit(None, None, None, 10, C.byref(m._spec), 3, 1, None, 5e-3, 1e-3, 8, 1, None, None, 0, None, None,
                           0, None)
    assert rc == _lib.HB_ERR_INVALID
    rc = lib.hb_gumbel_predict(None, None, 10, C.byref(m._spec), 3, 0.0, 1, None, None, None, None, None, -1, None, 0, 0,
                               None, None, None, 0, None)
    assert rc == _lib.HB_ERR_INVALID


def test_l1_set_is_the_weights():
    """GumbelDeepEnsemble.fit_one's L1 term covers names containing 'weight' (embedding tables, hidden, heads, prior
    weights), not biases or the logits: the fp32 restatement's mask equals that set over the host layout."""
    from oracle import gumbel_oracle as GO
    m = _m(0, 2, rand_prior=True, num_layers=2, num_hiddens=8, output_noise=False)
    net = GO.GumbelNet32([3, 3], "embedding", 2, 8, 1, rand_prior=True)
    assert net.P == m.P
    want = np.concatenate([np.full(int(np.prod(s)), "weight" in n) for n, s in m.layout])
    assert np.array_equal(net.is_weight, want)
    names = [n for n, _ in m.layout]
    assert "prior_net.0.bias" in names and "enum_layer.emb.0.weight" in names
    assert not any("weight" in n for n in names if n.endswith("bias") or n == "feature_select.logits")


def test_optimiser_gates_and_batchable():
    from hebo_b200 import HEBO_Embedding, HEBO_VectorContextual, MultiTaskModel
    from hebo_b200.suggest import HEBO
    from hebo_b200.space import DesignSpace
    from hebo_b200.noisy import NoisyOpt
    from hebo_b200.general import GeneralBO
    sp = DesignSpace().parse([{"name": "x", "type": "num", "lb": 0, "ub": 1}])
    HEBO(sp, model_name="gumbel", device="cpu")
    rejected = [lambda: NoisyOpt(sp, model_name="gumbel"), lambda: GeneralBO(sp, 1, 0, model_name="gumbel"),
                lambda: MultiTaskModel(1, 0, 2, base_model_name="gumbel"),
                lambda: HEBO_Embedding(sp, model_name="gumbel"),
                lambda: HEBO_VectorContextual(sp, {"x": 0.5}, model_name="gumbel")]
    for make in rejected:
        with pytest.raises(NotImplementedError, match="gumbel"):
            make()
    m = _m(3)
    assert not _batchable(m)
    m.params = torch.zeros(1)
    with pytest.raises(TypeError, match="GumbelDeepEnsemble"):
        EnsembleBatch([m])


def test_rejected_fit_leaves_the_model_unfitted():
    """The minibatch-envelope check runs before the initial weights are drawn, as DeepEnsemble's does."""
    m = GumbelDeepEnsemble(256, 0, 8, device="cpu", num_layers=3, num_hiddens=256, reduced_dim=129, batch_size=64)
    with pytest.raises(NotImplementedError):
        m.fit(torch.rand(64, 256), None, torch.randn(64, 8))
    assert not m.fitted
