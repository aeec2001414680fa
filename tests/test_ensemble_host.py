"""Host-side contract of hebo_b200.DeepEnsemble (no GPU): constructor keys and defaults of the reference
(deep_ensemble.py:36-51, BaseNet :189-205), rejected options, the envelope, the NaN-row filter, and the raw parameter
layout against BaseNet's registration order (oracle.ensemble_oracle.OracleNet) with its state_dict round trip."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from hebo_b200 import _lib
from hebo_b200.ensemble import DeepEnsemble, init_params, param_layout, raw_to_state_dict, state_dict_to_raw
from oracle import ensemble_oracle as EO

VARIANTS = [  # (num_cont, num_uniqs, enum_trans, num_layers, num_out, output_noise, rand_prior)
    (3, [], "embedding", 1, 1, True, False),
    (2, [4, 7], "embedding", 2, 2, True, True),
    (0, [3, 120], "embedding", 1, 1, False, False),
    (2, [3, 5], "onehot", 3, 2, False, True),
]


def test_defaults_match_the_reference():
    m = DeepEnsemble(2, 0, 1)
    assert dict(bootstrap=m.bootstrap, rand_prior=m.rand_prior, output_noise=m.output_noise, num_ensembles=m.num_ensembles,
                num_processes=m.num_process, num_epochs=m.num_epochs, print_every=m.print_every, num_layers=m.num_layers,
                num_hiddens=m.num_hiddens, l1=m.l1, batch_size=m.batch_size, lr=m.lr, adv_eps=m.adv_eps,
                verbose=m.verbose) == dict(bootstrap=False, rand_prior=False, output_noise=True, num_ensembles=5,
                                           num_processes=1, num_epochs=500, print_every=50, num_layers=1, num_hiddens=128,
                                           l1=1e-3, batch_size=32, lr=5e-3, adv_eps=0., verbose=False)
    assert m.noise_lb == 1e-4 and m.enum_trans == "embedding"
    assert m.support_ts and m.support_grad and m.support_multi_output and m.support_warm_start
    assert torch.equal(m.noise, torch.zeros(1))
    # the reference writes its defaults back into conf (conf.setdefault)
    assert m.conf["num_epochs"] == 500 and m.conf["lr"] == 5e-3


def test_rejected_options():
    class OtherNet(nn.Module):
        pass
    with pytest.raises(NotImplementedError, match="basenet_cls"):
        DeepEnsemble(1, 0, 1, basenet_cls=OtherNet)
    with pytest.raises(NotImplementedError, match="act"):
        DeepEnsemble(1, 0, 1, act=nn.Tanh())
    with pytest.raises(RuntimeError, match="Unknown enum"):
        DeepEnsemble(1, 1, 1, num_uniqs=[3], enum_trans="hash")
    DeepEnsemble(1, 0, 1, act=nn.ReLU(), num_processes=4, bootstrap=True, adv_eps=0.1)     # accepted


@pytest.mark.parametrize("key,value,limit", [("num_layers", 4, "3"), ("num_hiddens", 257, "256"), ("num_ensembles", 33, "32")])
def test_envelope_is_named(key, value, limit):
    with pytest.raises(NotImplementedError, match=f"{key}.*{limit}"):
        DeepEnsemble(2, 0, 1, **{key: value})
    with pytest.raises(NotImplementedError, match="num_out = 9 exceeds the limit of 8"):
        DeepEnsemble(2, 0, 9)
    with pytest.raises(NotImplementedError, match="input width"):
        DeepEnsemble(250, 1, 1, num_uniqs=[20], enum_trans="onehot")
    DeepEnsemble(256, 0, 8, num_layers=3, num_hiddens=256, rand_prior=True)          # the envelope corner


def test_batch_envelope_raises_before_any_device_work():
    m = DeepEnsemble(2, 0, 1, batch_size=64, num_hiddens=256, num_layers=3)
    assert m.batch_floats(64) > _lib.HB_DE_MAX_BATCH_FLOATS
    with pytest.raises(NotImplementedError, match="HB_DE_MAX_BATCH_FLOATS"):
        m.fit(torch.randn(100, 2), None, torch.randn(100, 1))
    corner = DeepEnsemble(256, 0, 8, num_layers=3, num_hiddens=256, rand_prior=True)
    assert corner.batch_floats(32) <= _lib.HB_DE_MAX_BATCH_FLOATS          # BaseNet's default batch at the corner


@pytest.mark.parametrize("v", VARIANTS)
def test_layout_is_basenet_registration_order(v):
    dc, uniqs, trans, L, O, noise, prior = v
    lay, din = param_layout(dc, uniqs, trans, L, 16, O, noise, prior)
    net = EO.OracleNet(dc, uniqs, trans, L, 16, O, noise, prior)
    assert [(n, tuple(p.shape)) for n, p in net.named_parameters()] == [(n, tuple(s)) for n, s in lay]
    spec = _lib.DeSpec(dc, len(uniqs), (C.c_int32 * max(1, len(uniqs)))(*uniqs),
                       _lib.HB_DE_EMBEDDING if trans == "embedding" else _lib.HB_DE_ONEHOT, L, 16, O, int(noise), int(prior), 1e-4)
    P = sum(int(np.prod(s)) for _, s in lay)
    assert _lib.lib().hb_de_num_params(C.byref(spec)) == P
    assert _lib.lib().hb_de_fit_workspace_bytes(C.byref(spec), 5) == 3 * 5 * P * 4
    # raw <-> state_dict without permutation
    raw = torch.randn(P)
    sd = raw_to_state_dict(raw, lay)
    assert torch.equal(state_dict_to_raw(sd, lay), raw)
    net.load_state_dict({k: t.double() for k, t in sd.items()})
    assert torch.equal(net.raw().float(), raw)


def test_envelope_in_the_library():
    lib = _lib.lib()
    u = (C.c_int32 * 1)(3)
    ok = _lib.DeSpec(4, 1, u, 0, 1, 128, 1, 1, 0, 1e-4)
    assert lib.hb_de_num_params(C.byref(ok)) > 0
    for field, bad in (("num_layers", 4), ("num_hiddens", 257), ("num_out", 9), ("num_cont", 256), ("enum_trans", 2)):
        s = _lib.DeSpec(4, 1, u, 0, 1, 128, 1, 1, 0, 1e-4)
        setattr(s, field, bad)
        assert lib.hb_de_num_params(C.byref(s)) == -1, field
    assert lib.hb_de_fit_workspace_bytes(C.byref(ok), 33) == -1
    assert lib.hb_de_num_params(None) == -1


def test_initialisation_follows_basenet():
    lay, _ = param_layout(2, [5], "embedding", 1, 128, 1, True, True)
    torch.manual_seed(3)
    raw = init_params(lay)
    torch.manual_seed(3)
    ref = []
    for name, shape in lay:
        t = torch.empty(shape)
        nn.init.zeros_(t) if "bias" in name else nn.init.xavier_uniform_(t, gain=nn.init.calculate_gain("relu"))
        ref.append(t.reshape(-1))
    assert torch.equal(raw, torch.cat(ref))
    sd = raw_to_state_dict(raw, lay)
    assert float(sd["enum_layer.emb.0.weight"].abs().max()) <= np.sqrt(2) * np.sqrt(6 / (5 + 3)) + 1e-6   # xavier, not N(0,1)
    assert all(float(sd[k].abs().max()) == 0 for k in sd if k.endswith("bias"))


def test_nan_rows_are_filtered_before_scaling():
    m = DeepEnsemble(1, 0, 2)
    X = torch.tensor([[0.], [1.], [2.], [10.]])
    y = torch.tensor([[1., float("nan")], [2., 3.], [float("nan"), float("nan")], [4., 5.]])
    valid = torch.isfinite(y).any(dim=1)
    m.fit_scaler(X[valid], None, y[valid])
    assert torch.allclose(m.xscaler.transform(torch.tensor([[0.], [10.]])), torch.tensor([[-1.], [1.]]))
    assert torch.allclose(m.yscaler.mean, torch.tensor([7 / 3, 4.0]))


@pytest.mark.parametrize("n", [1, 2, 3, 17, 32, 50, 200, 1000, 4097])
def test_oracle_order_is_a_permutation(n):
    for member, epoch in ((0, 0), (3, 7), (1, 499)):
        p = EO.perm(12345, member, epoch, n)
        assert np.array_equal(np.sort(p), np.arange(n))
    if n >= 17:
        assert not np.array_equal(EO.perm(1, 0, 0, n), EO.perm(1, 0, 1, n))
        assert not np.array_equal(EO.perm(1, 0, 0, n), EO.perm(1, 1, 0, n))


def test_fp32_adam_restatement_tracks_fp64():
    g = np.random.RandomState(0)
    p, gr = g.randn(1000).astype(np.float32), g.randn(1000).astype(np.float32)
    m, v = (g.randn(1000) * 0.1).astype(np.float32), (g.rand(1000) * 0.01).astype(np.float32)
    for step in (1, 2, 500):
        p32, m32, v32 = EO.adam_update_f32(p, gr, m, v, step, 5e-3)
        p64, m64, v64 = EO.adam_update(*(torch.tensor(t, dtype=torch.float64) for t in (p, gr, m, v)), step, 5e-3)
        assert np.abs(p32 - p64.numpy()).max() < 1e-6
        assert np.allclose(m32, m64.numpy(), rtol=1e-6, atol=1e-7) and np.allclose(v32, v64.numpy(), rtol=1e-5, atol=1e-10)


def test_out_of_range_categories_raise_like_the_reference():
    # nn.Embedding raises IndexError and F.one_hot RuntimeError in the reference; this model raises IndexError for both
    for trans in ("embedding", "onehot"):
        m = DeepEnsemble(1, 2, 1, num_uniqs=[3, 4], enum_trans=trans, num_epochs=1)
        X, y = torch.randn(10, 1), torch.randn(10, 1)
        for bad in (3, -1):
            Xe = torch.zeros(10, 2, dtype=torch.long)
            Xe[5, 0] = bad
            with pytest.raises(IndexError):
                m.fit(X, Xe, y)
            with pytest.raises(IndexError):
                m.predict(X, Xe)
            with pytest.raises(IndexError):
                m.predict_mace(X, 0.0, 1.0, Xe=Xe)
        Xe = torch.zeros(10, 2, dtype=torch.long)
        Xe[0, 1] = 4
        with pytest.raises(IndexError):
            m.fit(X, Xe, y)


def test_caller_given_order_is_checked():
    m = DeepEnsemble(1, 0, 1, num_ensembles=2, num_epochs=1)
    X, y = torch.randn(6, 1), torch.randn(6, 1)
    good = torch.stack([torch.randperm(6) for _ in range(2)]).reshape(2, 1, 6)
    with pytest.raises(ValueError, match="permutation"):
        bad = good.clone()
        bad[1, 0, 2] = 6
        m.fit(X, None, y, perm=bad)
    with pytest.raises(ValueError, match="permutation"):
        bad = good.clone()
        bad[0, 0, 0] = bad[0, 0, 1]
        m.fit(X, None, y, perm=bad)
    with pytest.raises(ValueError, match="num_epochs"):
        m.fit(X, None, y, perm=good[:, :, :5])


def test_basenet_cls_must_be_the_reference_class():
    class BaseNet(nn.Module):          # a look-alike with the same name outside the reference's module
        pass
    with pytest.raises(NotImplementedError, match="basenet_cls"):
        DeepEnsemble(1, 0, 1, basenet_cls=BaseNet)
    ref = type("BaseNet", (nn.Module,), {"__module__": "hebo.models.nn.deep_ensemble"})
    DeepEnsemble(1, 0, 1, basenet_cls=ref)
