"""oracle/ensemble_oracle.py against tests/golden/ref_deep_ensemble.npz, the stored outputs of the reference's own
DeepEnsemble (tests/golden/make_ref_deep_ensemble.py): the layout of the recorded state_dicts, the first Adam step and 3
epochs of fit_one replayed over the reference's own minibatch order, predict, noise and sample_f (no GPU)."""
import numpy as np
import pytest
import torch

from hebo_b200.ensemble import param_layout
from oracle import ensemble_oracle as EO
from tests.util import load_golden

G = load_golden("ref_deep_ensemble.npz")
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (0, [3, 5], "embedding"), (2, [3, 5], "onehot")]
H, BATCH, LR, L1 = 8, 8, 5e-3, 1e-3
VARIANTS = range(int(G["num_variants"]))


def variant(vi):
    p = f"v{vi}_"
    noise, prior, inp, O, L = (int(v) for v in G[p + "cfg"])
    dc, uniqs, trans = INPUTS[inp]
    return p, dict(noise=bool(noise), prior=bool(prior), dc=dc, uniqs=uniqs, trans=trans, O=O, L=L)


def nets(c, raws):
    return [EO.OracleNet(c["dc"], c["uniqs"], c["trans"], c["L"], H, c["O"], c["noise"], c["prior"]).load_raw(r) for r in raws]


def fit_data(p, c):
    xs = torch.from_numpy(G[p + "xs_fit"]).double()
    xe = torch.from_numpy(G[p + "xe_fit"]).long() if c["uniqs"] else None
    return xs, xe, torch.from_numpy(G[p + "ys_fit"]).double()


@pytest.mark.parametrize("vi", VARIANTS)
def test_recorded_state_dict_has_the_raw_layout(vi):
    p, c = variant(vi)
    lay, _ = param_layout(c["dc"], c["uniqs"], c["trans"], c["L"], H, c["O"], c["noise"], c["prior"])
    assert G[p + "init"].shape[1] == sum(int(np.prod(s)) for _, s in lay)


@pytest.mark.parametrize("vi", VARIANTS)
def test_first_step_and_three_epochs_replay_the_reference(vi):
    p, c = variant(vi)
    xs, xe, ys = fit_data(p, c)
    n = ys.shape[0]
    order = G[p + "order"]
    for e, net in enumerate(nets(c, G[p + "init"])):
        _, g = EO.step_grad(net, xs, xe, ys, order[e, 0, :BATCH], L1, n)
        z = torch.zeros_like(g)
        p1, _, _ = EO.adam_update(net.raw(), g, z, z, 1, LR)
        # the reference runs in fp32: one step moves every parameter by about lr, rounded at the parameter's scale
        assert float((p1 - torch.from_numpy(G[p + "step1"][e]).double()).abs().max()) < 2e-6
        EO.fit(net, xs, xe, ys, order[e], LR, L1, BATCH)
        assert float((net.raw() - torch.from_numpy(G[p + "epoch3"][e]).double()).abs().max()) < 2e-5


@pytest.mark.parametrize("vi", VARIANTS)
def test_predict_noise_and_sample_f_match_the_reference(vi):
    p, c = variant(vi)
    ns = nets(c, G[p + "epoch3"])
    Xs = torch.from_numpy(G[p + "Xs"]) if c["dc"] else None
    Xes = torch.from_numpy(G[p + "Xes"]).long() if c["uniqs"] else None
    xm, xa, ym, ys = (G[p + k] for k in ("x_scale", "x_min", "y_mean", "y_std"))
    with torch.no_grad():
        py, ps2 = EO.ensemble_predict(ns, Xs, Xes, xm, xa, ym, ys, c["noise"])
        scale = float(np.abs(ys).max())
        assert float((py - torch.from_numpy(G[p + "py"]).double()).abs().max()) < 1e-5 * scale
        ref = torch.from_numpy(G[p + "ps2"]).double()
        assert float(((ps2 - ref).abs() / (ref.abs() + 1e-6 * scale ** 2)).max()) < 1e-4
        if c["dc"]:
            for k in range(len(ns)):
                f = EO.member_mu(ns[k], Xs, Xes, xm, xa, ym, ys)
                assert float((f - torch.from_numpy(G[p + "sample_f"][k]).double()).abs().max()) < 1e-5 * scale
        # noise: mean squared error of predict on the training rows that have a finite entry (deep_ensemble.py:89-93)
        Xc, Xe, y = (torch.from_numpy(G[p + k]) for k in ("Xc", "Xe", "y"))
        tr, _ = EO.ensemble_predict(ns, Xc if c["dc"] else None, Xe.long() if c["uniqs"] else None, xm, xa, ym, ys, c["noise"])
        valid = torch.isfinite(y).any(1)
        noise = ((tr - y.double())[valid] ** 2).mean(0)
        assert np.allclose(noise.numpy(), G[p + "noise"], rtol=1e-4, atol=1e-7, equal_nan=True)


def test_reference_rmse_spread_is_stored():
    r = G["rmse_ref"]
    assert r.shape == (3, 2) and bool(np.isfinite(r).all()) and float(r.max()) < 0.1
