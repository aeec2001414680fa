"""hb_gumbel_fit / hb_gumbel_predict and hebo_b200.GumbelDeepEnsemble on the device: replay of the reference's own
GumbelDeepEnsemble fits (tests/golden/make_ref_gumbel_ensemble.py), run-to-run identity, per-call selection draws, the
temperature limits of the selection layer, and the optimisers with model_name='gumbel'."""
import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import BO, GumbelDeepEnsemble, LCB, Mean, Sigma, AbsEtaDifference
from hebo_b200.acq import ga_score
from hebo_b200.ensemble import gumbel_epoch_temperature
from hebo_b200.space import DesignSpace
from hebo_b200.suggest import HEBO
from oracle import rng_oracle as R
from tests.util import load_golden

pytestmark = pytest.mark.gpu

REF = load_golden("ref_gumbel_ensemble.npz")
REF_INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]


def _ref_model(p):
    noise, inp, O, rm, r, prior, N = (int(v) for v in REF[p + "cfg"])
    dc, uniqs, trans = REF_INPUTS[inp]
    m = GumbelDeepEnsemble(dc, len(uniqs), O, num_ensembles=2, num_epochs=3, batch_size=8, num_hiddens=8, num_layers=1,
                           output_noise=bool(noise), rand_prior=bool(prior), enum_trans=trans, num_uniqs=uniqs,
                           reduced_dim=r)
    return m, dc, uniqs


def _inputs(p, dc, uniqs, held_out=False):
    xc, xe = ("Xs", "Xes") if held_out else ("Xc", "Xe")
    return (torch.from_numpy(REF[p + xc]) if dc else None), (torch.from_numpy(REF[p + xe]) if uniqs else None)


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_three_epochs_track_the_reference_trajectory(vi):
    """3 epochs from the reference's initial weights over its own DataLoader order (no drop_last) and selection draws,
    against the parameters its fp32 fit reached, with the tolerance of the deep ensemble's replay."""
    p = f"v{vi}_"
    m, dc, uniqs = _ref_model(p)
    Xc, Xe = _inputs(p, dc, uniqs)
    y = torch.from_numpy(REF[p + "y"])
    m.params = torch.from_numpy(REF[p + "init"]).cuda().contiguous()
    m.fit(Xc, Xe, y, perm=torch.from_numpy(REF[p + "order"]).int(), draws=torch.from_numpy(REF[p + "draws"]),
          eval_draws=torch.from_numpy(REF[p + "noise_draws"]))
    torch.cuda.synchronize()
    assert m.params.shape == (2, m.P) and REF[p + "init"].shape == (2, m.P)
    for e in range(2):
        d = (m.params[e].cpu().double() - torch.from_numpy(REF[p + "epoch3"][e]).double()).abs()
        assert float((d > 1e-4).double().mean()) <= 0.01, float(d.max())
    for ep in range(3):
        assert (REF[p + "temps"][:, ep, :] == 0.8 ** ep + 0.1).all()
    assert m.temperature == gumbel_epoch_temperature(2) == float(np.float32(REF[p + "eval_temp"][0]))


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_predict_and_noise_from_the_reference_parameters(vi):
    """predict with the reference's fitted parameters, scalers and eval draws against its predict; noise likewise."""
    p = f"v{vi}_"
    m, dc, uniqs = _ref_model(p)
    Xc, Xe = _inputs(p, dc, uniqs)
    y = torch.from_numpy(REF[p + "y"])
    m.fit(Xc, Xe, y)
    m.params = torch.from_numpy(REF[p + "epoch3"]).cuda().contiguous()
    Xs, Xes = _inputs(p, dc, uniqs, held_out=True)
    py, ps2 = m.predict(Xs, Xes, draws=torch.from_numpy(REF[p + "pred_draws"]))
    ystd = float(m.yscaler.std.max())
    assert torch.allclose(py.double(), torch.from_numpy(REF[p + "py"]).double(), rtol=1e-4, atol=1e-4 * ystd)
    assert torch.allclose(ps2.double(), torch.from_numpy(REF[p + "ps2"]).double(), rtol=1e-3, atol=1e-6 * ystd ** 2)
    pn, _ = m.predict(Xc, Xe, draws=torch.from_numpy(REF[p + "noise_draws"]))
    valid = torch.isfinite(y).any(1)
    noise = ((pn - y)[valid] ** 2).mean(0)
    ref = torch.from_numpy(REF[p + "noise"])
    fin = torch.isfinite(ref)
    assert torch.allclose(noise[fin].double(), ref[fin].double(), rtol=1e-3, atol=1e-6)


def _data(n=50, d=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g) * 2 - 1
    y = (X[:, :1] ** 2 + 0.3 * X[:, 1:2]) + 0.01 * torch.randn(n, 1, generator=g)
    return X, y


def test_fit_is_identical_from_run_to_run_and_predict_follows_the_counter():
    X, y = _data()
    out = []
    for _ in range(2):
        torch.manual_seed(3)
        m = GumbelDeepEnsemble(4, 0, 1, num_epochs=20, num_hiddens=16)
        m.fit(X, None, y)
        out.append((m.params.clone(), m.fit_state()[2].clone(), m.losses.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    Xs = torch.rand(100, 4) * 2 - 1
    p1, v1 = m.predict(Xs, None, seed=7, counter=1)
    p1b, v1b = m.predict(Xs, None, seed=7, counter=1)
    p2, _ = m.predict(Xs, None, seed=7, counter=2)
    assert torch.equal(p1, p1b) and torch.equal(v1, v1b)
    assert not torch.equal(p1, p2)
    # every candidate tile of one call uses the same W per member: a split call with the same (seed, counter) equals it
    a, va = m.predict(Xs[:37], None, seed=7, counter=1)
    b, vb = m.predict(Xs[37:], None, seed=7, counter=1)
    assert torch.equal(torch.cat([a, b]), p1) and torch.equal(torch.cat([va, vb]), v1)


def _uniforms(seed, row, stream, half):
    w0, w1 = R.normal_words(seed, row, stream)
    return np.where(half, R.uniform(w1), R.uniform(w0))


def test_training_draws_follow_the_restated_philox_stream():
    """A fit on draws = the restated training stream (q / 2, member, 'GBFT') equals the fit on the device's own Philox
    draws bit for bit (the uniforms are exact)."""
    X, y = _data(40, 5)
    torch.manual_seed(8)
    m = GumbelDeepEnsemble(5, 0, 1, num_epochs=3, num_hiddens=16, num_ensembles=3, batch_size=16)
    m.fit(X, None, y)
    got, seed = m.params.cpu(), m.seed
    E, T, nb, r, dc = m.draws_shape(40)
    q = np.arange(T * nb * r * dc, dtype=np.uint64)
    draws = np.stack([_uniforms(seed, q >> np.uint64(1), np.full(q.shape, (0x47424654 << 32) | e, dtype=np.uint64),
                                (q & np.uint64(1)).astype(bool)) for e in range(E)]).reshape(E, T, nb, r, dc)
    torch.manual_seed(8)
    m2 = GumbelDeepEnsemble(5, 0, 1, num_epochs=3, num_hiddens=16, num_ensembles=3, batch_size=16)
    m2.fit(X, None, y, draws=torch.from_numpy(draws))
    assert m2.seed == seed and torch.equal(m2.params.cpu(), got)


def test_eval_draws_follow_the_restated_philox_stream():
    """predict on draws = the restated eval stream (counter, (member << 16) | q / 2, 'GBEV') equals predict on the
    device's own draws for that (seed, counter), bit for bit; sample_f's member likewise."""
    X, y = _data(40, 5)
    m = GumbelDeepEnsemble(5, 0, 1, num_epochs=10, num_hiddens=16, num_ensembles=3)
    m.fit(X, None, y)
    E, r, dc = 3, m.reduced_dim, 5
    q = np.arange(r * dc, dtype=np.uint64)
    draws = np.stack([_uniforms(77, np.full(q.shape, 5, dtype=np.uint64),
                                (0x47424556 << 32) | (e << 16) | (q >> np.uint64(1)), (q & np.uint64(1)).astype(bool))
                      for e in range(E)]).reshape(E, r, dc)
    a = m.predict(X, None, seed=77, counter=5)
    b = m.predict(X, None, draws=torch.from_numpy(draws).float())
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


class _AtDraws:
    """The model with predict pinned to one (seed, counter): acq.eval then sees the W the device scorer drew."""

    def __init__(self, m, seed, counter):
        self.m, self.seed, self.counter = m, seed, counter

    def predict(self, x, xe):
        return self.m.predict(x, xe, seed=self.seed, counter=self.counter)


@pytest.mark.parametrize("acq_cls", [LCB, Mean, Sigma, AbsEtaDifference])
def test_device_scorer_equals_eval_on_predict(acq_cls):
    X, y = _data(40, 4)
    m = GumbelDeepEnsemble(4, 0, 1, num_epochs=10, num_hiddens=16)
    m.fit(X, None, y)
    acq = acq_cls(m, kappa=2.0, eta=0.1) if acq_cls is AbsEtaDifference else acq_cls(m, kappa=2.0)
    score = ga_score(acq, seed=123)
    xc, xe = X.cuda().contiguous(), torch.zeros(40, 0, dtype=torch.int32, device="cuda")
    f = score(xc, xe, 4)
    g = score(xc, xe, 5)
    acq.model = _AtDraws(m, 123, 4)
    want = torch.as_tensor(acq.eval(xc, xe)).reshape(-1)
    assert torch.allclose(f, want.to(f.device, torch.float32), rtol=1e-6, atol=1e-6)
    assert not torch.equal(f, g)          # a new generation draws a new W


def test_selection_at_temperature_limits():
    """test_gumbel_linear's claim through predict: at T = 1e-6 with r = 1 W is one-hot on a single column; at T = 1e6 it
    is close to the uniform average of the columns."""
    d = 5
    m = GumbelDeepEnsemble(d, 0, 1, num_epochs=0, num_hiddens=8, reduced_dim=1, num_ensembles=1, output_noise=False)
    X, y = _data(20, d)
    m.fit(X, None, y)
    with torch.no_grad():          # the member's hidden input is x_sel: read it through a linear, bias-free net
        raw = m.state_dicts()[0]
        raw["hidden.0.weight"].zero_()
        raw["hidden.0.weight"][0, 0] = 1.0
        raw["hidden.0.bias"].zero_()
        raw["mu.weight"].zero_()
        raw["mu.weight"][0, 0] = 1.0
        raw["mu.bias"].zero_()
        raw["feature_select.logits"].copy_(torch.tensor([[0.0, 0.3, -0.2, 0.1, 0.0]]))
        from hebo_b200.ensemble import state_dict_to_raw
        m.params = state_dict_to_raw(raw, m.layout).reshape(1, -1).cuda().contiguous()
    Xs = torch.rand(64, d) * 2 - 1
    xs = m.xscaler.transform(Xs).double()
    ym, ys = float(m.yscaler.mean), float(m.yscaler.std)
    m.temperature = 1e-6
    for c in range(4):
        py, _ = m.predict(Xs, None, seed=11, counter=c)
        sel = (py.double().reshape(-1) - ym) / ys
        cols = [k for k in range(d) if torch.allclose(sel, xs[:, k].clamp_min(0), atol=1e-4)]
        assert len(cols) == 1
    m.temperature = 1e6
    py, _ = m.predict(Xs, None, seed=11, counter=0)
    assert torch.allclose((py.double().reshape(-1) - ym) / ys, xs.mean(1).clamp_min(0), atol=1e-4)


@pytest.mark.parametrize("noise", [True, False])
@pytest.mark.parametrize("prior", [True, False])
def test_deep_ens_gumbel(noise, prior):
    """test_deep_ensemble.py::test_deep_ens[GumbelDeepEnsemble]: a fit on one numeric column predicts finite values with
    positive variance, and sample_f returns one member's prediction."""
    X = torch.randn(10, 1)
    y = X ** 2
    m = GumbelDeepEnsemble(1, 0, 1, num_epochs=10, output_noise=noise, rand_prior=prior)
    m.fit(X, None, y)
    py, ps2 = m.predict(X, None)
    assert torch.isfinite(py).all() and (ps2 > 0).all()
    f = m.sample_f()
    assert f(X, None).shape == (10, 1)


def test_gumbel_ensemble_with_categories():
    """test_deep_ensemble.py::test_gumbel_ensemble / test_gumbel_net: mixed inputs, the default reduced_dim."""
    Xc = torch.randn(30, 6)
    Xe = torch.randint(0, 3, (30, 2))
    y = Xc[:, :1] + Xe[:, :1].float()
    m = GumbelDeepEnsemble(6, 2, 1, num_uniqs=[3, 3], num_epochs=20)
    assert m.reduced_dim == 4
    m.fit(Xc, Xe, y)
    py, ps2 = m.predict(Xc, Xe)
    assert py.shape == (30, 1) and torch.isfinite(py).all() and (ps2 > 0).all()


def _space():
    return DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(3)] +
                               [{"name": "c", "type": "cat", "categories": ["a", "b", "c"]}])


def _obj(df):
    return (df[["x0", "x1", "x2"]].values ** 2).sum(1, keepdims=True) + (df["c"] == "b").values[:, None]


@pytest.mark.parametrize("opt", ["hebo", "hebo_nsga2", "bo"])
def test_optimisers_run_with_gumbel(opt):
    sp = _space()
    if opt == "bo":
        o = BO(sp, model_name="gumbel", rand_sample=4, iters=5)
    else:
        o = HEBO(sp, model_name="gumbel", rand_sample=4, acq_optimizer="nsga2" if opt == "hebo_nsga2" else "sobol",
                 evo_iters=5, n_candidates=500)
    for _ in range(6):
        rec = o.suggest(1)
        assert isinstance(rec, pd.DataFrame) and len(rec) == 1
        o.observe(rec, _obj(rec))
    assert np.isfinite(o.y).all()
