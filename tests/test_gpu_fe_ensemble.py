"""hb_fe_fit / hb_fe_predict and hebo_b200.FeDeepEnsemble on the device: replay of the reference's own FeDeepEnsemble
fits (tests/golden/make_ref_fe_deep_ensemble.py), the Philox gate streams against their restatement, and the reference's
model and optimiser tests mirrored for model_name='fe_deep_ensemble' (HEBO/test/test_concrete.py, test_deep_ensemble.py,
test_optimizer.py)."""
import functools

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import BO, FeDeepEnsemble, LCB, Mean, Sigma, AbsEtaDifference
from hebo_b200.acq import ga_score
from hebo_b200.ensemble import fe_epoch_temperature, init_params
from hebo_b200.space import DesignSpace
from hebo_b200.suggest import HEBO
from oracle import rng_oracle as R
from tests.util import load_golden

pytestmark = pytest.mark.gpu

REF = load_golden("ref_fe_deep_ensemble.npz")
LAYERS = ["stg", "concrete", "hard_concrete"]
REF_INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]


def _ref_model(p, **kw):
    li, noise, inp, O, prior = (int(v) for v in REF[p + "cfg"])
    dc, uniqs, trans = REF_INPUTS[inp]
    m = FeDeepEnsemble(dc, len(uniqs), O, num_ensembles=2, num_epochs=3, batch_size=8, num_hiddens=8, num_layers=1,
                       output_noise=bool(noise), rand_prior=bool(prior), enum_trans=trans, num_uniqs=uniqs,
                       fe_layer=LAYERS[li], **kw)
    return m, dc, uniqs


def _inputs(p, dc, uniqs, held_out=False):
    xc, xe = ("Xs", "Xes") if held_out else ("Xc", "Xe")
    return (torch.from_numpy(REF[p + xc]) if dc else None), (torch.from_numpy(REF[p + xe]) if uniqs else None)


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_three_epochs_track_the_reference_trajectory(vi):
    """3 epochs from the reference's initial weights over its own DataLoader order and gate draws, against the parameters
    its fp32 fit reached, with the tolerance of the deep ensemble's replay (test_gpu_ensemble.py)."""
    p = f"v{vi}_"
    m, dc, uniqs = _ref_model(p)
    Xc, Xe = _inputs(p, dc, uniqs)
    y = torch.from_numpy(REF[p + "y"])
    m.params = torch.from_numpy(REF[p + "init"]).cuda().contiguous()
    m.fit(Xc, Xe, y, perm=torch.from_numpy(REF[p + "order"]).int(), draws=torch.from_numpy(REF[p + "draws"]),
          eval_draws=torch.from_numpy(REF[p + "noise_draws"]))
    torch.cuda.synchronize()
    assert m.params.shape == (2, m.P) and REF[p + "init"].shape == (2, m.P)
    steps = REF[p + "temps"].shape[2] * 3
    for e in range(2):
        d = (m.params[e].cpu().double() - torch.from_numpy(REF[p + "epoch3"][e]).double()).abs()
        assert float(d.max()) <= 2 * m.lr * steps
        assert float((d > 1e-4).double().mean()) <= 0.01, float(d.max())
    # the temperature of every training forward, and predict's
    temps = REF[p + "temps"]
    for ep in range(3):
        want = 1.0 if m.fe_layer == "stg" else fe_epoch_temperature(1.0, 0.1, 0.99, ep)
        assert (temps[:, ep, :] == np.float32(want)).all()
    assert m.gate_temperature == float(REF[p + "eval_temp"][0])


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_predict_and_noise_from_the_reference_parameters(vi):
    """predict with the reference's fitted parameters, scalers and eval draws against its predict; noise likewise."""
    p = f"v{vi}_"
    m, dc, uniqs = _ref_model(p)
    Xc, Xe = _inputs(p, dc, uniqs)
    y = torch.from_numpy(REF[p + "y"])
    m.fit(Xc, Xe, y)                        # the scalers (identical to the reference's: test_gpu_ensemble.py checks them)
    m.params = torch.from_numpy(REF[p + "epoch3"]).cuda().contiguous()
    m.gate_temperature = float(REF[p + "eval_temp"][0])
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


def _small(fe_layer, **kw):
    torch.manual_seed(3)
    g = torch.Generator().manual_seed(4)
    Xc = torch.rand(40, 4, generator=g) * 2 - 1
    Xe = torch.randint(0, 3, (40, 1), generator=g)
    y = (Xc[:, :1] ** 2 + Xe.float()) + 0.01 * torch.randn(40, 1, generator=g)
    conf = dict(num_ensembles=3, num_epochs=6, num_hiddens=16, num_uniqs=[3], fe_layer=fe_layer)
    conf.update(kw)
    m = FeDeepEnsemble(4, 1, 1, **conf)
    return m, Xc, Xe, y


@pytest.mark.parametrize("fe_layer", LAYERS)
def test_fit_is_bit_identical_from_run_to_run(fe_layer):
    outs = []
    for _ in range(2):
        m, Xc, Xe, y = _small(fe_layer)
        m.fit(Xc, Xe, y)
        outs.append((m.params.cpu(), m.losses.cpu(), m.noise.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    assert bool(torch.isfinite(outs[0][0]).all())


def _eval_draws_restated(m, seed, counter):
    """The raw eval draws [E, din] of hb_fe_predict's Philox stream: column k of member e takes half k % 2 of the block
    (counter, (e << 16) | k / 2, 0x46454556)."""
    E, din = m.num_ensembles, m.din
    e = np.repeat(np.arange(E, dtype=np.uint64), din)
    k = np.tile(np.arange(din, dtype=np.uint64), E)
    stream = (np.uint64(0x46454556) << np.uint64(32)) | (e << np.uint64(16)) | (k >> np.uint64(1))
    half = (k & np.uint64(1)).astype(bool)
    w0, w1 = R.normal_words(seed, np.full(E * din, counter, dtype=np.uint64), stream)
    if m.fe_layer == "stg":
        z0, z1, _, _ = R.box_muller(R.uniform(w0), R.uniform(w1))
        return torch.from_numpy(np.where(half, z1, z0).reshape(E, din)).float()
    return torch.from_numpy(np.where(half, R.uniform(w1), R.uniform(w0)).reshape(E, din))


@pytest.mark.parametrize("fe_layer", LAYERS)
def test_eval_masks_follow_the_restated_philox_stream(fe_layer):
    m, Xc, Xe, y = _small(fe_layer)
    m.fit(Xc, Xe, y)
    a = m.predict(Xc, Xe, seed=77, counter=5)
    b = m.predict(Xc, Xe, seed=77, counter=5)
    c = m.predict(Xc, Xe, seed=77, counter=6)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(a[0], c[0])
    r = m.predict(Xc, Xe, draws=_eval_draws_restated(m, 77, 5))
    if fe_layer == "stg":       # Box-Muller: the device's logf / sincospif against fp64, a few ulps per draw
        assert torch.allclose(r[0], a[0], rtol=1e-5, atol=1e-5) and torch.allclose(r[1], a[1], rtol=1e-4, atol=1e-6)
    else:                       # the uniforms are exact
        assert torch.equal(r[0], a[0]) and torch.equal(r[1], a[1])
    f = m.sample_f()
    assert f(Xc, Xe).shape == (40, 1)


@pytest.mark.parametrize("fe_layer", LAYERS)
def test_training_draws_follow_the_restated_philox_stream(fe_layer):
    """A fit with draws = the restated training stream equals the fit on the device's own Philox draws: bit for bit for
    the concrete layers (exact uniforms), within the Box-Muller's few ulps for stg."""
    m, Xc, Xe, y = _small(fe_layer, num_epochs=2, batch_size=16)
    m.fit(Xc, Xe, y)
    got, seed = m.params.cpu(), m.seed
    m2, *_ = _small(fe_layer, num_epochs=2, batch_size=16)
    E, T, nb, B, din = m2.draws_shape(40)
    q = np.arange(T * nb * B * din, dtype=np.uint64)
    draws = []
    for e in range(E):
        stream = np.full(q.shape, (0x46454654 << 32) | e, dtype=np.uint64)
        w0, w1 = R.normal_words(seed, q >> np.uint64(1), stream)
        half = (q & np.uint64(1)).astype(bool)
        if fe_layer == "stg":
            z0, z1, _, _ = R.box_muller(R.uniform(w0), R.uniform(w1))
            draws.append(np.where(half, z1, z0).astype(np.float32))
        else:
            draws.append(np.where(half, R.uniform(w1), R.uniform(w0)))
    draws = torch.from_numpy(np.stack(draws).reshape(E, T, nb, B, din))
    torch.manual_seed(3)                  # the same initial weights and seed
    m2.fit(Xc, Xe, y, draws=draws)
    assert m2.seed == seed
    if fe_layer == "stg":
        assert float((m2.params.cpu() - got).abs().max()) < 1e-3
    else:
        assert torch.equal(m2.params.cpu(), got)


# ---------------------------------------------------------------- HEBO/test/test_concrete.py, test_deep_ensemble.py
@pytest.mark.parametrize("fe_layer", LAYERS)
def test_fe_ensemble(fe_layer):
    torch.manual_seed(0)
    x = torch.randn(300, 10)
    y = x[:, 0].view(-1, 1)
    model = FeDeepEnsemble(x.shape[1], 0, 1, output_noise=False, num_ensembles=1, num_processes=1, num_epochs=1,
                           fe_layer=fe_layer)
    model.fit(x, None, y)
    with torch.no_grad():
        py, ps2 = model.predict(x, None)
    assert py.shape == (300, 1) and bool(torch.isfinite(py).all()) and bool((ps2 > 0).all())


@pytest.mark.parametrize("output_noise", [True, False], ids=["nll", "mse"])
@pytest.mark.parametrize("rand_prior", [True, False], ids=["with_prior", "no_prior"])
def test_deep_ens(output_noise, rand_prior):
    xc = torch.randn(16, 1)
    y = xc ** 2
    model = FeDeepEnsemble(1, 0, 1, output_noise=output_noise, rand_prior=rand_prior, num_processes=1, l1=0., num_epochs=1)
    model.fit(xc, None, y)
    assert model.params.shape[0] == model.num_ensembles
    with torch.no_grad():
        py, ps2 = model.predict(xc, None)
    assert py.shape == (16, 1) and bool(torch.isfinite(py).all()) and bool((ps2 > 0).all())
    s = model.sample_y(xc, None, n_samples=3)
    assert s.shape == (3, 16, 1) and bool(torch.isfinite(s).all())


def test_warm_start_continues_from_the_previous_members():
    m, Xc, Xe, y = _small("concrete")
    m.fit(Xc, Xe, y)
    p1 = m.params.clone()
    m.fit(Xc, Xe, y)
    assert not torch.equal(m.params, p1) and bool(torch.isfinite(m.params).all())


class _AtDraws:
    """The model with predict pinned to one (seed, counter): acq.eval then sees the masks the device scorer drew."""

    def __init__(self, m, seed, counter):
        self.m, self.seed, self.counter = m, seed, counter

    def predict(self, x, xe):
        return self.m.predict(x, xe, seed=self.seed, counter=self.counter)


@pytest.mark.parametrize("acq_cls", [LCB, Mean, Sigma, AbsEtaDifference])
def test_device_scorer_equals_eval_on_predict(acq_cls):
    m, Xc, Xe, y = _small("stg")
    m.fit(Xc, Xe, y)
    acq = acq_cls(m, kappa=2.0, eta=0.1) if acq_cls is AbsEtaDifference else acq_cls(m, kappa=2.0)
    score = ga_score(acq, seed=123)
    xc, xe = Xc.cuda().contiguous(), Xe.cuda().int().contiguous()
    f = score(xc, xe, 4)
    g = score(xc, xe, 5)
    acq.model = _AtDraws(m, 123, 4)
    want = torch.as_tensor(acq.eval(xc, xe)).reshape(-1)
    assert torch.allclose(f, want.to(f.device, torch.float32), rtol=1e-6, atol=1e-6)
    assert not torch.equal(f, g)          # a new generation draws new masks


# ---------------------------------------------------------------- HEBO/test/test_optimizer.py for 'fe_deep_ensemble'
def _obj(x: pd.DataFrame) -> np.ndarray:
    return x["x0"].values.astype(float).reshape(-1, 1) ** 2


@pytest.mark.parametrize("opt_cls", [BO, HEBO, functools.partial(HEBO, acq_optimizer="nsga2", evo_iters=30)],
                         ids=["bo", "hebo", "hebo-nsga2"])
def test_opt(opt_cls):
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    opt = opt_cls(space, rand_sample=8, model_name="fe_deep_ensemble")
    for i in range(11):
        rec = opt.suggest(n_suggestions=1)
        y = _obj(rec)
        opt.observe(rec, y)
    assert opt.y.shape[0] == 11 and np.isfinite(opt.y).all()
    assert ((opt.X["x0"] >= -3) & (opt.X["x0"] <= 7)).all()


def test_initial_gate_is_small_and_last():
    torch.manual_seed(1)
    m = FeDeepEnsemble(3, 0, 1, num_ensembles=2)
    raw = init_params(m.layout)
    assert raw.numel() == m.P and float(raw[-m.din:].abs().max()) < 0.05
