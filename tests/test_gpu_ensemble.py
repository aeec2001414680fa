"""hb_de_fit / hb_de_predict / hb_de_predict_grad and hebo_b200.DeepEnsemble on the device, against the fp64 restatement
of the reference (oracle/ensemble_oracle.py), and the reference's model and optimiser tests mirrored for
model_name='deep_ensemble' (HEBO/test/test_base_model.py, test_optimizer.py)."""
import functools
import itertools

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import BO, DeepEnsemble, MOMeanSigmaLCB, _lib
from hebo_b200.suggest import HEBO
from hebo_b200.ensemble import init_params
from hebo_b200.space import DesignSpace
from oracle import ensemble_oracle as EO
from tests.util import load_golden

pytestmark = pytest.mark.gpu

F64 = torch.float64
# (num_cont, num_uniqs, enum_trans)
INPUTS = {"cont": (3, [], "embedding"), "mixed": (2, [4, 7], "embedding"), "enum": (0, [3, 5], "embedding"),
          "onehot": (2, [3, 5], "onehot")}
VARIANTS = list(itertools.product([True, False], [False, True], list(INPUTS), [1, 2], [1, 2]))
VID = [f"{'nll' if a else 'mse'}-{'prior' if b else 'noprior'}-{c}-out{d}-L{e}" for a, b, c, d, e in VARIANTS]


def _data(dc, uniqs, O, n, seed, nan=True):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, dc, generator=g) * 4 - 1 if dc else None
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in uniqs], 1) if uniqs else None
    base = (Xc.sum(1, keepdim=True) if dc else 0) + (Xe.float().sum(1, keepdim=True) if uniqs else 0)
    y = torch.cat([torch.sin(base + k) for k in range(O)], 1) + 0.05 * torch.randn(n, O, generator=g)
    if O == 2 and nan:
        y[1, 0] = float("nan")       # one masked entry (the row stays: its other output is finite)
        y[4, :] = float("nan")       # one filtered row
    return Xc, Xe, y


def _model(v, E=2, **kw):
    noise, prior, inp, O, L = v
    dc, uniqs, trans = INPUTS[inp]
    conf = dict(num_ensembles=E, num_layers=L, num_hiddens=24, output_noise=noise, rand_prior=prior, enum_trans=trans,
                num_uniqs=uniqs)
    conf.update(kw)
    return DeepEnsemble(dc, len(uniqs), O, **conf), dc, uniqs, O


def _scaled(m, Xc, Xe, y):
    valid = torch.isfinite(y).any(dim=1)
    Xc_t, Xe_t, y_t = m.trans(Xc[valid] if Xc is not None else None, Xe[valid] if Xe is not None else None, y[valid])
    return Xc_t.double(), Xe_t, y_t.double()


def _nets(m, raw):
    dc = m.num_cont
    return [EO.OracleNet(dc, m.num_uniqs, m.enum_trans, m.num_layers, m.num_hiddens, m.num_out, m.output_noise, m.rand_prior,
                         m.noise_lb).load_raw(raw[i].double().cpu()) for i in range(raw.shape[0])]


def _fit_with(m, Xc, Xe, y, raw0, perm):
    m.params = raw0.clone().cuda().contiguous()
    m.fit(Xc, Xe, y, perm=perm)
    torch.cuda.synchronize()


@pytest.mark.parametrize("v", VARIANTS, ids=VID)
def test_one_step_gradient_and_adam_update(v):
    torch.manual_seed(0)
    m, dc, uniqs, O = _model(v, num_epochs=1, batch_size=9)
    Xc, Xe, y = _data(dc, uniqs, O, 14, 1)
    n = int(torch.isfinite(y).any(1).sum())
    raw0 = torch.stack([init_params(m.layout) for _ in range(2)])
    perm = torch.stack([torch.randperm(n) for _ in range(2)]).reshape(2, 1, n).int()
    _fit_with(m, Xc, Xe, y, raw0, perm)
    m1, m2, g = (t.cpu() for t in m.fit_state())
    xs, xe, ys = _scaled(m, Xc, Xe, y)
    for e, net in enumerate(_nets(m, raw0)):
        _, g64 = EO.step_grad(net, xs, xe, ys, perm[e, 0, :9], m.l1, n)
        tol = 1e-5 * float(g64.abs().max()) + 1e-7       # fp32 forward / backward over <= 24-term sums
        assert float((g[e].double() - g64).abs().max()) <= tol
        p32, mm, vv = EO.adam_update_f32(raw0[e].numpy(), g[e].numpy(), np.zeros(m.P, np.float32), np.zeros(m.P, np.float32), 1,
                                         m.lr)
        assert np.array_equal(m.params[e].cpu().numpy(), p32) and np.array_equal(m1[e].numpy(), mm)
        assert np.array_equal(m2[e].numpy(), vv)
    if m.rand_prior:       # prior biases start at 0, get a zero L1 gradient and never move
        sd = m.state_dicts()[0]
        assert all(float(sd[k].abs().max()) == 0 for k in sd if k.startswith("prior_net") and k.endswith("bias"))


def test_adam_lr_zero_and_500th_bias_correction():
    v = (True, False, "mixed", 1, 1)
    torch.manual_seed(1)
    Xc, Xe, y = _data(2, [4, 7], 1, 8, 2)
    m0, *_ = _model(v)
    raw0 = torch.stack([init_params(m0.layout) for _ in range(2)])
    perm = lambda T: torch.arange(8).repeat(2, T, 1).int()
    m, *_ = _model(v, num_epochs=3, batch_size=32, lr=0.0)
    _fit_with(m, Xc, Xe, y, raw0, perm(3))
    assert torch.equal(m.params.cpu(), raw0)
    a, *_ = _model(v, num_epochs=499, batch_size=32)
    _fit_with(a, Xc, Xe, y, raw0, perm(499))
    b, *_ = _model(v, num_epochs=500, batch_size=32)
    _fit_with(b, Xc, Xe, y, raw0, perm(500))
    am1, am2, _ = (t.cpu().numpy() for t in a.fit_state())
    bm1, bm2, bg = (t.cpu().numpy() for t in b.fit_state())
    for e in range(2):
        p, mm, vv = EO.adam_update_f32(a.params[e].cpu().numpy(), bg[e], am1[e], am2[e], 500, b.lr)
        assert np.array_equal(b.params[e].cpu().numpy(), p) and np.array_equal(bm1[e], mm) and np.array_equal(bm2[e], vv)


REF = load_golden("ref_deep_ensemble.npz")
REF_INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (0, [3, 5], "embedding"), (2, [3, 5], "onehot")]


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_three_epochs_track_the_reference_trajectory(vi):
    """3 epochs of fit_one from the reference's own initial weights over its own DataLoader order
    (tests/golden/make_ref_deep_ensemble.py), against the parameters the reference's fp32 fit reached."""
    p = f"v{vi}_"
    noise, prior, inp, O, L = (int(v) for v in REF[p + "cfg"])
    dc, uniqs, trans = REF_INPUTS[inp]
    m = DeepEnsemble(dc, len(uniqs), O, num_ensembles=2, num_epochs=3, batch_size=8, num_hiddens=8, num_layers=L,
                     output_noise=bool(noise), rand_prior=bool(prior), enum_trans=trans, num_uniqs=uniqs)
    Xc, Xe, y = (torch.from_numpy(REF[p + k]) for k in ("Xc", "Xe", "y"))
    _fit_with(m, Xc if dc else None, Xe if uniqs else None, y, torch.from_numpy(REF[p + "init"]),
              torch.from_numpy(REF[p + "order"]).int())
    if dc:      # same scalers as the reference's (sklearn's formulas restated)
        assert torch.allclose(m.xscaler.scale_, torch.from_numpy(REF[p + "x_scale"]), rtol=1e-6)
    assert torch.allclose(m.yscaler.std, torch.from_numpy(REF[p + "y_std"]), rtol=1e-6)
    steps = 3 * (int(torch.isfinite(y).any(1).sum()) // 8)
    for e in range(2):
        d = (m.params[e].cpu().double() - torch.from_numpy(REF[p + "epoch3"][e]).double()).abs()
        # both runs are fp32 with different summation orders, which alone moves a parameter by ~1e-5 here; Adam moves every
        # parameter by about lr per step whatever its gradient's size, so a near-zero gradient whose sign the rounding
        # flips moves that parameter the other way: allowed on at most 1 % of the elements, never beyond 2 lr per step
        assert float(d.max()) <= 2 * m.lr * steps
        assert float((d > 1e-4).double().mean()) <= 0.01, float(d.max())


def test_philox_order_is_deterministic_and_matches_the_restatement():
    v = (True, True, "mixed", 2, 2)
    Xc, Xe, y = _data(2, [4, 7], 2, 75, 4)
    n = int(torch.isfinite(y).any(1).sum())
    outs = []
    for _ in range(2):
        torch.manual_seed(5)
        m, *_ = _model(v, num_epochs=4, batch_size=16)
        m.fit(Xc, Xe, y)
        outs.append((m.params.cpu(), m.losses.cpu(), m.seed))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    torch.manual_seed(5)
    m, *_ = _model(v, num_epochs=4, batch_size=16)
    raw0 = torch.stack([init_params(m.layout) for _ in range(2)])
    perm = torch.tensor(np.stack([np.stack([EO.perm(outs[0][2], e, t, n) for t in range(4)]) for e in range(2)])).int()
    _fit_with(m, Xc, Xe, y, raw0, perm)
    assert torch.equal(m.params.cpu(), outs[0][0])


def test_default_fit_is_within_the_reference_rmse_spread():
    """Default DeepEnsemble (5 x 1 x 128, 500 epochs) at test_base_model.py's shapes on the data the reference was fitted
    on: train and held-out RMSE against the reference's three fits (rmse_ref [seed, (train, held-out)])."""
    ref = REF["rmse_ref"]
    got = []
    for s_ in range(3):
        X, y, Xt = (torch.from_numpy(REF[f"rmse_{k}{s_}"]) for k in ("X", "y", "Xt"))
        torch.manual_seed(s_)
        m = DeepEnsemble(1, 0, 1)
        m.fit(X, None, y)
        py, ps2 = m.predict(X, None)
        assert py.shape == (50, 1) and ps2.shape == (50, 1) and bool((ps2 > 0).all())
        got.append((float(((py - y) ** 2).mean().sqrt()), float(((m.predict(Xt, None)[0] - Xt ** 2) ** 2).mean().sqrt())))
    got = np.array(got)
    # median over the seeds within the reference's worst seed widened by half, every seed within twice it
    assert (np.median(got, 0) <= 1.5 * ref.max(0)).all() and (got <= 2 * ref.max(0)).all(), (got, ref)


def test_out_of_range_device_categories_give_nan_rows():
    torch.manual_seed(11)
    Xc, Xe, y = _data(2, [4, 7], 1, 40, 15)
    for trans in ("embedding", "onehot"):
        m = DeepEnsemble(2, 2, 1, num_uniqs=[4, 7], enum_trans=trans, num_ensembles=2, num_epochs=5)
        m.fit(Xc, Xe, y)
        xe = Xe.clone().int().cuda()
        xe[3, 0], xe[7, 1] = 4, -2_000_000_000          # outside the tables: the kernels must not read there
        mu, var = m.predict(Xc.cuda(), xe)
        ok = torch.ones(40, dtype=torch.bool)
        ok[[3, 7]] = False
        assert bool(torch.isnan(mu[[3, 7]]).all()) and bool(torch.isfinite(mu[ok.cuda()]).all())
        ref = m.predict(Xc[ok], Xe[ok])[0]
        assert torch.equal(mu[ok.cuda()].cpu(), ref)


def test_gradient_input_may_be_a_strided_view():
    torch.manual_seed(12)
    Xc, _, y = _data(3, [], 1, 40, 16)
    m = DeepEnsemble(3, 0, 1, num_ensembles=3, num_epochs=10)
    m.fit(Xc, None, y)
    wide = (torch.rand(30, 6) * 4 - 1).cuda()
    view = wide[:, ::2]                     # non-contiguous float32 device tensor
    a = view.clone().requires_grad_(True)
    b = view.detach().requires_grad_(True)
    assert not b.is_contiguous()
    pa, va = m.predict(a, None)
    pb, vb = m.predict(b, None)
    (pa.sum() + va.sum()).backward()
    (pb.sum() + vb.sum()).backward()
    assert torch.equal(pa, pb) and torch.equal(va, vb) and torch.equal(a.grad, b.grad)


@pytest.mark.parametrize("v", VARIANTS, ids=VID)
def test_predict_matches_fp64(v):
    torch.manual_seed(7)
    m, dc, uniqs, O = _model(v, E=3, num_epochs=20, batch_size=8)
    Xc, Xe, y = _data(dc, uniqs, O, 40, 8)
    m.fit(Xc, Xe, y)
    Xs, Xes, _ = _data(dc, uniqs, O, 1000, 9)
    xm, xa = (m.xscaler.scale_, m.xscaler.min_) if dc else (None, None)
    nets = _nets(m, m.params.cpu())
    with torch.no_grad():
        py64, ps64 = EO.ensemble_predict(nets, Xs, Xes, xm, xa, m.yscaler.mean, m.yscaler.std, m.output_noise)
    for rows in (slice(0, 1), slice(0, 15), slice(0, 16), slice(0, 17), slice(0, 1000)):
        py, ps2 = m.predict(Xs[rows] if dc else None, Xes[rows] if uniqs else None)
        ys = m.yscaler.std.double()
        assert float(((py.double() - py64[rows]).abs() / ys).max()) < 2e-5
        assert float(((ps2.double() - ps64[rows]).abs() / (ps64[rows].abs() + 1e-6 * ys ** 2)).max()) < 2e-4
    full = m.predict(Xs if dc else None, Xes if uniqs else None)
    part = m.predict(Xs[100:357] if dc else None, Xes[100:357] if uniqs else None)
    assert torch.equal(full[0][100:357], part[0]) and torch.equal(full[1][100:357], part[1])     # batching invariance


def test_single_member_and_mace():
    for noise in (True, False):
        torch.manual_seed(8)
        Xc, _, y = _data(3, [], 1, 40, 10)
        m = DeepEnsemble(3, 0, 1, num_ensembles=1, num_epochs=30, output_noise=noise, num_hiddens=32)
        m.fit(Xc, None, y)
        Xs = torch.rand(300, 3) * 4 - 1
        net = _nets(m, m.params.cpu())[0]
        with torch.no_grad():
            xs = Xs.double() * m.xscaler.scale_.double() + m.xscaler.min_.double()
            mu, s2 = net(xs, None)
        ps2 = m.predict(Xs, None)[1].double()
        ref = (s2 if noise else torch.full_like(mu, 1e-8)) * m.yscaler.std.double() ** 2
        assert float(((ps2 - ref).abs() / ref).max()) < 2e-4
        if noise:
            xi1, xi2 = torch.randn(300, 1), torch.randn(300, 1)
            F, mu_d, var_d = m.predict_mace(Xs.cuda(), 0.1, 2.0, 1e-4, xi1, xi2, return_mu_var=True)
            F2 = torch.empty_like(F)
            x1, x2 = xi1.cuda(), xi2.cuda()
            _lib.check(_lib.lib().hb_mace_epilogue(_lib.ptr(mu_d), _lib.ptr(var_d), 300, float(m.noise[0]), 0.1, 2.0, 1e-4,
                                                   _lib.ptr(x1), _lib.ptr(x2), 0, _lib.ptr(F2),
                                                   _lib.stream_ptr()), "mace")
            assert torch.equal(F, F2)


@pytest.mark.parametrize("v", [VARIANTS[i] for i in (0, 5, 10, 19, 26, 31)], ids=[VID[i] for i in (0, 5, 10, 19, 26, 31)])
def test_input_gradients_match_fp64_autograd(v):
    torch.manual_seed(9)
    m, dc, uniqs, O = _model(v, E=3, num_epochs=20, batch_size=8)
    if dc == 0:
        pytest.skip("no numeric column")
    Xc, Xe, y = _data(dc, uniqs, O, 40, 11)
    m.fit(Xc, Xe, y)
    Xs, Xes, _ = _data(dc, uniqs, O, 37, 12)
    X = Xs.clone().requires_grad_(True)
    py, ps2 = m.predict(X, Xes)
    w1, w2 = torch.randn(37, O), torch.randn(37, O)
    (py * w1 + ps2 * w2).sum().backward()
    X64 = Xs.double().requires_grad_(True)
    nets = _nets(m, m.params.cpu())
    py64, ps64 = EO.ensemble_predict(nets, X64, Xes, m.xscaler.scale_, m.xscaler.min_, m.yscaler.mean, m.yscaler.std,
                                     m.output_noise)
    (py64 * w1.double() + ps64 * w2.double()).sum().backward()
    scale = float(X64.grad.abs().max()) + 1e-6
    assert float((X.grad.double() - X64.grad).abs().max()) <= 1e-4 * scale
    assert torch.allclose(py.detach().double(), py64.detach(), rtol=1e-4, atol=1e-4)


def test_sample_f_warm_start_and_noise():
    torch.manual_seed(10)
    Xc, Xe, y = _data(2, [4, 7], 2, 60, 13)
    m = DeepEnsemble(2, 2, 2, num_uniqs=[4, 7], num_ensembles=3, num_epochs=30)
    m.fit(Xc, Xe, y)
    Xs, Xes, _ = _data(2, [4, 7], 2, 50, 14)
    nets = _nets(m, m.params.cpu())
    for k in range(4):
        f = m.sample_f()
        ref = EO.member_mu(nets[k % 3], Xs, Xes, m.xscaler.scale_, m.xscaler.min_, m.yscaler.mean, m.yscaler.std)
        assert torch.allclose(f(Xs, Xes).double(), ref.detach(), rtol=1e-4, atol=1e-4 * float(m.yscaler.std.max()))
    valid = torch.isfinite(y).any(1)
    py, _ = m.predict(Xc, Xe)
    # (py - y)[valid] keeps the NaN entry of a valid row, so that output's noise is NaN, as in the reference (:90-93)
    assert torch.allclose(m.noise, ((py - y)[valid] ** 2).mean(0), rtol=1e-6, equal_nan=True) and m.noise.shape == (2,)
    # warm start: the second fit starts from the current weights and keeps the scalers
    p1, sc = m.params.cpu().clone(), m.xscaler.scale_.clone()
    m.lr = 0.0
    m.fit(Xc * 3, Xe, y * 2)
    assert torch.equal(m.params.cpu(), p1) and torch.equal(m.xscaler.scale_, sc)


# ---------------------------------------------------------------- HEBO/test/test_base_model.py for 'deep_ensemble'
def test_reference_base_model_contract():
    Xc, Xe = torch.randn(50, 1), torch.randint(2, (50, 1))
    y = torch.randn(50, 1)
    for args, kw, xc, xe in (((1, 1, 1), dict(num_uniqs=[2]), Xc, Xe), ((1, 0, 1), {}, Xc, None), ((0, 1, 1), dict(num_uniqs=[2]), None, Xe)):
        m = DeepEnsemble(*args, num_epochs=1, **kw)
        m.fit(xc, xe, y)
        py, ps2 = m.predict(xc, xe)
        assert py.shape == (50, 1) and ps2.shape == (50, 1) and bool(torch.isfinite(py).all()) and bool((ps2 > 0).all())
    # NaN rows (test_fit_with_nan)
    y2 = y.clone()
    y2[0] = float("nan")
    m = DeepEnsemble(1, 0, 1, num_epochs=1)
    m.fit(Xc, None, y2)
    assert bool(torch.isfinite(m.predict(Xc, None)[0]).all())
    # Thompson sampling, grad, noise
    X = torch.randn(10, 1)
    m = DeepEnsemble(1, 0, 1, num_epochs=1)
    m.fit(X, None, X ** 2 + 1e-2 * torch.randn(10, 1))
    with torch.no_grad():
        assert m.sample_f()(X, None).shape == (10, 1)
    Xt = torch.randn(50, 1, requires_grad=True)
    m.predict(Xt, None)[0].sum().backward()
    assert Xt.grad is not None and Xt.grad.shape == (50, 1)
    assert m.noise.shape == (1,) and bool((m.noise >= 0).all())


# ---------------------------------------------------------------- HEBO/test/test_optimizer.py for 'deep_ensemble'
def _obj(x: pd.DataFrame) -> np.ndarray:
    return x["x0"].values.astype(float).reshape(-1, 1) ** 2


@pytest.mark.parametrize("opt_cls", [BO, HEBO, functools.partial(HEBO, acq_optimizer="nsga2", evo_iters=30),
                                     functools.partial(HEBO, acq_cls=MOMeanSigmaLCB)], ids=["bo", "hebo", "hebo-nsga2", "hebo-mo-lcb"])
def test_opt(opt_cls):
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    opt = opt_cls(space, rand_sample=8, model_name="deep_ensemble")
    for i in range(11):
        rec = opt.suggest(n_suggestions=1)
        y = _obj(rec)
        opt.observe(rec, y)
    assert opt.y.shape[0] == 11 and np.isfinite(opt.y).all()
    assert ((opt.X["x0"] >= -3) & (opt.X["x0"] <= 7)).all()


@pytest.mark.parametrize("opt_cls", [BO, HEBO], ids=["bo", "hebo"])
def test_best_xy(opt_cls):
    space = DesignSpace().parse([{"name": "x", "type": "num", "lb": 0, "ub": 1}])
    opt = opt_cls(space, rand_sample=100, model_name="deep_ensemble")
    with pytest.raises(RuntimeError):
        opt.best_x
    with pytest.raises(RuntimeError):
        opt.best_y
    rec = opt.suggest()
    y = rec["x"].values.reshape(-1, 1)
    opt.observe(rec, y)
    assert float(opt.best_y) == float(y.min())


def test_hebo_branin_beats_random():
    def branin(x):
        x1, x2 = x[:, 0] * 15 - 5, x[:, 1] * 15
        return ((x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x1) + 10)
    wins = 0
    for seed in range(3):
        torch.manual_seed(seed)
        np.random.seed(seed)
        opt = HEBO(torch.zeros(2), torch.ones(2), model_name="deep_ensemble", scramble_seed=seed)
        for _ in range(20):
            x = opt.suggest(1)
            opt.observe(x, branin(x.numpy()).reshape(-1, 1))
        rnd = branin(np.random.RandomState(100 + seed).rand(20, 2)).min()
        wins += opt.best_y < rnd
    assert wins >= 2
