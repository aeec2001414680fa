"""High-dimensional and wide mixed-variable models (d + sum(emb_sizes) up to HB_MAX_FEATURES = 4096) against the fp64
oracles, with the criteria of tests/test_gpu_parity.py: the fit trajectory, mu / sigma (exact training rows included),
loss and gradient of one MLL forward + backward (learned warp, shared lengthscale, wide embeddings), input gradients,
posterior samples and HEBO.suggest.  The kernels stream features in 32-wide chunks, so the shapes here also put feature
counts on both sides of a chunk edge and the numeric / embedding boundary inside a chunk."""
import numpy as np
import pandas as pd
import pytest
import torch

import hebo_b200
from oracle import emb_oracle as E
from oracle import gp_oracle as O
from oracle import warp_oracle as W
from tests.util import emb_hypers, mu_sigma_errors, oracle_posterior, scaled_xy, seeded_problem

pytestmark = pytest.mark.gpu


def _kernel_matrix_blocked(X1, X2, ls, kind, block=256, fchunk=64):
    """O.kernel_matrix (direct differences, same dtype) with the [rows, n, d] difference tensor bounded to
    [block, n, fchunk] and evaluated with torch on the GPU: the oracle's own blocking holds n x 1024 x d at once."""
    dev = torch.device("cuda")
    Z1, Z2 = (X1 / ls).to(dev), (X2 / ls).to(dev)
    rows = []
    for i in range(0, Z1.shape[0], block):
        acc = torch.zeros(min(block, Z1.shape[0] - i), Z2.shape[0], dtype=Z1.dtype, device=dev)
        for k in range(0, Z1.shape[1], fchunk):
            diff = Z1[i:i + block, None, k:k + fchunk] - Z2[None, :, k:k + fchunk]
            acc = acc + (diff * diff).sum(-1)
        rows.append(acc)
    return O.kernel_from_sqdist(torch.cat(rows), kind).to(X1.device)


@pytest.fixture
def blocked_oracle(monkeypatch):
    monkeypatch.setattr(O, "kernel_matrix", _kernel_matrix_blocked)


@pytest.mark.parametrize("d", [128, 200])
def test_fit_trajectory_past_the_former_shared_memory_limit(d):
    """d >= 128 used to be rejected by the MLL gradient launcher (per-warp accumulators of 8 (3 d + 3) floats)."""
    n = 512
    X, y = seeded_problem(n, d, 7 + d)
    np.random.seed(1)
    conf = dict(lr=0.01, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp0 = hebo_b200.GP(d, 0, 1, num_epochs=0, **conf)
    gp0.fit(X, None, y)
    # start away from the optimum of the mean constant: its gradient vanishes at the default start (~1e-8 of the largest
    # here), and RMSprop's first step is +-10 lr whatever the gradient's size, i.e. it would follow the sign of fp32 noise
    raw0 = gp0.raw_init.clone()
    raw0[1] += 0.5
    gp = hebo_b200.GP(d, 0, 1, num_epochs=5, init_raw=raw0, **conf)
    gp.fit(X, None, y)
    Xt64, yt64 = scaled_xy(gp, X, y)
    hp0 = O.Hypers.unpack(raw0.double(), 8e-4)
    hp, losses = O.fit_psgld(Xt64, yt64, hp0, "matern32", lr=0.01, num_epochs=5, record=True)
    dl = np.abs(gp.losses - np.array(losses))
    # the same normalisation makes a lengthscale whose gradient is tiny against the largest one carry the fp32 error of
    # that gradient relative to ITSELF into its trajectory: 1e-4 for the parameters with a gradient above 1e-3 of the
    # largest, the 30-epoch bound of tests/test_gpu_emb.py for the rest
    _, g0, _ = O.neg_mll_closed_form(Xt64, yt64, hp0, "matern32")
    err = (hp.pack() - gp.raw.double()).abs()
    big = g0.abs() >= 1e-3 * float(g0.abs().max())
    print(f"d={d}: loss diff {dl.max():.2e}; 5-epoch raw diff {float(err[big].max()):.2e} ({int(big.sum())} parameters), "
          f"{float(err.max()):.2e} (all)")
    assert dl.max() <= 2e-4 * max(1.0, np.abs(losses).max())
    assert float(err[big].max()) < 1e-4 and float(err.max()) < 2e-3


POSTERIOR_CASES = [(1024, 233, "matern32"), (1024, 233, "rbf"), (1024, 1024, "matern32"), (1024, 1024, "rbf"),
                   (512, 4096, "matern32"), (512, 4096, "rbf"),
                   # feature counts on both sides of the 32-wide chunk edges
                   (700, 31, "matern32"), (700, 33, "matern52"), (700, 65, "matern32")]


@pytest.mark.parametrize("n,d,kind", POSTERIOR_CASES)
def test_posterior_parity_at_high_d(n, d, kind, blocked_oracle):
    X, y = seeded_problem(n, d, 100 + d)
    np.random.seed(2)
    gp = hebo_b200.GP(d, 0, 1, kernel=kind, lr=0.01, num_epochs=3, noise_lb=8e-4, pred_likeli=False, langevin=False,
                      m_chunk=128)
    gp.fit(X, None, y)
    Xt64, yt64 = scaled_xy(gp, X, y)
    f = O.FittedGP(Xt64, O.Hypers.unpack(gp.raw.double(), 8e-4), kind, gp.xscaler.scale_.double(), gp.xscaler.min_.double(),
                   float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]))
    f._yt = yt64
    O.refactor(f)
    m = 400
    g = torch.Generator().manual_seed(5)
    Xs = torch.rand(m, d, generator=g) * 2.4 - 1.2
    Xs[:50] = X[:50]                                   # exact training points: the sigma^2 cancellation case
    mu, var = gp.predict(Xs, None)
    mu64, var64 = O.predict(f, Xs.double())
    ys = float(gp.yscaler.std[0])
    emu, esg = mu_sigma_errors(mu, var, mu64.numpy().reshape(-1), var64.numpy().reshape(-1), ys)
    mu32, var32, _ = oracle_posterior(X, y, gp.raw, kind, Xs, torch.float32)
    fmu, fsg = mu_sigma_errors(mu32, var32, mu64.numpy().reshape(-1), var64.numpy().reshape(-1), ys)
    print(f"{kind} n={n} d={d}: GPU mu/sigma err {emu:.2e}/{esg:.2e}; fp32-reference floor {fmu:.2e}/{fsg:.2e}")
    assert emu <= max(1e-4, 2 * fmu) and esg <= max(1e-4, 2 * fsg), (emu, esg, fmu, fsg)
    gp.m_chunk = 8192                                  # chunking must not change a single bit
    mu_b, var_b = gp.predict(Xs, None)
    assert torch.equal(mu, mu_b) and torch.equal(var, var_b)
    gp.tensor_cores = False                            # FP32 SIMT contraction: same K* rows, same mean
    mu_s, var_s = gp.predict(Xs, None)
    assert torch.equal(mu_s, mu)
    assert float(((var_s.double().sqrt() - var64.sqrt()).abs() / var64.sqrt()).max()) <= max(1e-4, 2 * fsg)


def _mixed_problem(n, d, num_uniqs, seed):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, d, generator=g) * 4 - 1
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in num_uniqs], 1)
    y = torch.sin(2 * Xc[:, 0]) + 0.3 * Xc[:, -1] ** 2 + 0.05 * torch.randn(n, generator=g)
    for c in range(len(num_uniqs)):
        y = y + 0.4 * torch.cos(Xe[:, c].float() * (c + 1.3))
    return Xc, Xe, y.reshape(-1, 1)


def _check_loss_grad(gp, oracle, what, steps=(0.0, 0.25)):
    P = gp._param_layout()["P"]
    g = torch.Generator().manual_seed(3)
    for sc in steps:
        raw = gp.raw_init + sc * torch.randn(P, generator=g)
        gp.set_hypers(raw)
        loss, grad = gp.evaluate_loss(return_grad=True)
        lo, go = oracle(raw)
        assert abs(loss - float(lo)) <= 1e-4 * max(1.0, abs(float(lo))), (what, sc, loss, float(lo))
        err = float((grad.double() - go).abs().max())
        print(f"{what}: loss {loss:.6f} vs {float(lo):.6f}, gradient err {err:.2e} of {float(go.abs().max()):.2e}")
        assert err <= 1e-4 * max(float(go.abs().max()), 0.1), (what, sc, err)
    return raw


@pytest.mark.parametrize("name,n,d,nu", [("wide_embeddings", 300, 8, [120] * 6), ("boundary_inside_chunk", 400, 20, [30, 9])])
def test_mixed_model_loss_gradient_posterior(name, n, d, nu):
    """8 numeric columns + 6 categoricals of 120 categories (De = 6 x 50 = 300), and a model whose numeric / embedding
    boundary (d = 20, De = 16 + 5) falls inside the first 32-wide chunk, against oracle/emb_oracle.py."""
    Xc, Xe, y = _mixed_problem(n, d, nu, 50 + n)
    torch.manual_seed(1)
    np.random.seed(1)
    gp = hebo_b200.GP(d, len(nu), 1, num_uniqs=nu, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False)
    gp.fit(Xc, Xe, y)
    if name == "wide_embeddings":
        assert gp.De == 300
    Xt, yt = scaled_xy(gp, Xc, y)
    raw = _check_loss_grad(gp, lambda r: E.neg_mll_emb_closed_form(Xt, Xe.long(), yt, emb_hypers(gp, r)), name)
    m = 300
    g = torch.Generator().manual_seed(9)
    Xs_c = torch.rand(m, d, generator=g) * 4.4 - 1.2
    Xs_e = torch.stack([torch.randint(0, u, (m,), generator=g) for u in nu], 1)
    Xs_c[:50], Xs_e[:50] = Xc[:50], Xe[:50]
    mu, var = gp.predict(Xs_c, Xs_e)
    Xs_t = gp.xscaler.scale_.double() * Xs_c.double() + gp.xscaler.min_.double()
    mu_o, var_o = E.predict_emb(Xt, Xe.long(), yt, emb_hypers(gp, raw), Xs_t, Xs_e.long())
    ys, ym = float(gp.yscaler.std[0]), float(gp.yscaler.mean[0])
    mu_o, var_o = mu_o * ys + ym, var_o * ys ** 2
    emu = float(((mu.double().reshape(-1) - mu_o).abs() / mu_o.abs().clamp_min(ys)).max())
    esg = float(((var.double().reshape(-1).sqrt() - var_o.sqrt()).abs() / var_o.sqrt()).max())
    print(f"{name}: mu err {emu:.2e} sigma err {esg:.2e}")
    assert emu <= 1e-4 and esg <= 1e-4, (emu, esg)


def test_learned_warp_loss_gradient_at_d300():
    n, d = 200, 300
    X, y = seeded_problem(n, d, 61)
    X = X * 1.5 + 0.2
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False, warp=True)
    gp.fit(X, None, y)
    Xt, yt = scaled_xy(gp, X, y)
    _check_loss_grad(gp, lambda r: W.neg_mll_autograd(Xt, yt, r.double()), "warp d=300", steps=(0.0, 0.3))


def test_shared_lengthscale_loss_gradient_at_d1024():
    n, d = 160, 1024
    X, y = seeded_problem(n, d, 62)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False, ard_kernel=False)
    gp.fit(X, None, y)
    Xt, yt = scaled_xy(gp, X, y)
    _check_loss_grad(gp, lambda r: E.neg_mll_emb_closed_form(Xt, torch.zeros(n, 0).long(), yt, emb_hypers(gp, r)),
                     "ard_kernel=False d=1024")


def test_input_gradients_and_samples_at_d1024(blocked_oracle):
    n, d, m = 300, 1024, 40
    X, y = seeded_problem(n, d, 63)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=5, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, None, y)
    g = torch.Generator().manual_seed(4)
    Xs = X[:m] + 0.05 * torch.randn(m, d, generator=g)
    Xs[:5] = X[:5]
    wm, wv = torch.randn(m, 1, generator=g), torch.randn(m, 1, generator=g)
    xa = Xs.clone().requires_grad_(True)
    mu1, var1 = gp.predict(xa, None)
    ((wm * mu1).sum() + (wv * var1).sum()).backward()
    dt = torch.float64
    Xt, yt = scaled_xy(gp, X, y)
    xb = Xs.to(dt).clone().requires_grad_(True)
    f = O.FittedGP(Xt, O.Hypers.unpack(gp.raw.to(dt), 8e-4), "matern32", torch.ones(d, dtype=dt), torch.zeros(d, dtype=dt),
                   float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]))
    f._yt = yt
    O.refactor(f)
    mu2, var2 = O.predict(f, gp.xscaler.scale_.to(dt) * xb + gp.xscaler.min_.to(dt))
    ((wm.to(dt) * mu2).sum() + (wv.to(dt) * var2).sum()).backward()
    ys = float(gp.yscaler.std[0])
    emu = float(((mu1.detach().double() - mu2.detach()).abs() / mu2.detach().abs().clamp_min(ys)).max())
    esg = ((var1.detach().double().sqrt() - var2.detach().sqrt()).abs() / var2.detach().sqrt()).reshape(-1)
    assert emu <= 1e-4 and float(esg[5:].max()) <= 1e-4 and float(esg[:5].max()) <= 5e-4, (emu, esg.max())
    ga, gb = xa.grad.double(), xb.grad
    scale, gerr = float(gb.abs().max()), float((ga - gb).abs().max())
    print(f"d=1024: input-gradient err {gerr / scale:.2e} of the gradient scale")
    assert torch.isfinite(ga).all() and gerr <= 1e-4 * scale, (gerr, scale)
    # joint posterior samples: empirical moments against predict()
    S = 4000
    with torch.no_grad():
        mu, var = gp.predict(Xs, None)
    torch.manual_seed(7)
    samp = gp.sample_y(Xs, None, S)
    assert samp.shape == (S, m, 1) and torch.isfinite(samp).all()
    sm, sv = samp.mean(0).reshape(-1), samp.var(0).reshape(-1)
    assert float(((sm - mu.reshape(-1)).abs() / var.reshape(-1).sqrt()).max()) < 5.0 / np.sqrt(S) * 1.5
    assert float((sv / (var.reshape(-1) + gp.sample_jitter * gp._y_std ** 2) - 1).abs().max()) < 0.15


def _check_rows(Xs, space_rows, q):
    assert len(Xs) == q
    assert not Xs.duplicated().any()
    for col, lo, hi in space_rows:
        v = Xs[col].to_numpy(dtype=float)
        assert np.isfinite(v).all() and (v >= lo).all() and (v <= hi).all(), col


@pytest.mark.parametrize("acq", ["sobol", "nsga2"])
def test_hebo_suggest_on_a_wide_mixed_space(acq):
    """300 numeric columns and two categoricals of 120 choices (De = 100): three rounds of q = 8."""
    from hebo_b200.suggest import HEBO
    d, cats = 300, [[f"c{i}" for i in range(120)], [f"k{i}" for i in range(120)]]
    spec = [{"name": f"x{i}", "type": "num", "lb": -2.0, "ub": 3.0} for i in range(d)]
    spec += [{"name": "u", "type": "cat", "categories": cats[0]}, {"name": "v", "type": "cat", "categories": cats[1]}]
    rows = [(f"x{i}", -2.0, 3.0) for i in range(d)]

    def f(df):
        x = df[[f"x{i}" for i in range(d)]].to_numpy(dtype=float)
        iu = df["u"].map({c: i for i, c in enumerate(cats[0])}).to_numpy(dtype=float)
        iv = df["v"].map({c: i for i, c in enumerate(cats[1])}).to_numpy(dtype=float)
        return (np.sin(x[:, :10]).sum(1) + 0.01 * (x ** 2).sum(1) + 0.3 * np.cos(iu / 7) - 0.2 * np.sin(iv / 5)).reshape(-1, 1)

    torch.manual_seed(0)
    np.random.seed(0)
    # (no Langevin term: with 64 rows in 302 columns most lengthscale gradients vanish, and pSGLD's noise on a parameter
    # with a vanishing gradient random-walks it until the fit gives up -- sgld.py:64-70, the reference does the same)
    opt = HEBO(spec, rand_sample=20, scramble_seed=3, acq_optimizer=acq, evo_pop=64, evo_iters=10,
               model_config={"lr": 0.01, "num_epochs": 20, "noise_lb": 8e-4, "pred_likeli": False, "langevin": False})
    X0 = opt.quasi_sample(64)
    opt.observe(X0, f(X0))
    for _ in range(3):
        X = opt.suggest(8)
        assert not opt.model._fit_failed and np.isfinite(opt.model.losses).all()
        assert isinstance(X, pd.DataFrame)
        _check_rows(X, rows, 8)
        assert set(X["u"]) <= set(cats[0]) and set(X["v"]) <= set(cats[1])
        opt.observe(X, f(X))
    assert opt.Xc.shape[0] == 64 + 24


def test_hebo_box_suggest_at_d1024():
    from hebo_b200.suggest import HEBO
    d = 1024
    lb, ub = -torch.ones(d), 2 * torch.ones(d)
    torch.manual_seed(0)
    np.random.seed(0)
    opt = HEBO(lb, ub, rand_sample=10, scramble_seed=5, model_config={"lr": 0.01, "num_epochs": 20, "noise_lb": 8e-4,
                                                                       "pred_likeli": False, "langevin": False})
    X0 = opt.quasi_sample(64)
    opt.observe(X0, (X0[:, :8] ** 2).sum(1).numpy())
    X = opt.suggest(8)
    assert not opt.model._fit_failed and np.isfinite(opt.model.losses).all()
    assert X.shape == (8, d) and torch.isfinite(X).all() and bool(((X >= lb) & (X <= ub)).all())
    assert torch.unique(X, dim=0).shape[0] == 8
