"""Learned (and fixed) Kumaraswamy input warp fused into the kernels (SURVEY 8f-4, BASELINE config 3) against
oracle/warp_oracle.py: loss and the gradient of EVERY parameter incl. the 2 d warp exponents (fp64 autograd), the training
trajectory, the posterior (candidates are warped inside the K* load stage), input gradients through the warp."""
import numpy as np
import pytest
import torch

import hebo_b200
from oracle import warp_oracle as W
from tests.util import seeded_problem

pytestmark = pytest.mark.gpu


def _setup(n, d, kernel="matern32", **conf):
    X, y = seeded_problem(n, d, 40 + n)
    X = X * 1.5 + 0.2                                      # raw scale; MinMax maps it to [-1, 1]
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False, kernel=kernel, **conf)
    gp.fit(X, None, y)
    dt = torch.float64
    Xt = gp.xscaler.scale_.to(dt) * X.to(dt) + gp.xscaler.min_.to(dt)
    yt = (y.to(dt).reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    return gp, X, y, Xt, yt


@pytest.mark.parametrize("n,d,kernel", [(300, 4, "matern32"), (260, 7, "matern52"), (200, 3, "rbf"), (260, 5, "matern12")])
def test_learned_warp_loss_gradient_trajectory_posterior(n, d, kernel):
    gp, X, y, Xt, yt = _setup(n, d, kernel, warp=True)
    P = 3 + 3 * d
    assert gp.raw.numel() == P and gp.warp_mode == 1
    a0 = W.exponents(gp.raw_init[1:1 + d].double())
    assert torch.allclose(a0, torch.ones(d, dtype=torch.float64), atol=1e-5)          # identity at initialisation
    g = torch.Generator().manual_seed(1)
    for k in range(2):
        raw = gp.raw_init + (0.3 * torch.randn(P, generator=g) if k else 0.0)
        gp.set_hypers(raw)
        loss, grad = gp.evaluate_loss(return_grad=True)
        lo, go = W.neg_mll_autograd(Xt, yt, raw.double(), kind=kernel)
        assert abs(loss - float(lo)) <= 1e-4 * max(1.0, abs(float(lo))), (k, loss, float(lo))
        err = float((grad.double() - go).abs().max())
        assert err <= 1e-4 * max(float(go.abs().max()), 0.1), (k, err, (grad.double() - go).abs().argmax())
        assert float(go[1:1 + 2 * d].abs().max()) > 1e-5                               # the exponents do receive gradient
    # posterior at the perturbed hypers
    m = 700
    Xs = torch.rand(m, d, generator=g) * 3.4 - 1.6
    Xs[:30] = X[:30]
    mu, var = gp.predict(Xs, None)
    Xs_t = gp.xscaler.scale_.double() * Xs.double() + gp.xscaler.min_.double()
    mu_o, var_o = W.predict(Xt, yt, raw.double(), Xs_t, kind=kernel)
    ys, ym = float(gp.yscaler.std[0]), float(gp.yscaler.mean[0])
    mu_o, var_o = mu_o * ys + ym, var_o * ys ** 2
    emu = float(((mu.double().reshape(-1) - mu_o).abs() / mu_o.abs().clamp_min(ys)).max())
    esg = (var.double().reshape(-1).sqrt() - var_o.sqrt()).abs() / var_o.sqrt()
    print(f"warp {kernel}: mu err {emu:.2e} sigma err {float(esg.max()):.2e}")
    assert emu <= 1e-4 and float(esg[30:].max()) <= 1e-4 and float(esg.max()) <= 2e-4
    # input gradients chain through the warp
    xg = Xs[40:60].clone().requires_grad_(True)
    pm, pv = gp.predict(xg, None)
    (pm.sum() + pv.sum()).backward()
    xo = Xs[40:60].double().clone().requires_grad_(True)
    mo, vo = W.predict(Xt, yt, raw.double(), gp.xscaler.scale_.double() * xo + gp.xscaler.min_.double(), kind=kernel)
    ((mo * ys + ym).sum() + (vo * ys ** 2).sum()).backward()
    assert float((xg.grad.double() - xo.grad).abs().max()) <= 1e-3 * float(xo.grad.abs().max())
    # 30 RMSprop epochs move the exponents like the oracle's
    gp2 = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=30, noise_lb=8e-4, pred_likeli=False, kernel=kernel, warp=True, langevin=False,
                       init_raw=gp.raw_init.clone())
    gp2.fit(X, None, y)
    vec1, losses = W.fit_psgld(Xt, yt, gp.raw_init.double(), lr=0.01, num_epochs=30, kind=kernel, record=True)
    dl = float(np.abs(gp2.losses - np.array(losses)).max())
    dr = float((gp2.raw.double() - vec1).abs().max())
    print(f"warp {kernel}: trajectory loss diff {dl:.2e} raw diff {dr:.2e}; a moved by {float((W.exponents(vec1[1:1+d]) - 1).abs().max()):.3f}")
    tol = 5.0 if kernel == "rbf" else 1.0
    assert dl <= tol * 2e-4 * max(1.0, np.abs(losses).max()) and dr <= tol * 2e-3


def test_fixed_warp_is_frozen_and_matches_the_learned_machinery():
    """warp_a / warp_b: the same fused kernels with the exponents excluded from the optimiser (and from `raw`)."""
    n, d = 240, 4
    g = torch.Generator().manual_seed(3)
    wa, wb = 0.5 + 1.5 * torch.rand(d, generator=g), 0.5 + 1.5 * torch.rand(d, generator=g)
    gp, X, y, Xt, yt = _setup(n, d, warp_a=wa.tolist(), warp_b=wb.tolist())
    assert gp.warp_mode == 2 and gp.raw.numel() == d + 3
    full = gp._expand_raw(gp.raw_init)
    assert full.numel() == 3 + 3 * d and torch.allclose(W.exponents(full[1:1 + d].double()).float(), wa, atol=1e-5)
    loss, grad = gp.evaluate_loss(return_grad=True)
    lo, go = W.neg_mll_autograd(Xt, yt, full.double())
    assert abs(loss - float(lo)) <= 1e-4 * max(1.0, abs(float(lo)))
    keep = torch.cat([torch.arange(0, 1), torch.arange(1 + 2 * d, 3 + 3 * d)])
    assert grad.numel() == d + 3                              # the frozen exponents are not part of the gradient either
    assert float((grad.double() - go[keep]).abs().max()) <= 1e-4 * max(float(go.abs().max()), 0.1)
    lang = torch.randn(20, d + 3, generator=g)
    gp2 = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=False, warp_a=wa.tolist(), warp_b=wb.tolist(),
                       langevin=lang, init_raw=gp.raw_init.clone())
    gp2.fit(X, None, y)
    assert torch.equal(gp2._raw_dev.cpu()[1:1 + 2 * d], full[1:1 + 2 * d])            # never touched, Langevin noise included
    vec1 = W.fit_psgld(Xt, yt, full.double(), lr=0.01, num_epochs=20, langevin=gp2._expand_raw(lang).double(), frozen=(1, 1 + 2 * d))
    assert float((gp2._raw_dev.cpu().double() - vec1).abs().max()) <= 5e-3
